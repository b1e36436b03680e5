"""Host logic of the training path on the CPU (no CUDA): TrainStep's one loss path is the fused kernel, and the flat
parameter bucket keeps nn.Module / optimizer semantics."""
import numpy as np
import torch

from frustum_convnet_b200 import config, synth


def _model():
    from frustum_convnet_b200.det_base import PointNetDet
    cfg, w = config.load_workload("refine_car")
    sd = synth.make_state_dict(w["arch"], 3, "KITTI", seed=11)
    m = PointNetDet(3, num_vec=3)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m, cfg


def test_loss_impl_is_the_fused_kernel_and_read_only():
    from frustum_convnet_b200.train_engine import TrainStep
    prop = TrainStep.__dict__["loss_impl"]
    assert isinstance(prop, property) and prop.fset is None
    assert prop.fget(None) == "kernel"


def test_flat_parameter_bucket_semantics():
    from frustum_convnet_b200.train_engine import FlatParams
    m, _ = _model()
    before = {k: v.detach().clone() for k, v in m.state_dict().items()}
    FlatParams.__init__.__globals__["torch"]          # (import check)
    m_cuda_like = m                                   # FlatParams asserts CUDA: emulate with a CPU variant
    ps = list(m_cuda_like.parameters())

    class CpuFlat(FlatParams):
        def __init__(self, module):
            ps_ = [p for p in module.parameters()]
            n = sum(p.numel() for p in ps_)
            self.param = torch.empty(n)
            self.grad = torch.zeros(n)
            self.offsets, off = {}, 0
            for p in ps_:
                k = p.numel()
                self.param[off: off + k].copy_(p.data.reshape(-1))
                p.data = self.param[off: off + k].view(p.shape)
                self.offsets[id(p)] = off
                off += k
            self.numel = n

    flat = CpuFlat(m)
    assert flat.numel == 3316777 == sum(p.numel() for p in ps)
    for k, v in m.state_dict().items():               # values unchanged, names unchanged
        assert torch.equal(v, before[k]), k
    # parameters are views of the bucket: an in-place update of the bucket is what the module sees
    first = next(m.parameters())
    flat.param[:first.numel()].add_(1.0)
    assert torch.equal(first.detach().reshape(-1), before[next(iter(before))].reshape(-1) + 1.0)
    # gradient views tile the bucket without gaps, in parameter order (feat_net first, conv_net + heads last)
    off = 0
    for p in m.parameters():
        assert flat.offsets[id(p)] == off
        assert flat.grad_view(p).shape == p.shape
        off += p.numel()
    split = flat.offsets[id(next(m.conv_net.parameters()))]
    assert 0 < split < flat.numel and split == sum(p.numel() for p in m.feat_net.parameters())
    # a stock optimizer built on the SAME Parameter objects keeps working after the re-pointing
    flat.expose_grads(m)
    flat.grad.fill_(0.5)
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    w0 = flat.param.clone()
    opt.step()
    assert torch.allclose(flat.param, w0 - 0.05)
