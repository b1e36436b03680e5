"""GPU: one training step on the hand-written kernels (TrainStep.forward_backward) against PyTorch autograd
(train_path.pointnet_det_torch) on the same weights, for detection workloads that no other whole-step comparison
covers: people (PointNet layers of 22 400 rows: the 256-row reduction and the 1024-row dW slices) and SUN-RGBD
(5 scales, the 8x transposed conv, 10 one-hot columns).

The reference is autograd in FLOAT64 (model and inputs in float64; the grouping, which selects integer indices,
runs on the fp32 coordinates, and the first PointNet layer reads the fp32 relative coordinates, exactly as the
kernels see them), so the comparison measures the error of the fp32 kernels alone and does not depend on the
summation order of a second fp32 implementation.  The fp32 autograd step (TF32 off) is run too and its error
against float64 is printed next to the kernels' error.

Bounds, against float64: losses 1e-4 * max(1, |loss|); every parameter gradient 2e-3 * max(1e-3, max|g|) per element
and 2e-4 * rms(g) + 2e-6 in RMS (the same absolute floor as the per-element bound: tensors whose gradient is that
small, such as the BN shifts of a layer feeding a max-pool, differ by whole ReLU decisions near 0); running
statistics 1e-4 * max(1, max|ref|); num_batches_tracked = 1.

Measured worst error / bound over all gradient tensors and the losses, fourteen runs per case (H100 80GB HBM3, 400 W
power limit): people 0.25-0.47 and SUN-RGBD 0.26-0.46 (both on feat_net.pointnet2.conv3.1.bias; fp32 autograd 0.63
and 0.55 on the same tensor).

The car workload is checked layer by layer in test_gpu_train_layers.py (every layer of a car B=2 step at full depth
against float64 from the layer's own inputs).  A whole car step is not compared here: at 17.5 m, B=4, the first
PointNet layer's weight and BN-scale gradients exceeded the bound by 4-5.5x in 2 of 18 runs while all other runs
stayed within 0.6 of it, and that run-to-run excursion is not yet explained.
"""
import pytest
import torch

import train_ref as tr

pytestmark = pytest.mark.gpu

@pytest.fixture
def no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _float64_model(wl, seed):
    m = tr.make_model(wl, seed).double()
    for mod in m.modules():
        if type(mod).__name__ == "QueryDepthPoint":     # grouping on the fp32 coordinates the kernels group
            mod.register_forward_pre_hook(lambda _m, args: tuple(a.float() for a in args))
        if type(mod).__name__ == "PointNetModule":
            # the kernels' first-layer input is the fp32 difference point - section centre: start from the same
            # values (the first layer's weight gradient cancels and would magnify this input rounding)
            mod.conv1.register_forward_pre_hook(lambda _m, args: (args[0].float().double(),))
    return m


def _grad_errors(pref, pgot):
    """-> {name: (max error / bound, rms error / bound)}."""
    out = {}
    for k, p in pref.items():
        gr, gg = p.grad.double(), pgot[k].grad.double()
        d = gg - gr
        out[k] = (float(d.abs().max()) / (2e-3 * max(1e-3, float(gr.abs().max()))),
                  float(d.pow(2).mean().sqrt()) / (2e-4 * float(gr.pow(2).mean().sqrt()) + 2e-6))
    return out


@pytest.mark.parametrize("wl,B,md", [("people", 2, 7.0), ("sunrgbd", 3, None)])
def test_train_step_matches_float64_autograd(wl, B, md, no_tf32):
    from frustum_convnet_b200 import synth, train_path
    from frustum_convnet_b200.train_engine import TrainStep
    data = {k: torch.from_numpy(v).cuda() for k, v in synth.make_frustums(wl, B, seed=90 + B, max_depth=md,
                                                                            with_labels=True).items()}
    m64 = _float64_model(wl, 31)
    l64, _ = train_path.pointnet_det_torch(m64, {k: (v.double() if v.is_floating_point() else v)
                                                  for k, v in data.items()})
    l64["total_loss"].backward()
    m32 = tr.make_model(wl, 31)
    l32, _ = train_path.pointnet_det_torch(m32, data)
    l32["total_loss"].backward()
    mk = tr.make_model(wl, 31)
    lk, _ = TrainStep(mk).forward_backward(data)
    torch.cuda.synchronize()
    worst = 0.0
    for k in l64:
        ref = float(l64[k].detach())
        r = abs(float(lk[k]) - ref) / (1e-4 * max(1.0, abs(ref)))
        worst = max(worst, r)
        assert r <= 1.0, (k, float(lk[k]), ref)
    p64 = dict(m64.named_parameters())
    ek = _grad_errors(p64, dict(mk.named_parameters()))
    e32 = _grad_errors(p64, dict(m32.named_parameters()))
    for k, (em, er) in ek.items():
        assert em <= 1.0, (k, "max", em)
        assert er <= 1.0, (k, "rms", er)
    wk = max(ek, key=lambda k: max(ek[k]))
    w32 = max(e32, key=lambda k: max(e32[k]))
    worst = max(worst, max(ek[wk]))
    print("%s B=%d worst error / bound: kernels %.3f (%s), losses included; fp32 autograd %.3f (%s)"
          % (wl, B, worst, wk, max(e32[w32]), w32))
    b64, bk = dict(m64.named_buffers()), dict(mk.named_buffers())
    for k in b64:
        if k.endswith("num_batches_tracked"):
            assert int(b64[k]) == int(bk[k]) == 1, k
        else:
            assert float((b64[k] - bk[k].double()).abs().max()) <= 1e-4 * max(1.0, float(b64[k].abs().max())), k
