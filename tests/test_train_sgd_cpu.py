"""CPU: the fused SGD entry (fcn_sgd_step) - argument validation before any CUDA call and a kernel without stack
frame or spills - and TrainStep.optimizer's torch state-dict handling for SGD (train_engine.FlatSGD) on a CPU
stand-in for the flat parameter bucket: torch.optim.SGD states load into the flat momentum buffer and come back in
torch's format, and states the fused step cannot continue are rejected with the optimizer left as it was."""
import io

import numpy as np
import pytest
import torch

from toolchain import compile_cuda


def test_sgd_step_rejects_bad_arguments_before_any_launch():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    buf = np.zeros(64, dtype=np.float32)
    p = buf.ctypes.data
    cases = [((None, p, p, 4, 0.9), b"NULL"), ((p, None, p, 4, 0.9), b"NULL"), ((p, p, None, 4, 0.9), b"momentum"),
             ((p, p, p, -1, 0.9), b"n < 0"), ((None, p, None, -1, 0.0), b"NULL")]
    for (pp, gg, bb, n, mom), word in cases:
        assert lib.fcn_sgd_step(pp, gg, bb, n, 1e-2, mom, 0.0, 0, 1.0, None) == -1, (pp, gg, bb, n, mom)
        assert word in lib.fcn_last_error(), (pp, gg, bb, n, mom, lib.fcn_last_error())
    assert lib.fcn_sgd_step(p, p, None, 0, 1e-2, 0.0, 1e-4, 0, 1.0, None) == 0      # no buffer without momentum
    assert lib.fcn_sgd_step(p, p, p, 0, 1e-2, 0.9, 1e-4, 1, 1.0, None) == 0         # n == 0: nothing to launch
    with pytest.raises(RuntimeError, match="momentum_buffer"):
        _lib.call("fcn_sgd_step", p, p, None, 4, 1e-2, 0.9, 0.0, 1, 1.0, None)


def test_sgd_kernel_has_no_stack_frame_or_spills():
    usage = {m: k.local_memory for m, k in compile_cuda("train.cu").kernels.items()}
    found = [v for k, v in usage.items() if "train_sgd_kernel" in k]
    assert found == [(0, 0, 0)], usage


class _CpuFlat:
    """The two attributes of FlatParams that FlatSGD reads, for CPU parameters."""

    def __init__(self, module):
        ps = list(module.parameters())
        self.param = torch.cat([p.detach().reshape(-1) for p in ps])
        self.offsets, off = {}, 0
        for p in ps:
            self.offsets[id(p)] = off
            off += p.numel()


def _module(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(5, 4), torch.nn.ReLU(), torch.nn.Linear(4, 3))


def _grads(module, scale):
    for p in module.parameters():
        p.grad = torch.randn_like(p) * scale


def _torch_sgd_after(steps, module, momentum=0.9, **kw):
    opt = torch.optim.SGD(module.parameters(), lr=2e-2, momentum=momentum, weight_decay=1e-4, **kw)
    for i in range(steps):
        _grads(module, i + 1)
        opt.step()
    return opt


def _roundtrip(sd):
    f = io.BytesIO()
    torch.save(sd, f)
    f.seek(0)
    return torch.load(f)


def _flat_sgd(module, **kw):
    from frustum_convnet_b200.train_engine import FlatSGD
    return FlatSGD(module, _CpuFlat(module), **kw)


def test_torch_sgd_state_loads_into_the_flat_buffer_and_saves_back():
    src = _module()
    opt = _torch_sgd_after(3, src)
    mine = _module(1)
    fs = _flat_sgd(mine)
    assert fs.state_dict()["state"] == {} and not fs.has_buffers
    fs.load_state_dict(_roundtrip(opt.state_dict()))
    assert fs.has_buffers
    g = fs.param_groups[0]
    assert (g["lr"], g["momentum"], g["weight_decay"], g["dampening"]) == (2e-2, 0.9, 1e-4, 0)
    for p, q in zip(mine.parameters(), src.parameters()):
        off, n = fs.flat.offsets[id(p)], p.numel()
        assert torch.equal(fs.momentum_buffer[off:off + n], opt.state[q]["momentum_buffer"].reshape(-1))
        assert fs.state[p]["momentum_buffer"].data_ptr() == fs.momentum_buffer[off:].data_ptr()   # flat views
    back = fs.state_dict()
    ref = opt.state_dict()
    assert back["param_groups"] == ref["param_groups"]
    assert sorted(back["state"]) == sorted(ref["state"])
    for k, st in ref["state"].items():
        assert list(back["state"][k]) == ["momentum_buffer"]
        assert torch.equal(back["state"][k]["momentum_buffer"], st["momentum_buffer"])
    fs.load_state_dict(torch.optim.SGD(_module(3).parameters(), lr=0.1, momentum=0.9).state_dict())  # never stepped
    assert not fs.has_buffers and fs.state_dict()["state"] == {} and not fs.momentum_buffer.any()
    assert fs.param_groups[0]["lr"] == 0.1


def test_momentum_zero_states_load_as_no_buffers():
    src = _module()
    sd = _roundtrip(_torch_sgd_after(2, src, momentum=0.0).state_dict())
    assert sd["state"] == {}
    mine = _module(1)
    fs = _flat_sgd(mine, momentum=0.9)
    fs.momentum_buffer.fill_(0.5)
    fs.has_buffers = True
    fs._bind()
    fs.load_state_dict(sd)
    assert not fs.has_buffers and fs.state_dict()["state"] == {} and not fs.momentum_buffer.any()
    assert fs.param_groups[0]["momentum"] == 0.0
    old = _roundtrip(sd)                                    # torch < 2 stored a None buffer per parameter
    old["state"] = {k: {"momentum_buffer": None} for k in old["param_groups"][0]["params"]}
    fs.load_state_dict(old)
    assert not fs.has_buffers and fs.state_dict()["state"] == {}


def test_loading_the_optimizers_own_state_keeps_its_buffers():
    """torch keeps a loaded tensor that already has the parameter's dtype and device, so loading an optimizer's own
    state_dict() hands the loader views of the flat buffer itself; torch.optim.SGD treats that load as a no-op."""
    src = _module()
    ref = _torch_sgd_after(2, src)
    want = [ref.state[p]["momentum_buffer"].clone() for p in src.parameters()]
    ref.load_state_dict(ref.state_dict())
    assert all(torch.equal(ref.state[p]["momentum_buffer"], w) for p, w in zip(src.parameters(), want))
    mine = _module(1)
    fs = _flat_sgd(mine, momentum=0.9)
    fs.load_state_dict(_roundtrip(ref.state_dict()))
    before = fs.momentum_buffer.clone()
    assert before.abs().max() > 0
    fs.load_state_dict(fs.state_dict())
    assert fs.has_buffers and torch.equal(fs.momentum_buffer, before)
    assert all(fs.state[p]["momentum_buffer"].data_ptr() == b.data_ptr() for p, b in fs._views())
    fs.momentum_buffer.fill_(0.5)
    fs.load_state_dict(fs.state_dict())
    assert fs.has_buffers and bool((fs.momentum_buffer == 0.5).all())


def _rejects(sd, match):
    mine = _module(1)
    fs = _flat_sgd(mine, lr=5e-4, momentum=0.8)
    fs.momentum_buffer.fill_(0.5)
    fs.has_buffers = True
    fs._bind()
    before = fs.state_dict()
    with pytest.raises(ValueError, match=match):
        fs.load_state_dict(sd)
    after = fs.state_dict()
    assert after["param_groups"] == before["param_groups"] and fs.has_buffers
    assert bool((fs.momentum_buffer == 0.5).all())
    assert all(fs.state[p]["momentum_buffer"].data_ptr() == b.data_ptr() for p, b in fs._views())


def test_states_the_fused_step_cannot_continue_are_rejected():
    src = _module()
    sd = _torch_sgd_after(2, src).state_dict()
    some = _roundtrip(sd)
    del some["state"][1]
    _rejects(some, "momentum buffers on 3 of 4 parameters")
    adam = torch.optim.Adam(src.parameters(), lr=1e-3)
    adam.step()                                             # the grads of _torch_sgd_after are still there
    _rejects(adam.state_dict(), "no momentum .not an SGD state")
    adam_state = _roundtrip(sd)
    adam_state["state"] = adam.state_dict()["state"]
    _rejects(adam_state, "parameter 0: the loaded state has exp_avg / exp_avg_sq / step .not an SGD state")
    other = torch.nn.Sequential(torch.nn.Linear(5, 4), torch.nn.ReLU(), torch.nn.Linear(4, 2))
    _rejects(_torch_sgd_after(1, other).state_dict(), "shape")
    two = torch.optim.SGD([{"params": list(src[0].parameters())}, {"params": list(src[2].parameters())}], lr=0.1)
    _rejects(two.state_dict(), "2 parameter groups")
    fewer = torch.optim.SGD(list(src[0].parameters()), lr=0.1).state_dict()
    _rejects(fewer, "2 parameters, the model has 4")
    for flag, value in (("nesterov", True), ("dampening", 0.1), ("maximize", True)):
        bad = _roundtrip(sd)
        bad["param_groups"][0][flag] = value
        _rejects(bad, flag)


def test_step_rechecks_the_group():
    mine = _module(1)
    fs = _flat_sgd(mine, momentum=0.9)
    for flag, value in (("nesterov", True), ("dampening", 0.5), ("maximize", True)):
        fs.param_groups[0][flag] = value
        with pytest.raises(ValueError, match=flag):
            fs.step()
        fs.param_groups[0][flag] = type(value)(0)
    assert fs.step_count == 0 and not fs.has_buffers


def test_train_step_rejects_an_unknown_optimizer_before_touching_the_model():
    from frustum_convnet_b200.train_engine import TrainStep
    mine = _module(1)
    with pytest.raises(ValueError, match="'rmsprop' is not supported"):
        TrainStep(mine, optimizer="rmsprop")
    assert not hasattr(mine, "_flat_params")
