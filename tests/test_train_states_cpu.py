"""CPU: the training meters' C entry (fcn_train_states_append) - argument validation before any CUDA call and a
kernel without stack frame or spills - and TrainStep.optimizer's torch state-dict handling (train_engine.FlatAdam)
on a CPU stand-in for the flat parameter bucket: torch.optim.Adam states load into the flat moments and come back
in torch's format, and states the fused step cannot continue are rejected with the optimizer left as it was."""
import io

import numpy as np
import pytest
import torch

from toolchain import compile_cuda


def test_append_rejects_bad_arguments_before_any_launch():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    buf = np.zeros(64, dtype=np.float32)
    p = buf.ctypes.data
    cases = [((None, 4, p, 8, p), b"NULL"), ((p, 4, None, 8, p), b"NULL"), ((p, 4, p, 8, None), b"NULL"),
             ((p, 4, p, 0, p), b"capacity"), ((p, 4, p, -3, p), b"capacity"), ((p, 0, p, 8, p), b"B"),
             ((p, -1, p, 8, p), b"B")]
    for args, word in cases:
        assert lib.fcn_train_states_append(*args, None) == -1, args
        assert word in lib.fcn_last_error(), (args, lib.fcn_last_error())
    with pytest.raises(RuntimeError, match="capacity"):
        _lib.call("fcn_train_states_append", p, 4, p, 0, p, None)


def test_append_kernel_has_no_stack_frame_or_spills():
    usage = {m: k.local_memory for m, k in compile_cuda("validate.cu").kernels.items()}
    for name in ("train_states_append_kernel", "val_final_kernel"):      # both append through one helper
        found = [v for k, v in usage.items() if name in k]
        assert found == [(0, 0, 0)], (name, usage)


class _CpuFlat:
    """The two attributes of FlatParams that FlatAdam reads, for CPU parameters."""

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


def _torch_adam_after(steps, module):
    opt = torch.optim.Adam(module.parameters(), lr=2e-3, betas=(0.8, 0.99), eps=1e-7, weight_decay=1e-4)
    for i in range(steps):
        for p in module.parameters():
            p.grad = torch.randn_like(p) * (i + 1)
        opt.step()
    return opt


def _roundtrip(sd):
    f = io.BytesIO()
    torch.save(sd, f)
    f.seek(0)
    return torch.load(f)


def test_torch_adam_state_loads_into_the_flat_moments_and_saves_back():
    from frustum_convnet_b200.train_engine import FlatAdam
    src = _module()
    opt = _torch_adam_after(3, src)
    mine = _module(1)
    fa = FlatAdam(mine, _CpuFlat(mine))
    fa.load_state_dict(_roundtrip(opt.state_dict()))
    assert fa.step_count == 3
    g = fa.param_groups[0]
    assert (g["lr"], tuple(g["betas"]), g["eps"], g["weight_decay"]) == (2e-3, (0.8, 0.99), 1e-7, 1e-4)
    for p, q in zip(mine.parameters(), src.parameters()):
        off, n = fa.flat.offsets[id(p)], p.numel()
        assert torch.equal(fa.exp_avg[off:off + n], opt.state[q]["exp_avg"].reshape(-1))
        assert torch.equal(fa.exp_avg_sq[off:off + n], opt.state[q]["exp_avg_sq"].reshape(-1))
        assert fa.state[p]["exp_avg"].data_ptr() == fa.exp_avg[off:].data_ptr()       # views of the flat buffer
    back = fa.state_dict()
    ref = opt.state_dict()
    assert back["param_groups"] == ref["param_groups"]
    for k, st in ref["state"].items():
        assert float(back["state"][k]["step"]) == float(st["step"])
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(back["state"][k][key], st[key])
    fa.step_count = 7                        # the live count is what a later save writes
    assert all(float(s["step"]) == 7 for s in fa.state_dict()["state"].values())
    other = _module(2)
    fresh = FlatAdam(other, _CpuFlat(other))
    fresh.load_state_dict(torch.optim.Adam(_module(3).parameters()).state_dict())    # a torch Adam never stepped
    assert fresh.step_count == 0 and not fresh.exp_avg.any() and not fresh.exp_avg_sq.any()


def _rejects(sd, match):
    from frustum_convnet_b200.train_engine import FlatAdam
    mine = _module(1)
    fa = FlatAdam(mine, _CpuFlat(mine), lr=5e-4)
    fa.exp_avg.fill_(0.5)
    with pytest.raises(ValueError, match=match):
        fa.load_state_dict(sd)
    assert fa.step_count == 0 and fa.param_groups[0]["lr"] == 5e-4 and bool((fa.exp_avg == 0.5).all())


def test_states_the_fused_step_cannot_continue_are_rejected():
    src = _module()
    sd = _torch_adam_after(2, src).state_dict()
    differ = _roundtrip(sd)
    differ["state"][1]["step"] = torch.tensor(1.0)
    _rejects(differ, "step counts differ")
    for flag in ("amsgrad", "maximize", "decoupled_weight_decay"):
        bad = _roundtrip(sd)
        bad["param_groups"][0][flag] = True
        _rejects(bad, flag)
    two = torch.optim.Adam([{"params": list(src[0].parameters())}, {"params": list(src[2].parameters())}])
    _rejects(two.state_dict(), "2 parameter groups")
    fewer = torch.optim.Adam(list(src[0].parameters())).state_dict()
    _rejects(fewer, "2 parameters, the model has 4")
    other = torch.nn.Sequential(torch.nn.Linear(5, 4), torch.nn.ReLU(), torch.nn.Linear(4, 2))
    _rejects(_torch_adam_after(1, other).state_dict(), "shape")
    sgd = torch.optim.SGD(src.parameters(), lr=0.1, momentum=0.9)
    for p in src.parameters():
        p.grad = torch.ones_like(p)
    sgd.step()
    _rejects(sgd.state_dict(), "no exp_avg")
