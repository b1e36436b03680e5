"""GPU: training with SGD on the fused path - TrainStep(optimizer="sgd") and its optimizer (train_engine.FlatSGD,
one fcn_sgd_step launch over the flat bucket) against torch.optim.SGD, torch checkpoints and torch lr schedulers.

SGD has no sqrt, division or pow: fcn_sgd_step rounds every operation where torch's single-tensor step does
(torch/optim/sgd.py::_single_tensor_sgd, with add(x, y, alpha=) as one FMA), so parameters and momentum buffers are
compared bit for bit."""
import copy
import io
import os
import socket
import sys

import numpy as np
import pytest
import torch

import train_ref as tr
from conftest import ROOT

pytestmark = pytest.mark.gpu


def _data(wl, B, seed):
    from frustum_convnet_b200 import synth
    d = synth.make_frustums(wl, B, seed=seed, with_labels=True, max_depth=(17.5 if wl == "car" else None))
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def _flat_grad(ts, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(ts.flat.numel, generator=g, device="cuda") * torch.rand(ts.flat.numel, generator=g,
                                                                              device="cuda")


def _torch_step(model, grad, opt):
    off = 0                                                    # FlatParams order is model.parameters() order
    for p in model.parameters():
        p.grad = grad[off: off + p.numel()].view(p.shape).clone()
        off += p.numel()
    opt.step()


def _flat_of(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()])


def _buffers_of(model, opt):
    return torch.cat([opt.state[p]["momentum_buffer"].reshape(-1) for p in model.parameters()])


def _save_load(obj):
    f = io.BytesIO()
    torch.save(obj, f)
    f.seek(0)
    return torch.load(f)


def _ulps(a, b):
    """Largest distance in float32 units in the last place between two finite tensors of one sign pattern."""
    ia, ib = a.view(torch.int32).long(), b.view(torch.int32).long()
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int((ia - ib).abs().max())


@pytest.mark.parametrize("wl", ["refine_car", "sunrgbd"])
@pytest.mark.parametrize("momentum", [0.0, 0.9])
@pytest.mark.parametrize("wd", [0.0, 1e-4])
def test_fused_sgd_matches_torch_sgd_bit_for_bit(wl, momentum, wd):
    from frustum_convnet_b200.train_engine import TrainStep
    mine = tr.make_model(wl, 5)
    ts = TrainStep(mine, optimizer="sgd", lr=0.02, momentum=momentum, weight_decay=wd)
    single, foreach = tr.make_model(wl, 5), tr.make_model(wl, 5)
    o_single = torch.optim.SGD(single.parameters(), lr=0.02, momentum=momentum, weight_decay=wd, foreach=False)
    o_foreach = torch.optim.SGD(foreach.parameters(), lr=0.02, momentum=momentum, weight_decay=wd)
    assert torch.equal(ts.flat.param, _flat_of(single))
    for i in range(3):                                         # the first step creates the buffers
        grad = _flat_grad(ts, 100 + i)
        ts.flat.grad.copy_(grad)
        ts.optimizer.step()
        _torch_step(single, grad, o_single)
        _torch_step(foreach, grad, o_foreach)
        torch.cuda.synchronize()
        got, want = ts.flat.param, _flat_of(single)
        assert torch.equal(got, want), (i, int((got != want).sum()), _ulps(got, want))
        assert torch.equal(_flat_of(foreach), want), (i, "foreach", _ulps(_flat_of(foreach), want))
        if momentum:
            assert ts.optimizer.has_buffers
            assert torch.equal(ts.optimizer.momentum_buffer, _buffers_of(single, o_single)), i
            assert torch.equal(_buffers_of(foreach, o_foreach), _buffers_of(single, o_single)), i
        else:
            assert not ts.optimizer.has_buffers and ts.optimizer.state_dict()["state"] == {}
            assert not ts.optimizer.momentum_buffer.any()
    assert ts.step_count == 3


@pytest.mark.parametrize("direction", ["torch_to_trainstep", "trainstep_to_torch"])
def test_optimizer_state_interoperates_with_torch_sgd(direction):
    from frustum_convnet_b200.train_engine import TrainStep
    mine = tr.make_model("refine_car", 6)
    ts = TrainStep(mine, optimizer="sgd", lr=0.01, momentum=0.5)
    ref = tr.make_model("refine_car", 6)
    topt = torch.optim.SGD(ref.parameters(), lr=0.03, momentum=0.9, weight_decay=1e-4, foreach=False)
    if direction == "torch_to_trainstep":
        for i in range(2):
            _torch_step(ref, _flat_grad(ts, i), topt)
        ts.optimizer.load_state_dict(_save_load(topt.state_dict()))
        mine.load_state_dict(ref.state_dict())
        g = ts.optimizer.param_groups[0]
        assert (g["lr"], g["momentum"], g["weight_decay"]) == (0.03, 0.9, 1e-4)
    else:
        for k, v in (("lr", 0.03), ("momentum", 0.9), ("weight_decay", 1e-4)):
            ts.optimizer.param_groups[0][k] = v
        for i in range(2):
            ts.flat.grad.copy_(_flat_grad(ts, i))
            ts.optimizer.step()
        topt.load_state_dict(_save_load(ts.optimizer.state_dict()))
        ref.load_state_dict(mine.state_dict())
    assert ts.optimizer.has_buffers and len(topt.state) == len(list(ref.parameters()))
    assert torch.equal(ts.optimizer.momentum_buffer, _buffers_of(ref, topt))
    grad = _flat_grad(ts, 7)
    ts.flat.grad.copy_(grad)
    ts.optimizer.step()
    _torch_step(ref, grad, topt)
    torch.cuda.synchronize()
    assert torch.equal(ts.flat.param, _flat_of(ref))
    assert torch.equal(ts.optimizer.momentum_buffer, _buffers_of(ref, topt))


def test_resume_from_a_checkpoint_is_exact():
    """The reference loop (INTEGRATION.md section 3) with TRAIN.OPTIMIZER sgd: TrainStep from the config, steps,
    a checkpoint of the reference's keys, and a new TrainStep that resumes from it.  The gradient kernels accumulate
    with float atomics, so the continuation is fed the gradient of the uninterrupted run; everything the checkpoint
    carries (weights, momentum buffers, hyper-parameters) must reproduce its update bit for bit."""
    from frustum_convnet_b200 import config
    from frustum_convnet_b200.train_engine import TrainStep
    TRAIN = copy.deepcopy(config.load_workload("refine_car")[0].TRAIN)      # the yaml's section, then OPTIMIZER: sgd
    TRAIN.OPTIMIZER, TRAIN.BASE_LR = "sgd", 2e-3

    def build(model):
        return TrainStep(model, optimizer=TRAIN.OPTIMIZER, lr=TRAIN.BASE_LR, momentum=TRAIN.MOMENTUM,
                         weight_decay=TRAIN.WEIGHT_DECAY)

    m = tr.make_model("refine_car", 11)
    ts = build(m)
    batches = [_data("refine_car", 4, 900 + i) for i in range(4)]
    ts.states.reset()
    for d in batches[:3]:
        ts.step(d)
    assert len(ts.states.finalize()) == 14
    ckpt = _save_load({"epoch": 1, "state_dict": m.state_dict(), "optimizer": ts.optimizer.state_dict()})
    assert len(ckpt["optimizer"]["state"]) == len(list(m.parameters()))
    ts.forward_backward(batches[3])
    grad = ts.flat.grad.clone()
    ts.optimizer.step()
    m2 = tr.make_model("refine_car", 12)                      # other weights until the checkpoint is loaded
    ts2 = TrainStep(m2, optimizer="sgd", lr=0.5)               # other hyper-parameters too
    m2.load_state_dict(ckpt["state_dict"])
    ts2.optimizer.load_state_dict(ckpt["optimizer"])
    g = ts2.optimizer.param_groups[0]
    assert (ts2.lr, g["momentum"], ts2.wd) == (2e-3, TRAIN.MOMENTUM, TRAIN.WEIGHT_DECAY)
    ts2.flat.grad.copy_(grad)
    ts2.optimizer.step()
    torch.cuda.synchronize()
    assert torch.equal(ts2.flat.param, ts.flat.param)
    assert torch.equal(ts2.optimizer.momentum_buffer, ts.optimizer.momentum_buffer)
    lo, _ = ts2.step(batches[0])                               # and the resumed TrainStep trains on
    assert torch.isfinite(lo["total_loss"])
    with pytest.raises(AttributeError, match="Adam only"):
        ts2.m


def test_lr_schedules_and_the_min_lr_clamp_drive_the_fused_step():
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200.train_engine import TrainStep
    m = tr.make_model("car", 13)
    ts = TrainStep(m, optimizer="sgd", lr=1e-2, momentum=0.9, weight_decay=1e-4)
    opt = ts.optimizer
    step_lr = torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.5)
    MIN_LR = 3e-3
    seen = []

    def fused_step_equals_kernel_at(lr, seed):
        ts.flat.grad.copy_(_flat_grad(ts, seed))
        p, buf = ts.flat.param.clone(), opt.momentum_buffer.clone()
        _lib.call("fcn_sgd_step", p.data_ptr(), ts.flat.grad.data_ptr(), buf.data_ptr(), ts.flat.numel, lr, 0.9,
                  1e-4, int(not opt.has_buffers), 1.0, torch.cuda.current_stream().cuda_stream)
        opt.step()
        torch.cuda.synchronize()
        assert torch.equal(ts.flat.param, p) and torch.equal(opt.momentum_buffer, buf), lr

    for epoch in range(6):                                     # train_net_det.py:98-103 around each epoch
        if step_lr.get_last_lr()[0] < MIN_LR:
            for g in opt.param_groups:
                g["lr"] = MIN_LR
        seen.append(ts.lr)
        fused_step_equals_kernel_at(opt.param_groups[0]["lr"], epoch)
        step_lr.step()
    assert seen == [1e-2, 1e-2, 5e-3, 5e-3, MIN_LR, MIN_LR]
    base = opt.param_groups[0]["lr"]
    multi = torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[1, 3], gamma=0.1)
    for epoch in range(4):
        fused_step_equals_kernel_at(opt.param_groups[0]["lr"], 10 + epoch)
        seen.append(opt.param_groups[0]["lr"])
        multi.step()
    assert base == MIN_LR * 0.5 and np.allclose(seen[6:], [base, base * 0.1, base * 0.1, base * 0.01], rtol=1e-12)


@pytest.mark.parametrize("wl,B", [("car", 2), ("sunrgbd", 2), ("refine_car", 4)])
def test_sgd_train_steps_give_finite_losses_and_append_states(wl, B):
    from frustum_convnet_b200.train_engine import TrainStep
    m = tr.make_model(wl, 14)
    ts = TrainStep(m, optimizer="sgd", lr=1e-3, momentum=0.9, weight_decay=1e-4)
    p0 = ts.flat.param.clone()
    for i in range(3):
        losses, metrics = ts.step(_data(wl, B, 40 + i))
        assert all(bool(torch.isfinite(v)) for v in losses.values()), (i, losses)
    torch.cuda.synchronize()
    assert ts.states.per_step().shape == (3, 14) and ts.step_count == 3
    assert bool(torch.isfinite(ts.flat.param).all()) and not torch.equal(ts.flat.param, p0)
    assert ts.optimizer.has_buffers and bool(ts.optimizer.momentum_buffer.any())
    assert len(ts.states.finalize()) == 14
    with pytest.raises(ValueError, match="not supported"):
        TrainStep(tr.make_model(wl, 14), optimizer="Adam")  # cfg.TRAIN.OPTIMIZER values are lower case


def test_sgd_steps_run_without_a_host_sync():
    from frustum_convnet_b200.train_engine import TrainStep
    m = tr.make_model("refine_car", 15)
    ts = TrainStep(m, optimizer="sgd", lr=1e-3, momentum=0.9, weight_decay=1e-4)
    batches = [_data("refine_car", 4, 700 + i) for i in range(4)]
    for d in batches:                                          # warm-up: engines, graphs and loss objects
        ts.step(d)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for i in range(20):
            ts.step(batches[i % 4])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert ts.states.per_step().shape == (24, 14)
    assert ts.step_count == 24


# ----------------------------------------------------------------------------------------------- two ranks
def _two_rank_steps(rank):
    """Two TrainStep(optimizer="sgd") steps on this rank's batches -> per step (parameters before the step, this rank's
    gradient as the step hands it to the all-reduce, the reduced bucket, parameters and buffer after the step)."""
    import torch.distributed as dist
    from frustum_convnet_b200.train_engine import TrainStep
    m = tr.make_model("refine_car", 16)
    ts = TrainStep(m, optimizer="sgd", lr=1e-2, momentum=0.9, weight_decay=1e-4)
    pieces, all_reduce = [], dist.all_reduce

    def recording_all_reduce(t, *args, **kw):       # runs on the step's comm stream, ahead of the reduction
        pieces.append((t.data_ptr(), t.clone()))
        return all_reduce(t, *args, **kw)

    dist.all_reduce = recording_all_reduce
    try:
        out = []
        for i in range(2):
            d = _data("refine_car", 4 + rank, 1100 + 10 * i + rank)
            p0 = ts.flat.param.clone()
            pieces.clear()
            ts.step(d)
            torch.cuda.synchronize()
            local = torch.full_like(ts.flat.grad, float("nan"))
            for ptr, t in pieces:                        # the bucket's two pieces
                off = (ptr - ts.flat.grad.data_ptr()) // 4
                local[off: off + t.numel()] = t
            out.append(tuple(t.cpu().numpy() for t in (p0, local, ts.flat.grad, ts.flat.param,
                                                       ts.optimizer.momentum_buffer)))
        return out
    finally:
        dist.all_reduce = all_reduce


def _worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        ret[rank] = _two_rank_steps(rank)
    finally:
        dist.destroy_process_group()


def _check_two_rank_steps(r0, r1):
    ref = tr.make_model("refine_car", 16)
    topt = torch.optim.SGD(ref.parameters(), lr=1e-2, momentum=0.9, weight_decay=1e-4, foreach=False)
    for a, b in zip(r0, r1):
        (p0, l0, s0, q0, b0), (p1, l1, s1, q1, b1) = [[torch.from_numpy(x) for x in r] for r in (a, b)]
        assert torch.equal(p0, p1) and torch.equal(p0, _flat_of(ref).cpu())
        assert not l0.isnan().any() and not l1.isnan().any()      # the two pieces cover the bucket
        assert torch.equal(s0, s1)                             # the all-reduced sum is the same on both ranks
        # a sum of two float32 values is rounded once, in whichever order the collective adds them (up to a
        # collective that flushes subnormal results to zero)
        assert bool(((s0 - (l0 + l1)).abs() <= 2.0 ** -126).all())
        _torch_step(ref, s0.cuda() * float(np.float32(1.0 / 2)), topt)      # grad_scale = float32(1 / world)
        torch.cuda.synchronize()
        assert torch.equal(q0, q1) and torch.equal(q0, _flat_of(ref).cpu())
        assert torch.equal(b0, b1) and torch.equal(b0, _buffers_of(ref, topt).cpu())


def test_two_ranks_step_on_the_scaled_sum_of_the_ranks_gradients():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=True)
    _check_two_rank_steps(ret[0], ret[1])
