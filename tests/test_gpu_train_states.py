"""GPU: training without a host sync per step - TrainStep.states (validate.TrainStates over fcn_train_states_append
and fcn_val_finalize) against the fused loss's own result blocks and a float64 AverageMeter replay, and
TrainStep.optimizer (train_engine.FlatAdam) against torch.optim.Adam, torch checkpoints and torch lr schedulers.

Adam bar for the torch interop: each side is within the bound of tests/test_gpu_train_layers.py section (f) of the
float64 restatement (4 ulp of the result + 1e-6 * lr + 2^-18 * sc + the powf error of the bias corrections), so the
two agree within twice that bound."""
import io
import math
import os
import socket
import sys

import numpy as np
import pytest
import torch

import train_ref as tr
from conftest import ROOT

pytestmark = pytest.mark.gpu

CASES = [("refine_car", 4), ("car", 2)]


def _model(wl, seed=11):
    from frustum_convnet_b200 import config, synth
    from frustum_convnet_b200.det_base import PointNetDet
    cfg, w = config.load_workload(wl)
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=seed)
    m = PointNetDet(3, num_vec=w["num_vec"])
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m.cuda().train(), cfg


def _data(wl, B, seed):
    from frustum_convnet_b200 import synth
    d = synth.make_frustums(wl, B, seed=seed, with_labels=True, max_depth=(17.5 if wl == "car" else None))
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def _replay(rows):
    """utils/utils.py AverageMeter over (values, n) rows in float64, in row order -> the 14 averages."""
    out = []
    for k in range(14):
        s, c = 0.0, 1e-14
        for r in rows:
            s = s + float(r[k]) * float(r[14])
            c = c + float(r[14])
        out.append(s / c)
    return np.array(out)


def _same(a, b):
    return np.array_equal(np.asarray(a, np.float64), np.asarray(b, np.float64), equal_nan=True)


@pytest.mark.parametrize("wl,B", CASES)
def test_every_step_appends_its_cached_fused_loss_block_and_finalize_replays_average_meter(wl, B):
    from frustum_convnet_b200.train_engine import TrainStep
    m, cfg = _model(wl)
    ts = TrainStep(m, lr=1e-3, weight_decay=1e-4)
    sizes = [B, B, B + 1, B, B, B, B]                           # one step with a different batch size
    want = []
    for i, b in enumerate(sizes):
        d = _data(wl, b, 500 + i)
        ts.step(d)
        torch.cuda.synchronize()
        want.append(ts._fused_losses[(False, b, d["center_ref2"].shape[2])].out.cpu().numpy())
    rows = ts.states.per_step(full=True)
    assert rows.shape == (7, 18)
    for i, (r, o, b) in enumerate(zip(rows, want, sizes)):
        assert _same(r[:14], o[:14]), (i, r[:14], o[:14])
        assert (r[14], r[15], r[16], r[17]) == (b, o[14], o[15], 0.0), (i, r[14:])
    assert _same(ts.states.per_step(), rows[:, :14])
    last = ts.states.last()
    assert list(last) == list(ts.states.keys) and _same(list(last.values()), rows[-1, :14])
    states = ts.states.finalize()
    assert list(states) == ["total_loss", "cls_loss", "center_loss", "head_cls_loss", "head_res_loss",
                            "size_cls_loss", "size_res_loss", "corners_loss", "cls_acc", "head_acc", "size_acc",
                            "IoU_2D", "IoU_3D", "IoU_" + str(cfg.IOU_THRESH)]
    assert _same(list(states.values()), _replay(rows))
    ts.states.reset()                                          # a new epoch starts from row 0
    ts.step(_data(wl, B, 600))
    assert ts.states.per_step().shape == (1, 14)


def test_steps_run_without_a_host_sync():
    from frustum_convnet_b200.train_engine import TrainStep
    m, _ = _model("refine_car")
    ts = TrainStep(m, lr=1e-3, weight_decay=1e-4)
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


def test_overflow_and_a_step_without_foreground_are_reported():
    from frustum_convnet_b200.train_engine import TrainStep
    m, _ = _model("car")
    ts = TrainStep(m, states_capacity=2)
    for i in range(3):
        ts.step(_data("car", 2, 800 + i))
    with pytest.raises(RuntimeError, match="3 steps were added but the capacity is 2.*states_capacity=3"):
        ts.states.finalize()
    with pytest.raises(RuntimeError, match="capacity"):
        ts.states.last()
    ts = TrainStep(m)
    for i in range(4):
        d = _data("car", 2, 810 + i)
        if i in (1, 3):
            d["cls_label"].clamp_(max=0)                       # no row labelled 1
        ts.step(d)
    with pytest.raises(RuntimeError, match="step 1 of the epoch has no foreground row"):
        ts.states.finalize()
    ts.states.reset()
    ts.step(_data("car", 2, 820))
    assert len(ts.states.finalize()) == 14


def test_captured_appends_replay_like_eager_appends():
    from frustum_convnet_b200.validate import TrainStates
    g = torch.Generator(device="cuda").manual_seed(5)
    blocks = []
    for i in range(5):
        b = torch.rand(16, generator=g, device="cuda")
        b[14], b[15] = float(3 + i), float(40 + i)
        blocks.append(b)
    sizes = [4, 4, 5, 4, 3]
    eager = TrainStates("cuda", capacity=16)
    for _ in range(2):
        for b, n in zip(blocks, sizes):
            eager.append(b, n)
    graphed = TrainStates("cuda", capacity=16)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for b, n in zip(blocks, sizes):
                graphed.append(b, n)
    torch.cuda.current_stream().wait_stream(side)
    graphed.reset()
    graph.replay()
    graph.replay()
    a, b = eager.per_step(full=True), graphed.per_step(full=True)
    assert a.shape == (10, 18) and np.array_equal(a, b)
    assert _same(list(eager.finalize().values()), list(graphed.finalize().values()))


def _save_load(obj):
    f = io.BytesIO()
    torch.save(obj, f)
    f.seek(0)
    return torch.load(f)


def test_resume_from_a_checkpoint_is_exact():
    """The gradient kernels accumulate with float atomics, so two runs of the same step may differ in the last bits
    of the gradient; the continuation is therefore fed the gradient of the uninterrupted run, and everything the
    checkpoint carries (weights, moments, step count, hyper-parameters) must reproduce its update bit for bit."""
    from frustum_convnet_b200.train_engine import TrainStep
    m, _ = _model("refine_car")
    ts = TrainStep(m, lr=2e-3, weight_decay=1e-4)
    batches = [_data("refine_car", 4, 900 + i) for i in range(4)]
    for d in batches[:3]:
        ts.step(d)
    ckpt = _save_load({"state_dict": m.state_dict(), "optimizer": ts.optimizer.state_dict()})
    ts.forward_backward(batches[3])
    grad = ts.flat.grad.clone()
    ts.optimizer.step()
    m2, _ = _model("refine_car", seed=12)                      # other weights until the checkpoint is loaded
    ts2 = TrainStep(m2)
    m2.load_state_dict(ckpt["state_dict"])
    ts2.optimizer.load_state_dict(ckpt["optimizer"])
    assert ts2.step_count == 3 and ts2.lr == 2e-3 and ts2.wd == 1e-4
    ts2.flat.grad.copy_(grad)
    ts2.optimizer.step()
    torch.cuda.synchronize()
    assert torch.equal(ts2.flat.param, ts.flat.param)
    assert torch.equal(ts2.m, ts.m) and torch.equal(ts2.v, ts.v) and ts2.step_count == 4
    lo, _ = ts2.step(batches[0])                               # and the resumed TrainStep trains on
    assert torch.isfinite(lo["total_loss"])


def _adam_tol(p0, g, m0, v0, group, step):
    b1, b2 = group["betas"]
    ep, _, _, sc = tr.adam_ref(p0.cpu(), g.cpu(), m0.cpu(), v0.cpu(), group["lr"], b1, b2, group["eps"],
                               group["weight_decay"], step, 1.0)
    f1, f2 = tr.f32(b1), tr.f32(b2)
    bc_rel = 2.0 ** -21 * f1 ** step / (1 - f1 ** step) + 2.0 ** -22 * f2 ** step / (1 - f2 ** step)
    ulp = (torch.nextafter(ep.float(), torch.tensor(math.inf)) - ep.float()).abs().double()
    bar = 4 * ulp + 1e-6 * group["lr"] + 2.0 ** -18 * sc + bc_rel * (p0.cpu().double() - ep).abs()
    return 2 * bar


def _flat_grad(ts, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(ts.flat.numel, generator=g, device="cuda") * torch.rand(ts.flat.numel, generator=g,
                                                                              device="cuda")


def _torch_adam_step(model, grad, opt):
    off = 0                                                    # FlatParams order is model.parameters() order
    for p in model.parameters():
        p.grad = grad[off: off + p.numel()].view(p.shape).clone()
        off += p.numel()
    opt.step()


def _flat_of(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()])


@pytest.mark.parametrize("direction", ["torch_to_trainstep", "trainstep_to_torch"])
def test_optimizer_state_interoperates_with_torch_adam(direction):
    from frustum_convnet_b200.train_engine import TrainStep
    mine, _ = _model("refine_car")
    ts = TrainStep(mine)
    ref, _ = _model("refine_car")
    topt = torch.optim.Adam(ref.parameters(), lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-4)
    if direction == "torch_to_trainstep":
        for i in range(2):
            _torch_adam_step(ref, _flat_grad(ts, i), topt)
        ts.optimizer.load_state_dict(_save_load(topt.state_dict()))
        mine.load_state_dict(ref.state_dict())
    else:
        ts.optimizer.param_groups[0]["weight_decay"] = 1e-4
        for i in range(2):
            ts.flat.grad.copy_(_flat_grad(ts, i))
            ts.optimizer.step()
        topt.load_state_dict(_save_load(ts.optimizer.state_dict()))
        ref.load_state_dict(mine.state_dict())
    assert ts.step_count == 2 and all(float(s["step"]) == 2 for s in topt.state.values())
    grad = _flat_grad(ts, 7)
    p0, m0, v0 = ts.flat.param.clone(), ts.m.clone(), ts.v.clone()
    ts.flat.grad.copy_(grad)
    ts.optimizer.step()
    _torch_adam_step(ref, grad, topt)
    torch.cuda.synchronize()
    a, b = ts.flat.param.cpu().double(), _flat_of(ref).cpu().double()
    tol = _adam_tol(p0, grad, m0, v0, topt.param_groups[0], 3)
    bad = (a - b).abs() > tol
    assert not bool(bad.any()), (int(bad.sum()), float((a - b).abs().max()))


def test_lr_schedules_and_the_min_lr_clamp_drive_the_fused_step():
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200.train_engine import TrainStep
    m, _ = _model("car")
    ts = TrainStep(m, lr=1e-3, weight_decay=1e-4)
    opt = ts.optimizer
    step_lr = torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.5)
    MIN_LR = 3e-4
    seen = []

    def fused_step_equals_kernel_at(lr, seed):
        ts.flat.grad.copy_(_flat_grad(ts, seed))
        p, mm, vv = ts.flat.param.clone(), ts.m.clone(), ts.v.clone()
        _lib.call("fcn_adam_step", p.data_ptr(), ts.flat.grad.data_ptr(), mm.data_ptr(), vv.data_ptr(),
                  ts.flat.numel, lr, 0.9, 0.999, 1e-8, 1e-4, ts.step_count + 1, 1.0,
                  torch.cuda.current_stream().cuda_stream)
        opt.step()
        torch.cuda.synchronize()
        assert torch.equal(ts.flat.param, p) and torch.equal(ts.m, mm) and torch.equal(ts.v, vv), lr

    for epoch in range(6):                                     # train_net_det.py:98-103 around each epoch
        if step_lr.get_last_lr()[0] < MIN_LR:
            for g in opt.param_groups:
                g["lr"] = MIN_LR
        seen.append(ts.lr)
        fused_step_equals_kernel_at(opt.param_groups[0]["lr"], epoch)
        step_lr.step()
    assert seen == [1e-3, 1e-3, 5e-4, 5e-4, MIN_LR, MIN_LR]
    base = opt.param_groups[0]["lr"]
    multi = torch.optim.lr_scheduler.MultiStepLR(opt, milestones=[1, 3], gamma=0.1)
    for epoch in range(4):
        fused_step_equals_kernel_at(opt.param_groups[0]["lr"], 10 + epoch)
        seen.append(opt.param_groups[0]["lr"])
        multi.step()
    assert base == MIN_LR * 0.5 and np.allclose(seen[6:], [base, base * 0.1, base * 0.1, base * 0.01], rtol=1e-12)
    ts.lr = 2e-4                                               # the old attribute writes the param group
    assert opt.param_groups[0]["lr"] == 2e-4
    fused_step_equals_kernel_at(2e-4, 20)


# ----------------------------------------------------------------------------------------------- two ranks
def _worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from frustum_convnet_b200.train_engine import TrainStep
        m, _ = _model("refine_car")
        ts = TrainStep(m, lr=1e-3)
        for i in range(3):
            ts.step(_data("refine_car", 4 + rank, 1000 + 10 * i + rank))
        rows = ts.states.per_step(full=True)
        states = ts.states.finalize()
        ret[rank] = (rows, list(states.values()))
    finally:
        dist.destroy_process_group()


def test_two_ranks_finalize_the_mean_over_replicas():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=True)
    (r0, s0), (r1, s1) = ret[0], ret[1]
    mean = (r0[:, :14] + r1[:, :14]) / np.float32(2)            # float32, as the replicas' losses are averaged
    rows = np.concatenate([mean, (r0[:, 14:15] + r1[:, 14:15])], 1)
    want = _replay(rows)
    assert _same(s0, want) and _same(s1, want)
