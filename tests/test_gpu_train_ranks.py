"""GPU: seeded multi-rank training in deterministic mode.  Every rank of a group runs ``TrainStep(deterministic=True)``
on its own shard of every step; afterwards every rank must hold the same parameters, optimizer state and BN buffers,
and those bits must equal a one-process replay: each shard's ``forward_backward`` (the whole backward at once, where
the step runs it in two stages), the float32 sum of the shards' gradients in rank order, grad_scale = 1/G, the
optimizer step, and the BN buffers of shard 0.  ``TrainStates.finalize`` and ``Validator(group=).finalize`` must
return the same bits on every rank, the float64 replay of the rank-ordered sum of the ranks' rows.

gloo groups of 2 and 3 processes share one GPU (three ranks are needed to see an order: at two, the one add
commutes); the NCCL group needs one GPU per rank and is skipped on fewer than 2."""
import os
import pickle
import traceback

import numpy as np
import pytest
import torch

import train_ref as tr
from rank_fold_ref import left_fold
from test_gpu_train_states import _replay, _same

pytestmark = pytest.mark.gpu

CASES = [("refine_car", 4), ("car", 2)]
OPTIMIZERS = ("adam", "sgd")
STEPS = 3
VAL_BATCHES = (9, 7, 12)                 # frustums per validation batch, split over the ranks by shard_slice


def _shard(wl, B, step, rank):
    from frustum_convnet_b200 import synth
    d = synth.make_frustums(wl, B, seed=7000 + 100 * step + rank, with_labels=True,
                            max_depth=(17.5 if wl == "car" else None))
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def _val_batches(wl):
    from frustum_convnet_b200 import synth
    out = []
    for i, B in enumerate(VAL_BATCHES):
        d = synth.make_frustums(wl, B, seed=9100 + i, with_labels=True, max_depth=(17.5 if wl == "car" else None))
        out.append({k: torch.from_numpy(v).cuda() for k, v in d.items()})
    return out


def _chunk(data, rank, world):
    from frustum_convnet_b200.sharding import shard_slice
    sl = shard_slice(int(data["point_cloud"].shape[0]), rank, world)
    return {k: v[sl].contiguous() for k, v in data.items()}


def _snapshot(ts, model):
    torch.cuda.synchronize()
    opt = ts.optimizer
    state = [opt.exp_avg, opt.exp_avg_sq] if isinstance(opt, torch.optim.Adam) else [opt.momentum_buffer]
    return dict(param=ts.flat.param.cpu().numpy().copy(), state=[t.cpu().numpy().copy() for t in state],
                buffers={n: b.cpu().numpy().copy() for n, b in model.named_buffers()})


def _message(fn):
    try:
        fn()
    except (ValueError, RuntimeError) as e:
        return "%s: %s" % (type(e).__name__, e)
    return "no error"


# ------------------------------------------------------------------------------------------------ one rank
def _rank_cases(pg, rank, world):
    from frustum_convnet_b200.train_engine import TrainStep
    from frustum_convnet_b200.validate import Validator
    got = {}
    for wl, B in CASES:
        for opt in OPTIMIZERS:
            model = tr.make_model(wl, seed=21)
            ts = TrainStep(model, lr=1e-3, optimizer=opt, momentum=0.9, weight_decay=1e-4, deterministic=True)
            for i in range(STEPS):
                ts.step(_shard(wl, B, i, rank))
            snap = _snapshot(ts, model)
            snap["rows"] = ts.states.per_step(full=True)
            snap["final"] = list(ts.states.finalize().values())
            got["train", wl, opt] = snap
        model = tr.make_model(wl, seed=21).eval()
        batches = _val_batches(wl)
        val, own = Validator(model, group=pg), Validator(model)
        for d in batches:
            val.add(_chunk(d, rank, world))
            own.add(_chunk(d, rank, world))
        got["val", wl] = dict(rows=val.per_batch(full=True), final=list(val.finalize().values()),
                              own_rows=own.per_batch(full=True), own=list(own.finalize().values()))
        val.reset()
        for d in batches[: (len(batches) - 1 if rank == world - 1 else len(batches))]:
            val.add(_chunk(d, rank, world))
        got["uneven", wl] = _message(val.finalize)
        val.reset()                                    # the group is still usable after the error
        for d in batches:
            val.add(_chunk(d, rank, world))
        got["after_error", wl] = list(val.finalize().values())
    return got


def _worker(rank, world, port, backend, out_path):
    import torch.distributed as dist
    from spawn_group import init_group
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    init_group(rank, world, port, backend, **({"device_id": dev} if backend == "nccl" else {}))
    got = {}
    try:
        got = _rank_cases(dist.group.WORLD, rank, world)
    except Exception:
        got = {"FAILED": traceback.format_exc()}
    finally:
        with open(out_path % rank, "wb") as f:
            pickle.dump(got, f)
        dist.destroy_process_group()


def _launch(backend, world, tmp_path, tag):
    from spawn_group import run_group
    path = os.path.join(str(tmp_path), tag + "_rank%d.pkl")
    run_group(_worker, world, (backend, path), timeout=1200)
    got = [pickle.load(open(path % r, "rb")) for r in range(world)]
    failed = [g["FAILED"] for g in got if "FAILED" in g]
    assert not failed, "\n".join(failed)
    return got


# ------------------------------------------------------------------------------------------------ replays
def _replay_training(wl, B, opt, world):
    """One process, no process group: the shards of every step through forward_backward, their gradients summed
    in rank order in float32, grad_scale = 1/world, the optimizer step; BN buffers from shard 0 only."""
    from frustum_convnet_b200.train_engine import TrainStep
    model = tr.make_model(wl, seed=21)
    ts = TrainStep(model, lr=1e-3, optimizer=opt, momentum=0.9, weight_decay=1e-4, deterministic=True)
    for i in range(STEPS):
        grads = []
        for r in range(world):
            ts.forward_backward(_shard(wl, B, i, r), update_running=(r == 0))
            grads.append(ts.flat.grad.cpu().numpy().copy())
        ts.flat.grad.copy_(torch.from_numpy(left_fold(np.stack(grads))))
        ts.optimizer.grad_scale = 1.0 / world
        ts.optimizer.step()
    return _snapshot(ts, model)


def _mean_rows(tables, world):
    """The ranks' (n, 18) rows summed in rank order, the 14 values divided by world as the meter table does it
    (the same torch division on the device)."""
    t = torch.from_numpy(left_fold(np.stack(tables))).cuda()
    t[:, :14] /= world
    return t.cpu().numpy()


def _bits_equal(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _check_snapshot(a, b, what):
    assert _bits_equal(a["param"], b["param"]), what + ": parameters"
    assert all(_bits_equal(x, y) for x, y in zip(a["state"], b["state"])), what + ": optimizer state"
    assert a["buffers"].keys() == b["buffers"].keys()
    for n in a["buffers"]:
        assert _bits_equal(a["buffers"][n], b["buffers"][n]), what + ": buffer " + n


def _check(got, world):
    for wl, B in CASES:
        for opt in OPTIMIZERS:
            what = "%s %s world=%d" % (wl, opt, world)
            runs = [g["train", wl, opt] for g in got]
            for r in range(1, world):                                          # (a)
                _check_snapshot(runs[r], runs[0], what + " rank %d vs rank 0" % r)
            _check_snapshot(runs[0], _replay_training(wl, B, opt, world), what + " vs the replay")   # (b)
            want = _replay(_mean_rows([g["rows"] for g in runs], world))      # (d)
            assert all(_same(g["final"], want) for g in runs), (what, [g["final"] for g in runs], want)
        vals = [g["val", wl] for g in got]                                      # (e)
        want = _replay(_mean_rows([v["rows"] for v in vals], world))
        assert all(_same(v["final"], want) for v in vals), (wl, [v["final"] for v in vals], want)
        assert sum(len(v["rows"]) for v in vals) == world * len(VAL_BATCHES)
        for v in vals:                                                          # (g)
            assert _same(v["own"], _replay(v["own_rows"]))
        msgs = [g["uneven", wl] for g in got]                                   # (f)
        assert all(m == msgs[0] for m in msgs), msgs
        assert msgs[0].startswith("ValueError: Validator: the ranks of the group added different numbers of batches")
        assert all(_same(g["after_error", wl], want) for g in got)


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_ranks_on_one_gpu_hold_one_model(world, tmp_path):
    got = _launch("gloo", world, tmp_path, "first")
    _check(got, world)
    if world == 3:                                                              # (c)
        again = _launch("gloo", world, tmp_path, "second")
        for wl, _ in CASES:
            for opt in OPTIMIZERS:
                for r in range(world):
                    _check_snapshot(again[r]["train", wl, opt], got[r]["train", wl, opt],
                                    "%s %s second launch, rank %d" % (wl, opt, r))


def test_nccl_one_gpu_per_rank(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = min(torch.cuda.device_count(), 3)
    _check(_launch("nccl", world, tmp_path, "nccl"), world)
