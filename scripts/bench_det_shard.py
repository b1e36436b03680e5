#!/usr/bin/env python
"""Finalizing a sharded detection pass: ``DetectionCollector(.., group=pg).finalize_device()`` on every rank against
one collector's ``finalize_device()`` over the union of the ranks' adds, on the KITTI-size set of
scripts/bench_det_eval.py (oracle/kitti_synth.py, seed 0, 3 769 images, method 'top').

    python scripts/bench_det_shard.py [--world 2] [--images 3769] [--batch 32] [--calls 20] [--warmup 3]
    torchrun --nproc-per-node N scripts/bench_det_shard.py [...]

Without torchrun, --world processes share GPU 0 over gloo; under torchrun every rank takes its own GPU over NCCL.
Every rank adds its shard_slice chunk of every batch of --batch frustums.  Per call: host wall time of
finalize_device() between two device synchronizes, the merged call on every rank at once (after a barrier), then the
single collector over the union on rank 0.  Medians over --calls calls after --warmup.  Also reports the bytes every
rank receives in the two all_gathers (the counters and added flags, then max(counts) 48-byte records per rank), and
whether the merged and single results are bit-identical.  Rank 0 prints one JSON line with the card name and its
power limit.  Writes nothing to the tree."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _wall(fn, sync):
    sync()
    t0 = time.perf_counter()
    res = fn()
    sync()
    return (time.perf_counter() - t0) * 1e3, res


def run(rank, world, backend, dev, args):
    import torch
    import torch.distributed as dist
    from bench_detect import gpu_identity
    from det_feed_sets import collector_for, kitti_set
    from det_shard_sets import add_shard, rebatch, recorded_pass
    from frustum_convnet_b200.detect import DetectionCollector
    sync = lambda: torch.cuda.synchronize(dev)
    _, dets = kitti_set(args.images, seed=0)
    (ctor, adds), _ = recorded_pass(lambda: collector_for(dets, "KITTI", device=dev))
    adds = rebatch(adds, args.batch)
    pos, kw = ctor
    kw = dict(kw, device=dev)
    col = DetectionCollector(*pos, group=dist.group.WORLD, **kw)
    add_shard(col, adds, rank, world)
    one = None
    if rank == 0:
        one = DetectionCollector(*pos, **kw)
        for r in range(world):
            add_shard(one, adds, r, world)
    sync()
    counts = [None] * world
    dist.all_gather_object(counts, int(col.counter.item()))
    merged_ms, single_ms = [], []
    for it in range(args.warmup + args.calls):
        dist.barrier()
        t, merged = _wall(col.finalize_device, sync)
        dist.barrier()
        if rank == 0:
            ts, single = _wall(one.finalize_device, sync)
            if it >= args.warmup:
                merged_ms.append(t)
                single_ms.append(ts)
    if rank != 0:
        return
    a, b = merged.to_dict(), single.to_dict()
    same = list(a) == list(b) and all(list(a[i]) == list(b[i]) and
                                      all(a[i][c].tobytes() == b[i][c].tobytes() for c in b[i]) for i in b)
    n = col.num_frustums
    out = {"bench": "det_shard", "backend": backend, "world": world, "images": args.images, "frustums": n,
           "batch": args.batch, "calls": args.calls, "rows_per_rank": counts, "rows": int(sum(counts)),
           "kept": merged.host_keep_count.sum().item(),
           "gathered_bytes_per_rank": {"flags": world * (8 + n), "records": world * max(counts) * 48},
           "merged_finalize_ms": float(np.median(merged_ms)), "single_finalize_ms": float(np.median(single_ms)),
           "identical": bool(same)}
    out.update(gpu_identity(dev))
    print(json.dumps(out), flush=True)


def _spawned(rank, world, port, args):
    import torch
    import torch.distributed as dist
    from spawn_group import init_group
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    init_group(rank, world, port, "gloo")
    try:
        run(rank, world, "gloo", dev, args)
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=2, help="gloo processes on GPU 0 (ignored under torchrun)")
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_det_shard.py needs a CUDA device; there is no CPU fallback"
    if "WORLD_SIZE" in os.environ:                                   # torchrun: one GPU per rank, NCCL
        import torch.distributed as dist
        rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
        dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
        torch.cuda.set_device(dev)
        dist.init_process_group("nccl", device_id=dev)
        try:
            run(rank, world, "nccl", dev, args)
        finally:
            dist.destroy_process_group()
    else:
        from spawn_group import run_group
        run_group(_spawned, args.world, (args,), timeout=1800)


if __name__ == "__main__":
    main()
