#!/usr/bin/env python
"""What the rank-ordered gradient sum of deterministic multi-GPU training costs.

    python scripts/bench_train_ranks.py [--iters 200] [--regions 7]
    torchrun --nproc_per_node=<GPUs> scripts/bench_train_ranks.py [--batch 32] [--steps 30] [--regions 5]

One process (no torchrun): device time of fcn_rank_fold over the KITTI (3 316 777 floats) and SUN-RGBD (6 667 589)
gradient buckets cut by shard_plan at G = 2, 4 and 8, i.e. one rank's fold of its shard over G rows of shard
floats.  CUDA events around `--iters` launches, median over `--regions` regions, with the bytes the fold reads
(G * shard floats) and writes (shard floats) and the rate they imply.

Under torchrun with world >= 2 (NCCL, one GPU per rank): ms per TrainStep.step, deterministic=False (one NCCL
all-reduce per piece, each rank its own BN buffers) against deterministic=True (all-to-all, fold, all-gather per
piece and rank 0's BN buffers broadcast), refine_car at B = --batch per rank on resident synthetic batches, Adam,
alternated regions of `--steps` steps, host clock around a region that ends in a device synchronise.

Prints one JSON line (rank 0) with the card name and power limit.  Writes nothing to the tree."""
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

from bench_detect import gpu_identity  # noqa: E402

BUCKETS = {"kitti": 3316777, "sunrgbd": 6667589}


def bench_fold(dev, iters, regions):
    import torch
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200.train_engine import shard_plan
    out = {}
    for name, n in BUCKETS.items():
        for G in (2, 4, 8):
            shard, padded = shard_plan(n, G)
            src = torch.randn(padded, device=dev)
            dst = torch.empty(shard, device=dev)
            st = torch.cuda.current_stream(dev).cuda_stream

            def launch():
                _lib.call("fcn_rank_fold", src.data_ptr(), shard, G, shard, dst.data_ptr(), st)

            for _ in range(20):
                launch()
            times = []
            for _ in range(regions):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(iters):
                    launch()
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b) * 1e3 / iters)
            us = float(np.median(times))
            read, written = 4 * G * shard, 4 * shard
            out["%s_G%d" % (name, G)] = {"shard_floats": shard, "us": us, "min_us": float(min(times)),
                                         "max_us": float(max(times)), "bytes_read": read, "bytes_written": written,
                                         "GB_per_s": (read + written) / (us * 1e-6) / 1e9}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--regions", type=int, default=7)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "bench_train_ranks.py needs a CUDA device; there is no CPU fallback"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world == 1:
        dev = torch.device("cuda", 0)
        torch.cuda.set_device(dev)
        line = {"fold": bench_fold(dev, args.iters, args.regions), "multi_gpu_step": "not measured (one process)"}
        line.update(gpu_identity(dev))
        print(json.dumps(line))
        return

    import torch.distributed as dist
    from bench_train_deterministic import _model
    from frustum_convnet_b200 import synth
    from frustum_convnet_b200.train_engine import TrainStep
    rank = int(os.environ["RANK"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    try:
        B, K = args.batch, args.steps
        batches = []
        for s in range(4):
            d = synth.make_frustums("refine_car", B, seed=40 + 10 * s + rank, with_labels=True)
            batches.append({k: torch.from_numpy(v).to(dev) for k, v in d.items()})
        steps = {}
        for det in (False, True):
            m, cfg = _model("refine_car", dev)
            steps[det] = TrainStep(m, lr=cfg.TRAIN.BASE_LR, weight_decay=cfg.TRAIN.WEIGHT_DECAY, deterministic=det)

        def region(ts):
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            for i in range(K):
                ts.step(batches[i % len(batches)])
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3 / K

        for ts in steps.values():
            for i in range(8):
                ts.step(batches[i % len(batches)])
        times = {False: [], True: []}
        for _ in range(args.regions):
            for det in (False, True):
                times[det].append(region(steps[det]))
        if rank == 0:
            res = {("deterministic" if det else "default"): {"ms_per_step": float(np.median(t)),
                                                              "min": float(min(t)), "max": float(max(t))}
                   for det, t in times.items()}
            res["overhead_pct"] = 100.0 * (res["deterministic"]["ms_per_step"] / res["default"]["ms_per_step"] - 1.0)
            line = {"workload": "refine_car", "batch_per_rank": B, "world": world, "steps_per_region": K,
                    "regions": args.regions, "step": res}
            line.update(gpu_identity(dev))
            print(json.dumps(line))
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
