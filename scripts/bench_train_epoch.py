#!/usr/bin/env python
"""What a host sync per training step costs: the reference train() loop reads its 14 losses and metrics with
`.item()` after every step (train/train_net_det.py:131-132), which stops the host from preparing step n+1 while step
n runs.  TrainStep.states keeps them on the device instead and is read every `cfg.disp` steps.

    python scripts/bench_train_epoch.py [--batch 32] [--steps 100] [--regions 5] [--frustums 4096]

Workloads: refine_car (refinement batches, N=512), car detection (N=1024, max depth 70) and SUN-RGBD (N=2048, max
depth 8), B = --batch, batches from TrainBatchBuilder over a resident synthetic dataset (the datasets of
scripts/bench_train_inputs.py).  Each step draws its random augmentation on the host (draw) and builds its batch on
the device (build) inside the timed loop, because that host work is what a per-step sync serialises.  Two loops over
the same batches, timed in alternating regions of `--steps` steps (host clock around a region that ends in a device
synchronise):
  item_ms_per_step    TrainStep.step, then `.item()` on the 14 values, every step;
  states_ms_per_step  TrainStep.step with TrainStep.states, `last()` every 50 steps (cfg.disp) and `finalize()` at
                      the end of the region (one epoch).
Prints one JSON line with medians, min / max per loop and the card name and power limit.  Writes nothing to the
tree."""
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
from bench_train_inputs import CAR, MAX_DEPTH, REFINE, SUN, synthetic_lists, synthetic_sun_lists  # noqa: E402

DISP = 50
WORKLOADS = (("refine_car", "refine", REFINE, 512), ("car", "det", CAR, 1024), ("sunrgbd", "sunrgbd", SUN, 2048))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--frustums", type=int, default=4096)
    args = ap.parse_args()

    import torch
    from frustum_convnet_b200 import config, synth
    from frustum_convnet_b200.train_engine import TrainStep
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    assert torch.cuda.is_available(), "bench_train_epoch.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, K = args.batch, args.steps
    line = {"batch": B, "steps_per_region": K, "regions": args.regions, "disp": DISP}
    for workload, kind, strides, N in WORKLOADS:
        L = synthetic_sun_lists(args.frustums, seed=3) if kind == "sunrgbd" else synthetic_lists(kind, args.frustums,
                                                                                                 seed=3)
        tb = TrainBatchBuilder(kind, strides, N, max_depth=MAX_DEPTH[kind])
        tb.set_dataset(L["input_list"], L["type_list"], **{k: v for k, v in L.items()
                                                           if k not in ("input_list", "type_list")})
        cfg, w = config.load_workload(workload)
        if kind == "sunrgbd":
            from frustum_convnet_b200.det_base_sunrgbd import PointNetDet
        else:
            from frustum_convnet_b200.det_base import PointNetDet
        sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=7)
        m = PointNetDet(3, num_vec=w["num_vec"])
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
        ts = TrainStep(m.to(dev).train(), lr=cfg.TRAIN.BASE_LR, weight_decay=cfg.TRAIN.WEIGHT_DECAY)
        rng = np.random.RandomState(0)
        order = np.concatenate([rng.permutation(args.frustums) for _ in range(1 + K * B // args.frustums)])
        idx = [order[i * B: (i + 1) * B] for i in range(K)]

        def step(i):
            return ts.step(tb.build(idx[i], tb.draw(idx[i], rng)))

        def loop_item():
            for i in range(K):
                losses, metrics = step(i)
                [v.item() for v in losses.values()] + [v.item() for v in metrics.values()]

        def loop_states():
            ts.states.reset()
            for i in range(K):
                step(i)
                if (i + 1) % DISP == 0:
                    ts.states.last()
            ts.states.finalize()

        def timed(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3 / K

        timed(loop_item)                                  # warm-up: engines, graphs, loss objects, builder buffers
        timed(loop_states)
        item, states = [], []
        for _ in range(args.regions):
            item.append(timed(loop_item))
            states.append(timed(loop_states))
        line[workload] = {"item_ms_per_step": float(np.median(item)), "states_ms_per_step": float(np.median(states)),
                          "saved_ms_per_step": float(np.median(item) - np.median(states)),
                          "item_min_max": [min(item), max(item)], "states_min_max": [min(states), max(states)],
                          "npoints": N}
        del ts, m, tb
        torch.cuda.empty_cache()
    line["measured_on"] = gpu_identity(dev)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
