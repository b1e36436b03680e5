#!/usr/bin/env python
"""What the deterministic training mode costs: ms per TrainStep.step with deterministic=False (the default kernels)
against deterministic=True (fcn_train_*_deterministic and fcn_det_loss_deterministic).

    python scripts/bench_train_deterministic.py [--batch 32] [--steps 50] [--regions 5]

Workloads: refine_car (N=512), car detection (N=1024) and SUN-RGBD (N=2048) at B = --batch, on a few resident
synthetic batches (synth.make_frustums), so the step alone is timed.  Both modes step their own copy of one model
with Adam; after warm-up steps (which capture the step's CUDA graphs) the two are timed in alternating regions of
`--steps` steps, host clock around a region that ends in a device synchronise.  Prints one JSON line: per workload
and mode the median and min / max ms per step and the TrainEngine workspace bytes, with the card name and power
limit.  Writes nothing to the tree."""
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

WORKLOADS = ("refine_car", "car", "sunrgbd")


def _model(workload, dev):
    import torch
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload(workload)
    if w["arch"].num_scales == 5:
        from frustum_convnet_b200.det_base_sunrgbd import PointNetDet
    else:
        from frustum_convnet_b200.det_base import PointNetDet
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=7)
    m = PointNetDet(3, num_vec=w["num_vec"])
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m.to(dev).train(), cfg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--regions", type=int, default=5)
    args = ap.parse_args()

    import torch
    from frustum_convnet_b200 import synth
    from frustum_convnet_b200.train_engine import TrainStep
    assert torch.cuda.is_available(), "bench_train_deterministic.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, K = args.batch, args.steps
    line = {"batch": B, "steps_per_region": K, "regions": args.regions}
    for workload in WORKLOADS:
        batches = []
        for s in range(4):
            d = synth.make_frustums(workload, B, seed=40 + s, with_labels=True,
                                    max_depth=(17.5 if workload == "car" else None))
            batches.append({k: torch.from_numpy(v).to(dev) for k, v in d.items()})
        steps = {}
        for det in (False, True):
            m, cfg = _model(workload, dev)
            steps[det] = TrainStep(m, lr=cfg.TRAIN.BASE_LR, weight_decay=cfg.TRAIN.WEIGHT_DECAY, deterministic=det)

        def region(ts):
            torch.cuda.synchronize()
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
        res = {}
        for det in (False, True):
            t = times[det]
            eng = next(iter(steps[det].engines.values()))
            res["deterministic" if det else "default"] = {
                "ms_per_step": float(np.median(t)), "min": float(min(t)), "max": float(max(t)),
                "workspace_bytes": int(eng.workspace.numel() * 4)}
        res["overhead_pct"] = 100.0 * (res["deterministic"]["ms_per_step"] / res["default"]["ms_per_step"] - 1.0)
        line[workload] = res
        del steps, batches
        torch.cuda.empty_cache()
    line.update(gpu_identity(dev))
    print(json.dumps(line))


if __name__ == "__main__":
    main()
