#!/usr/bin/env python
"""Cost of the device detection step (frustum_convnet_b200/detect.py, csrc/detect.cu) next to the eval forward.

    python scripts/bench_detect.py [--workload car|people|sunrgbd] [--batch 32] [--steps 200] [--regions 5]

One step = one graph-replayed forward of `--batch` synthetic frustums on one stream.  Regions of `--steps` steps
alternate between the plain forward and the forward followed by one `DetectionCollector.add` (same stream), timed
with CUDA events; `extra_ms_per_step` = median(with add) - median(plain).  Then `finalize()` (sort, NMS at the
reference's default cfg.TEST.THRESH 0.1, one host sync, copy of the kept rows) over the last region's frustums,
grouped 8 per image, timed with a host clock, median of 5 calls.  Prints one JSON line with the card name and its
power limit.  Writes nothing to the tree."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_identity(dev):
    """Card name and power limit (W), read in the same run as the measurement."""
    import torch
    ident = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(dev.index or 0)], capture_output=True, text=True, timeout=30)
        ident["power_limit_w"] = float(out.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return ident


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="car", choices=["car", "people", "sunrgbd"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--regions", type=int, default=5)
    args = ap.parse_args()

    import torch
    from frustum_convnet_b200 import config, synth
    from frustum_convnet_b200.detect import DetectionCollector
    assert torch.cuda.is_available(), "bench_detect.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg, w = config.load_workload(args.workload)
    modname = "det_base_sunrgbd" if w["arch"].num_scales == 5 else "det_base"
    mod = __import__("frustum_convnet_b200." + modname, fromlist=["PointNetDet"])
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=7)
    model = mod.PointNetDet(3, num_vec=w["num_vec"])
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    model = model.to(dev).eval()
    model.use_cuda_graph = True
    model.freeze()
    B = args.batch
    pool = [{k: torch.from_numpy(v).to(dev) for k, v in synth.make_frustums(args.workload, B, seed=1234 + i).items()}
            for i in range(8)]
    extra = {"rot_angle": torch.linspace(-0.6, 0.6, B, device=dev)}
    F = args.steps * B
    cls = {"car": "Car", "people": "Pedestrian", "sunrgbd": "bed"}[args.workload]
    with torch.no_grad():
        T2 = int(model(pool[0])[0].shape[1])
    col = DetectionCollector([f // 8 for f in range(F)], [cls] * F, np.zeros((F, 4), np.float32),
                             dataset=cfg.DATA.DATASET_NAME, method="nms", thresh=0.1, capacity=F * T2, device=dev)

    def region(with_add):
        col.reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        with torch.no_grad():
            for i in range(args.steps):
                out = model(pool[i % len(pool)])
                if with_add:
                    col.add(out, extra, first=i * B)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    region(False)                                   # warm-up: graph capture, module loads, clocks
    region(True)
    plain, added = [], []
    for _ in range(args.regions):
        plain.append(region(False))
        added.append(region(True))
    fin = []
    for _ in range(5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = col.finalize()
        fin.append((time.perf_counter() - t0) * 1e3)
    line = {
        "workload": args.workload, "batch": B, "steps": args.steps, "regions": args.regions,
        "resident_ms_per_step": float(np.median(plain)), "resident_ms_per_step_with_add": float(np.median(added)),
        "extra_ms_per_step": float(np.median(added) - np.median(plain)),
        "plain_ms_per_step_min_max": [min(plain), max(plain)], "with_add_ms_per_step_min_max": [min(added), max(added)],
        "finalize_ms_median": float(np.median(fin)), "finalize_ms_min_max": [min(fin), max(fin)],
        "frustums": F, "images": (F + 7) // 8, "lists": sum(len(v) for v in res.values()),
        "candidates": col.last_counts["rows"], "kept": col.last_counts["kept"], "thresh": 0.1,
        "measured_on": gpu_identity(dev),
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
