#!/usr/bin/env python
"""Scoring a DetectionCollector's rows: ``finalize()`` + ``evaluate(dict)`` against ``finalize_device()`` +
``evaluate_collected`` for KITTI and SUN-RGBD at validation size.

    python scripts/bench_det_eval.py [--kitti-images 3769] [--sunrgbd-images 5050] [--calls 20] [--warmup 3]

The sets are those of scripts/bench_kitti_eval.py (oracle/kitti_synth.py, seed 0) and scripts/bench_sunrgbd_eval.py
(oracle/sunrgbd_synth.py, seed 0).  Their detections are fed through a collector (one frustum per row, method 'top',
tests/det_feed_sets.py), added once; each call finalizes and evaluates.  Per path: host wall time of the whole call
(finalize, evaluation and the result's read back) and the device time of the evaluation, between CUDA events recorded
before its first device entry (the feed kernel on the device path, the evaluator after the record upload on the dict
path) and after its last evaluator entry.  Medians over ``--calls`` calls after ``--warmup``, the two paths
alternating.  Prints one JSON line with the card name and its power limit.  Writes nothing to the tree."""
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


def time_paths(col, ev, calls, warmup, stream):
    import torch
    rec = {k: [] for k in ("dict_wall", "dict_device", "device_wall", "device_device")}
    last = {}
    for it in range(warmup + calls):
        for path in ("dict", "device"):
            marks = {}

            def timer(name):
                e = torch.cuda.Event(enable_timing=True)
                e.record(stream)
                marks[name] = e

            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if path == "dict":
                res = ev.evaluate(col.finalize(), stream=stream, timer=timer)
            else:
                res = ev.evaluate_collected(col.finalize_device(), stream=stream, timer=timer)
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            last[path] = res
            if it < warmup:
                continue
            end = [k for k in marks if k.startswith("fcn_")][-1]
            rec[path + "_wall"].append(wall)
            rec[path + "_device"].append(marks["feed_start" if path == "device" else "start"].elapsed_time(marks[end]))
    return {k + "_ms": float(np.median(v)) for k, v in rec.items()}, last


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kitti-images", type=int, default=3769)
    ap.add_argument("--sunrgbd-images", type=int, default=5050)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from bench_detect import gpu_identity
    from bench_sunrgbd_eval import ground_truth, make_bench_set
    from det_feed_sets import collector_for, kitti_set
    from frustum_convnet_b200.kitti_eval import KittiEvaluator, KittiGroundTruth
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator
    assert torch.cuda.is_available(), "bench_det_eval.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.current_stream(dev)
    out = {"bench": "det_eval", "calls": args.calls}

    gts, dets = kitti_set(args.kitti_images, seed=0)
    ev = KittiEvaluator(KittiGroundTruth(list(range(len(gts))), gts, dev))
    col = collector_for(dets, "KITTI", device=dev)
    med, last = time_paths(col, ev, args.calls, args.warmup, stream)
    same = all(np.array_equal(last["dict"].precision[m][c], last["device"].precision[m][c])
               for m in last["dict"].precision for c in last["dict"].precision[m])
    out["kitti"] = {"images": len(gts), "rows": col.last_counts["kept"], **med, "precision_identical": same,
                    "ap_3d_car": [float(v) for v in last["device"].ap["3d"].get("car", [])]}

    gt_rows, gt_ids, sdets = make_bench_set(args.sunrgbd_images)
    sev = SunrgbdEvaluator(ground_truth(gt_rows, gt_ids, dev))
    scol = collector_for(sdets, "SUNRGBD", device=dev)
    med, last = time_paths(scol, sev, args.calls, args.warmup, stream)
    out["sunrgbd"] = {"images": args.sunrgbd_images, "rows": scol.last_counts["kept"], **med,
                      "mean_ap_dict": last["dict"].mean_ap, "mean_ap_device": last["device"].mean_ap}
    out.update(gpu_identity(dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
