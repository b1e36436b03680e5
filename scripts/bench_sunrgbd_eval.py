#!/usr/bin/env python
"""Device time of the SUN-RGBD evaluator (frustum_convnet_b200/sunrgbd_eval.py, csrc/sunrgbd_eval.cu) at validation
size.

    python scripts/bench_sunrgbd_eval.py [--images 5050] [--calls 20] [--warmup 3]

The set is synthetic (oracle/sunrgbd_synth.py, seed 0): 5 050 images (the val split), about 17 k ground-truth boxes
over the 10 classes and about 150 k detections, most of them false positives, as the frustums of the 2-D detections
give.  Each call runs the two device entries on one stream; CUDA events around each give the match phase (overlaps,
sort, claims) and the curves phase (rec, prec, AP) and their total; the host wall time of a whole ``evaluate`` call
(corner construction, the upload, workspace allocation, the one read back) is reported too.  Medians over ``--calls``
calls after ``--warmup``.  Prints one JSON line with the card name and its power limit.  Writes nothing to the tree."""
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


def make_bench_set(n_images=5050, seed=0):
    """-> (gt rows {class: (n, 10)}, gt ids {class: (n,)}, det_results): the benchmark's synthetic val-size set."""
    from oracle import sunrgbd_eval as ose
    from oracle import sunrgbd_synth as ss
    return ss.make_set(seed, n_images, ose.CLASS_NAMES, check_margins=False, gt_mean=0.26, fp_rate=2.5)


def ground_truth(gt_rows, gt_ids, dev):
    from frustum_convnet_b200.sunrgbd_eval import CLASS_NAMES, SunrgbdGroundTruth, gt_corners
    return SunrgbdGroundTruth({c: (gt_corners(gt_rows[c]), gt_ids[c]) for c in CLASS_NAMES}, device=dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=5050)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from bench_detect import gpu_identity
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator
    assert torch.cuda.is_available(), "bench_sunrgbd_eval.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gt_rows, gt_ids, det_results = make_bench_set(args.images)
    ev = SunrgbdEvaluator(ground_truth(gt_rows, gt_ids, dev))
    stream = torch.cuda.current_stream(dev)

    phases = ("fcn_sunrgbd_eval_match", "fcn_sunrgbd_eval_curves")
    rec = {p: [] for p in ("match", "curves", "total", "call_wall")}
    res = None
    for it in range(args.warmup + args.calls):
        marks = {}

        def timer(name):
            e = torch.cuda.Event(enable_timing=True)
            e.record(stream)
            marks[name] = e

        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = ev.evaluate(det_results, stream=stream, timer=timer)
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
        if it < args.warmup:
            continue
        t_m = marks["start"].elapsed_time(marks[phases[0]])
        t_c = marks[phases[0]].elapsed_time(marks[phases[1]])
        rec["match"].append(t_m)
        rec["curves"].append(t_c)
        rec["total"].append(t_m + t_c)
        rec["call_wall"].append(wall)
    med = {k + "_ms": float(np.median(v)) for k, v in rec.items()}
    out = {"bench": "sunrgbd_eval", "images": args.images, "gt_boxes": int(sum(len(r) for r in gt_rows.values())),
           "detections": int(sum(len(v) for by in det_results.values() for v in by.values())), "calls": args.calls,
           **med, "total_ms_min": float(np.min(rec["total"])), "total_ms_max": float(np.max(rec["total"])),
           "mean_ap": res.mean_ap, **gpu_identity(dev)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
