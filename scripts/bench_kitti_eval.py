#!/usr/bin/env python
"""Device time of the KITTI evaluator (frustum_convnet_b200/kitti_eval.py, csrc/kitti_eval.cu) at validation size.

    python scripts/bench_kitti_eval.py [--images 3769] [--calls 20] [--warmup 3]

The set is synthetic (oracle/kitti_synth.py, seed 0): 3 769 images (the KITTI val split), about 9 ground-truth lines
(DontCare included) and 15 detections per image.  Each call runs the three device entries on one stream; CUDA events
around each give the overlap pass, pass 1 (TP scores, sort, thresholds), pass 2 (statistics and the final vectors)
and their total; the host wall time of a whole ``evaluate_records`` call (record upload, workspace allocation, the
one read back) is reported too.  Medians over ``--calls`` calls after ``--warmup``.  Prints one JSON line with the
card name and its power limit.  Writes nothing to the tree."""
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


def make_bench_set(n_images=3769, seed=0):
    """-> (label line lists, result line lists): the benchmark's synthetic validation-size set."""
    from oracle import kitti_synth as ks
    return ks.make_set(seed, n_images, n_obj=8, det_rate=0.8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from bench_detect import gpu_identity
    from frustum_convnet_b200.kitti_eval import KittiEvaluator, KittiGroundTruth
    from oracle import kitti_synth as ks
    assert torch.cuda.is_available(), "bench_kitti_eval.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    labels, results = make_bench_set(args.images)
    gts = [ks.parse_label_lines(l) for l in labels]
    dets = [ks.parse_result_lines(r) for r in results]
    ev = KittiEvaluator(KittiGroundTruth(list(range(len(gts))), gts, dev))
    stream = torch.cuda.current_stream(dev)

    phases = ("fcn_kitti_eval_overlaps", "fcn_kitti_eval_thresholds", "fcn_kitti_eval_statistics")
    rec = {p: [] for p in ("overlaps", "pass1", "pass2", "total", "call_wall")}
    res = None
    for it in range(args.warmup + args.calls):
        marks = {}

        def timer(name):
            e = torch.cuda.Event(enable_timing=True)
            e.record(stream)
            marks[name] = e

        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = ev.evaluate_records(dets, stream=stream, timer=timer)
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
        if it < args.warmup:
            continue
        t_ov = marks["start"].elapsed_time(marks[phases[0]])
        t_p1 = marks[phases[0]].elapsed_time(marks[phases[1]])
        t_p2 = marks[phases[1]].elapsed_time(marks[phases[2]])
        rec["overlaps"].append(t_ov)
        rec["pass1"].append(t_p1)
        rec["pass2"].append(t_p2)
        rec["total"].append(t_ov + t_p1 + t_p2)
        rec["call_wall"].append(wall)
    med = {k + "_ms": float(np.median(v)) for k, v in rec.items()}
    out = {"bench": "kitti_eval", "images": len(gts), "gt_lines": int(sum(len(g) for g in gts)),
           "detections": int(sum(len(d) for d in dets)), "calls": args.calls, **med,
           "total_ms_min": float(np.min(rec["total"])), "total_ms_max": float(np.max(rec["total"])),
           "ap_3d_car": [float(v) for v in res.ap["3d"].get("car", [])], **gpu_identity(dev)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
