#!/usr/bin/env python
"""Time of the KITTI first-stage ground-truth extractor (frustum_convnet_b200/gt_extract.py, csrc/gt_extract.cu) per
frame.

    python scripts/bench_gt_extract.py [--frames 64] [--points 120000] [--boxes 8] [--calls 20] [--warmup 3]

The scenes are synthetic (oracle/kitti_refine_synth.large_scene, seed 0): KITTI-sized scans (~120k points) with 8
ground-truth objects a frame and 2-D detections made from their result lines, 64 frames per call, whitelist Car.
Modes: train (from_ground_truth, perturb, augment = 5: --gen_train), val (from_ground_truth: --gen_val) and matched
(from_matched_detections, perturb, augment = 5: the _det extension).  Reported per frame and mode, medians over
``--calls`` calls after ``--warmup``:
  count_us / write_us  CUDA events around the two device entries, scans already on the device;
  e2e_us               host wall time of a whole call from scans in pinned host memory: the H2D copy, the host job
                       table (perturbation and matching included), both passes and the one read back, until the outputs
                       are complete;
  oracle_us            oracle/gt_extract.extract (numpy, half-space test) on the host, one run.
Prints one JSON line with the card name and its power limit.  Writes nothing to the tree."""
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

WHITELIST = ("Car",)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--points", type=int, default=120000)
    ap.add_argument("--boxes", type=int, default=8)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from bench_detect import gpu_identity
    from frustum_convnet_b200.frustum_extract import read_rgb_detections
    from frustum_convnet_b200.gt_extract import GtFrustumExtractor
    from oracle import gt_extract as ogx
    from oracle import kitti_refine_synth as krs
    from oracle.make_golden_gt_extract import det_lines
    assert torch.cuda.is_available(), "bench_gt_extract.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scans, calibs, hw, labels, results = krs.large_scene(0, args.frames, args.points, args.boxes)
    keys = sorted(scans)
    # The synthetic labels clip 2-D boxes to the image, which can leave an object outside it with xmin == xmax; the
    # reference's random_shift_box2d asserts on such a box (so does the extractor), and KITTI's labels have none.
    gt = {k: [o for o in v if o.xmin < o.xmax and o.ymin < o.ymax] for k, v in krs.objects(labels).items()}
    dets = read_rgb_detections([ln for ln in det_lines(results)
                                if (lambda b: b[0] < b[2] and b[1] < b[3])([float(x) for x in ln.split(" ")[3:7]])])
    pinned = torch.from_numpy(np.concatenate([scans[k] for k in keys])).pin_memory()
    off = np.concatenate([[0], np.cumsum([len(scans[k]) for k in keys])])
    dev_scans = {k: torch.from_numpy(scans[k]).to(dev) for k in keys}
    ex = GtFrustumExtractor(WHITELIST, dev)
    stream = torch.cuda.current_stream(dev)
    calls = {
        "train": lambda s, t: ex.from_ground_truth(s, calibs, hw, keys, gt, perturb=True, augment=5,
                                                   rng=np.random.RandomState(1), timer=t),
        "val": lambda s, t: ex.from_ground_truth(s, calibs, hw, keys, gt, timer=t),
        "matched": lambda s, t: ex.from_matched_detections(s, calibs, hw, keys, *dets, gt, perturb=True, augment=5,
                                                           rng=np.random.RandomState(1), timer=t),
    }
    oracle = {
        "train": lambda: ogx.extract("gt", scans, calibs, hw, keys, gt, WHITELIST, True, 5, np.random.RandomState(1)),
        "val": lambda: ogx.extract("gt", scans, calibs, hw, keys, gt, WHITELIST),
        "matched": lambda: ogx.extract("matched", scans, calibs, hw, keys, gt, WHITELIST, True, 5,
                                       np.random.RandomState(1), dets),
    }
    out = {"bench": "gt_extract", "frames": args.frames, "scan_points": int(off[-1]), "calls": args.calls}
    for mode, call in calls.items():
        rec = {"count": [], "write": [], "e2e": []}
        fr = None
        for it in range(args.warmup + args.calls):
            marks = {}

            def timer(name):
                e = torch.cuda.Event(enable_timing=True)
                e.record(stream)
                marks[name] = e

            torch.cuda.synchronize()
            fr = call(dev_scans, timer)
            torch.cuda.synchronize()
            t_count = marks["start"].elapsed_time(marks["count"])
            t_write = marks["write_start"].elapsed_time(marks["write"])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            flat = pinned.to(dev, non_blocking=True)
            call({k: flat[off[i]:off[i + 1]] for i, k in enumerate(keys)}, None)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            if it < args.warmup:
                continue
            rec["count"].append(t_count * 1e3 / args.frames)
            rec["write"].append(t_write * 1e3 / args.frames)
            rec["e2e"].append(wall * 1e6 / args.frames)
        t0 = time.perf_counter()
        ref = oracle[mode]()
        t_oracle = time.perf_counter() - t0
        assert ref["id_list"] == fr.id_list and fr.counts.tolist() == [len(p) for p in ref["input_list"]], \
            "device and oracle disagree (%s)" % mode
        out[mode] = {"frustums": len(fr), "frustum_points": int(fr.counts.sum()),
                     **{k + "_us_per_frame": float(np.median(v)) for k, v in rec.items()},
                     "oracle_us_per_frame": t_oracle * 1e6 / args.frames}
    out.update(gpu_identity(dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
