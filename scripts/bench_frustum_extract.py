#!/usr/bin/env python
"""Time of the KITTI frustum extractor (frustum_convnet_b200/frustum_extract.py, csrc/frustum_extract.cu) per frame.

    python scripts/bench_frustum_extract.py [--frames 64] [--points 120000] [--dets 8] [--calls 20] [--warmup 3]

The scenes are synthetic (oracle/kitti_scan_synth.large_scene, seed 0): KITTI-sized scans (~120k points) with 8
detections a frame, 64 frames per call, whitelist Car, Pedestrian, Cyclist.  Reported per frame, medians over
``--calls`` calls after ``--warmup``:
  kernel_us_per_frame  CUDA events around the two device entries (count pass; write pass), scans already on the device;
  e2e_us_per_frame     host wall time of a whole call from scans in pinned host memory: the H2D copy, the extractor
                       (upload of calib and boxes, both passes, the one read back) until the outputs are complete;
  oracle_us_per_frame  oracle/frustum_extract.extract (the reference's loop restated in numpy) on the host, one run.
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

WHITELIST = ("Car", "Pedestrian", "Cyclist")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--points", type=int, default=120000)
    ap.add_argument("--dets", type=int, default=8)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from bench_detect import gpu_identity
    from frustum_convnet_b200.frustum_extract import FrustumExtractor
    from oracle import frustum_extract as ofx
    from oracle import kitti_scan_synth as ks
    assert torch.cuda.is_available(), "bench_frustum_extract.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scans, calibs, hw, ids, types, probs, boxes = ks.large_scene(0, args.frames, args.points, args.dets)
    keys = sorted(scans)
    n_points = sum(len(scans[k]) for k in keys)
    pinned = torch.from_numpy(np.concatenate([scans[k] for k in keys])).pin_memory()
    off = np.concatenate([[0], np.cumsum([len(scans[k]) for k in keys])])
    dev_scans = {k: torch.from_numpy(scans[k]).to(dev) for k in keys}
    ex = FrustumExtractor(WHITELIST, dev)
    stream = torch.cuda.current_stream(dev)

    rec = {"kernel": [], "count": [], "write": [], "e2e": []}
    fr = None
    for it in range(args.warmup + args.calls):
        marks = {}

        def timer(name):
            e = torch.cuda.Event(enable_timing=True)
            e.record(stream)
            marks[name] = e

        torch.cuda.synchronize()
        fr = ex.extract(dev_scans, calibs, hw, ids, types, probs, boxes, timer=timer)
        torch.cuda.synchronize()
        t_count = marks["start"].elapsed_time(marks["count"])
        t_write = marks["write_start"].elapsed_time(marks["write"])

        torch.cuda.synchronize()
        t0 = time.perf_counter()
        flat = pinned.to(dev, non_blocking=True)
        views = {k: flat[off[i]:off[i + 1]] for i, k in enumerate(keys)}
        ex.extract(views, calibs, hw, ids, types, probs, boxes)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        if it < args.warmup:
            continue
        rec["count"].append(t_count * 1e3 / args.frames)
        rec["write"].append(t_write * 1e3 / args.frames)
        rec["kernel"].append((t_count + t_write) * 1e3 / args.frames)
        rec["e2e"].append(wall * 1e6 / args.frames)

    t0 = time.perf_counter()
    ref = ofx.extract(scans, calibs, hw, ids, types, probs, boxes, WHITELIST)
    t_oracle = time.perf_counter() - t0
    assert len(ref[0]) == len(fr) and fr.counts.tolist() == [len(p) for p in ref[2]], "device and oracle disagree"
    out = {"bench": "frustum_extract", "frames": args.frames, "scan_points": n_points,
           "detections": len(ids), "kept": len(fr), "frustum_points": int(fr.counts.sum()), "calls": args.calls,
           **{k + "_us_per_frame": float(np.median(v)) for k, v in rec.items()},
           "kernel_us_per_frame_min": float(np.min(rec["kernel"])),
           "kernel_us_per_frame_max": float(np.max(rec["kernel"])),
           "oracle_us_per_frame": t_oracle * 1e6 / args.frames, **gpu_identity(dev)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
