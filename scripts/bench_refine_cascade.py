#!/usr/bin/env python
"""Time of the handoff between the KITTI stages: the first stage's DetectionCollector -> the refinement frustums ->
the refinement batch table, through the host dict and straight from the collector's device rows.

    python scripts/bench_refine_cascade.py [--frames 64] [--points 120000] [--images 3769] [--calls 10] [--warmup 2]

The scenes are synthetic (oracle/kitti_refine_synth.large_scene, seed 0): KITTI-sized scans with 8 objects a frame,
their result lines fed through a DetectionCollector as first-stage outputs (tests/det_feed_sets.collector_for), whose
segment table spans `--images` images (the KITTI val split's 3769; the images without a scene have frustums that are
never added), whitelist Car, Pedestrian, Cyclist.  Paths, alternated call by call:
  dict    col.finalize() -> from_detections / from_matched_detections -> TrainBatchBuilder.from_frustums (host table);
  device  col.finalize_device() -> from_collected / from_matched_collected -> from_frustums (device records).
Reported per mode (det, matched) and path, medians over ``--calls`` calls after ``--warmup``: wall_ms, host wall time
of the whole handoff from the collector to the installed builder (scans already on the device); device_ms, CUDA events
from the extractor's first device call to its last.  Prints one JSON line with the card name and its power limit.
Writes nothing to the tree."""
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

WHITELIST = ("Car", "Pedestrian", "Cyclist")
STRIDES = [0.1, 0.2, 0.4, 0.8]          # cfgs/refine_car.yaml


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--points", type=int, default=120000)
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch
    from bench_detect import gpu_identity
    from det_feed_sets import collector_for
    from frustum_convnet_b200.refine_extract import RefineFrustumExtractor
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    from oracle import kitti_refine_synth as krs
    assert torch.cuda.is_available(), "bench_refine_cascade.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    scans, calibs, hws, labels, results = krs.large_scene(0, n_frames=args.frames, n_points=args.points)
    ids = sorted(scans)
    dets = {}
    for i, objs in krs.objects(results).items():
        rows = {}
        for o in objs:
            rows.setdefault(o.type, []).append(list(o.box2d) + list(o.t) + [o.h, o.w, o.l, o.ry, o.score])
        dets[i] = {c: np.array(r, np.float32) for c, r in rows.items()}
    others = [i for i in range(args.images) if i not in scans]
    col = collector_for(dets, "KITTI", extra_frustums=[(i, "Car") for i in others], device=dev)
    image_ids = sorted(set(range(args.images)) | set(ids))
    gt = krs.objects(labels)
    gt = {i: gt.get(i, []) for i in image_ids}
    dscans = {k: torch.from_numpy(v).to(dev) for k, v in scans.items()}
    x = RefineFrustumExtractor(WHITELIST, device=dev)
    stream = torch.cuda.current_stream(dev)

    def run(mode, path, timer):
        if path == "dict":
            d = col.finalize()
            fr = (x.from_detections(dscans, calibs, hws, image_ids, d, timer=timer) if mode == "det" else
                  x.from_matched_detections(dscans, calibs, hws, image_ids, d, gt, remove_diff=True, timer=timer))
        else:
            c = col.finalize_device()
            fr = (x.from_collected(dscans, calibs, hws, image_ids, c, timer=timer) if mode == "det" else
                  x.from_matched_collected(dscans, calibs, hws, image_ids, c, gt, remove_diff=True, timer=timer))
        TrainBatchBuilder.from_frustums(fr, "refine", strides=STRIDES, npoints=512)
        return len(fr)

    out = {"frames": args.frames, "points": args.points, "images": args.images, "calls": args.calls}
    for mode in ("det", "matched"):
        rec = {k: [] for k in ("dict_wall", "dict_device", "device_wall", "device_device")}
        n = {}
        for it in range(args.warmup + args.calls):
            for path in ("dict", "device"):
                marks = {}

                def timer(name):
                    e = torch.cuda.Event(enable_timing=True)
                    e.record(stream)
                    marks[name] = e

                torch.cuda.synchronize()
                t0 = time.perf_counter()
                n[path] = run(mode, path, timer)
                torch.cuda.synchronize()
                wall = (time.perf_counter() - t0) * 1e3
                if it < args.warmup:
                    continue
                rec[path + "_wall"].append(wall)
                rec[path + "_device"].append(marks["start"].elapsed_time(marks[list(marks)[-1]]))
        assert n["dict"] == n["device"], n
        out[mode] = dict({k + "_ms": round(float(np.median(v)), 3) for k, v in rec.items()}, frustums=n["device"])
    out.update(gpu_identity(dev))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
