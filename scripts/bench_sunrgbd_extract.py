#!/usr/bin/env python
"""Time of the SUN-RGBD frustum extractor (frustum_convnet_b200/sunrgbd_extract.py, csrc/sunrgbd_extract.cu) per
frame.

    python scripts/bench_sunrgbd_extract.py [--frames 64] [--calls 5] [--warmup 2]

The frames are synthetic at SUN-RGBD scale (oracle/sunrgbd_scene_synth.large_set, seed 0): a 530 x 730 depth grid
(386,900 points a frame) and 8 objects of the 10 classes plus a lamp, most frustums above 2048 points; detections are
the label boxes jittered.  Sets: train (from_ground_truth, perturb, augment = 5: --gen_train), val (from_ground_truth:
--gen_val) and det (from_rgb_detections: --gen_val_rgb_detection).  Reported per frame and set, medians over ``--calls``
calls after ``--warmup``:
  project_us / count_us / select_us / write_us  CUDA events around each device entry (count: summed over the rounds),
                                                clouds already on the device;
  rounds                                        count rounds of one call;
  replay_us                                     the host's draws alone (sunrgbd_extract.replay with the counts known:
                                                the box perturbations and np.random.choice's permutation(n));
  e2e_us                                        host wall time of a whole call from clouds in pinned host memory;
  oracle_us                                     oracle/sunrgbd_extract (numpy, the reference's order) on the host, once;
  count_l2_bytes_per_frame                      from shapes: each counted job reads its frame's 16 bytes of u, v a
                                                point.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import torch
    from bench_detect import gpu_identity
    from frustum_convnet_b200 import sunrgbd_extract as sx
    from oracle import sunrgbd_extract as osx
    from oracle import sunrgbd_scene_synth as sss
    assert torch.cuda.is_available(), "bench_sunrgbd_extract.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    points, calibs, labels, dets = sss.large_set(0, n_frames=args.frames)
    keys = sorted(points)
    pinned = torch.from_numpy(np.concatenate([points[k] for k in keys])).pin_memory()
    off = np.concatenate([[0], np.cumsum([len(points[k]) for k in keys])])
    dev_points = {k: torch.from_numpy(points[k]).to(dev) for k in keys}
    ex = sx.SunrgbdFrustumExtractor(device=dev)
    stream = torch.cuda.current_stream(dev)
    calls = {
        "train": lambda p, t, rng: ex.from_ground_truth(p, calibs, keys, labels, perturb=True, augment=5, rng=rng,
                                                        timer=t),
        "val": lambda p, t, rng: ex.from_ground_truth(p, calibs, keys, labels, rng=rng, timer=t),
        "det": lambda p, t, rng: ex.from_rgb_detections(p, calibs, *dets, rng=rng, timer=t),
    }
    oracle = {
        "train": lambda: osx.from_ground_truth(points, calibs, keys, labels, perturb=True, augment=5,
                                               rng=np.random.RandomState(1)),
        "val": lambda: osx.from_ground_truth(points, calibs, keys, labels, rng=np.random.RandomState(1)),
        "det": lambda: osx.from_rgb_detections(points, calibs, *dets, rng=np.random.RandomState(1)),
    }
    out = {"bench": "sunrgbd_extract", "frames": args.frames, "cloud_points": int(off[-1]), "calls": args.calls}
    for mode, call in calls.items():
        rec = {k: [] for k in ("project", "count", "select", "write", "replay", "e2e")}
        fr = None
        for it in range(args.warmup + args.calls):
            marks, rounds = {}, []

            def timer(name):
                e = torch.cuda.Event(enable_timing=True)
                e.record(stream)
                if name == "round_start":
                    rounds.append([e])
                elif name == "round_end":
                    rounds[-1].append(e)
                else:
                    marks[name] = e

            torch.cuda.synchronize()
            fr = call(dev_points, timer, np.random.RandomState(1))
            torch.cuda.synchronize()
            t = {"project": marks["start"].elapsed_time(marks["project"]),
                 "count": sum(a.elapsed_time(b) for a, b in rounds),
                 "select": marks["count"].elapsed_time(marks["select"]),
                 "write": marks["write_start"].elapsed_time(marks["write"])}
            # the host's draws alone: replay with the counts this call learnt
            slots = _slots(mode, keys, labels, dets, sx)
            n_of = _counts_of(fr, slots, mode, points, calibs, osx) if it == 0 else n_of
            t0 = time.perf_counter()
            sx.replay(slots, mode == "train", np.random.RandomState(1), lambda b, e, c: n_of[b:e])
            t["replay"] = (time.perf_counter() - t0) * 1e3
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            flat = pinned.to(dev, non_blocking=True)
            call({k: flat[off[i]:off[i + 1]] for i, k in enumerate(keys)}, None, np.random.RandomState(1))
            torch.cuda.synchronize()
            t["e2e"] = (time.perf_counter() - t0) * 1e3
            if it >= args.warmup:
                for k, v in t.items():
                    rec[k].append(v * 1e3 / args.frames)
        t0 = time.perf_counter()
        ref, _ = oracle[mode]()
        t_oracle = time.perf_counter() - t0
        assert ref["id"] == fr.id_list and fr.counts.tolist() == [len(p) for p in ref["input"]], \
            "device and oracle disagree (%s)" % mode
        live = [s for s in slots if not s["skip"]]
        out[mode] = {"jobs": len(live), "frustums": len(fr), "frustum_points": int(fr.counts.sum()),
                     "rounds": int(fr.rounds),
                     **{k + "_us_per_frame": float(np.median(v)) for k, v in rec.items()},
                     "oracle_us_per_frame": t_oracle * 1e6 / args.frames,
                     "count_l2_bytes_per_frame": 16.0 * sum(len(points[s["frame"]]) for s in live) / args.frames}
    out.update(gpu_identity(dev))
    print(json.dumps(out))


def _slots(mode, keys, labels, dets, sx):
    if mode == "det":
        ids, types, boxes, _ = dets
        return [dict(frame=i, box=b, skip=False) for i, t, b in zip(ids, types, boxes) if t in sx.TYPE_WHITELIST]
    aug = 5 if mode == "train" else 1
    return [dict(frame=k, box=o.box2d, skip=sx.zero_extent(o)) for k in keys for o in labels[k]
            if o.classname in sx.TYPE_WHITELIST for _ in range(aug)]


def _counts_of(fr, slots, mode, points, calibs, osx):
    """Every live job's in-box count, from the oracle's projection (the counts the device returned)."""
    live = [s for s in slots if not s["skip"]]
    count = osx.counter(points, calibs, slots)
    if mode != "train":
        return count(0, len(live), np.array([s["box"] for s in live]))
    from frustum_convnet_b200 import sunrgbd_extract as sx
    cuts, n, _, _ = sx.replay(slots, True, np.random.RandomState(1), count)
    return n[[k for k, s in enumerate(slots) if not s["skip"]]]


if __name__ == "__main__":
    main()
