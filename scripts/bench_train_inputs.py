#!/usr/bin/env python
"""Cost of building labelled training batches on the device (frustum_convnet_b200/train_inputs.py,
csrc/train_inputs.cu) next to the reference-equivalent host path.

    python scripts/bench_train_inputs.py [--frustums 8192] [--steps 200] [--regions 5] [--ref-batches 10]

Workloads: car detection (B=32, N=1024, strides 0.25..2, max depth 70), refinement (B=32, N=512, strides 0.1..0.8)
and SUN-RGBD (B=32, N=2048, strides 0.1..1.6, max depth 8, synthetic tilted K / Rtilt, float32 box2d, 6-column
points) over a resident synthetic dataset of `--frustums` frustums (refine predicted-box widths in [1.91, 1.95] m, so
every batch has T = (20, 10, 5, 3) and one training-step shape).  Per workload:
  build_ms_per_batch     device time of `--steps` build() calls (one H2D copy of the draws + one launch), CUDA events,
                         draws prepared in advance;
  launch_ms_per_batch    the same for the kernel alone (launch());
  draw_ms_per_batch      host time of draw() (the np.random calls that stay on the CPU);
  reference_ms_per_batch host time of the reference-equivalent numpy path, single process: the providers' per-item
                         numpy code (oracle/train_inputs.py) with scipy Delaunay inside-box tests as the reference's
                         in_hull does, the collate and torch.from_numpy, no H2D copy;
and for refinement and SUN-RGBD, train_extra_ms_per_step: regions of `--steps` TrainStep.step calls on one prebuilt
batch alternate with regions where build() precedes each step (same stream), median(with) - median(without).
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

from bench_detect import gpu_identity  # noqa: E402

CAR, REFINE, SUN = (0.25, 0.5, 1.0, 2.0), (0.1, 0.2, 0.4, 0.8), (0.1, 0.2, 0.4, 0.8, 1.6)
MAX_DEPTH = {"det": 70.0, "refine": 70.0, "sunrgbd": 8.0}


def synthetic_sun_lists(F, seed):
    """F SUN-RGBD frustums in the prepared pickles' dtypes (float32 points with 6 columns, float32 box2d, bool seg)."""
    from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES, compute_box_3d
    rng = np.random.default_rng(seed)
    n = rng.integers(200, 2500, F)
    L = {k: [] for k in ("input_list", "type_list", "box2d_list", "frustum_angle_list", "calib_K_list",
                         "calib_R_list", "label_list", "box3d_list", "heading_list", "size_list")}
    for i in range(F):
        K = np.array([[529.5, 0, 365.0], [0, 531.0, 262.0], [0, 0, 1]])
        ax = rng.uniform(-0.15, 0.15)
        R = np.array([[1, 0, 0], [0, np.cos(ax), -np.sin(ax)], [0, np.sin(ax), np.cos(ax)]])
        C = np.array([rng.uniform(-2, 2), rng.uniform(-0.5, 1.0), rng.uniform(1, 7.5)])
        size, heading = rng.uniform(0.4, 2.2, 3), rng.uniform(-np.pi, np.pi)
        up = R.T @ np.array([C[0], C[2], -C[1]])                     # upright camera -> depth -> pixel
        u, v = K[0, 0] * up[0] / up[1] + K[0, 2], K[1, 1] * -up[2] / up[1] + K[1, 2]
        L["input_list"].append(np.concatenate([C + rng.normal(0, 0.5, (n[i], 3)), rng.uniform(0, 1, (n[i], 3))],
                                              1).astype(np.float32))
        L["type_list"].append(SUNRGBD_CLASSES[rng.integers(0, 10)])
        L["box2d_list"].append(np.array([u - 40, v - 30, u + 40, v + 30], dtype=np.float32))
        L["frustum_angle_list"].append(float(-np.arctan2(C[2], C[0])))
        L["calib_K_list"].append(K)
        L["calib_R_list"].append(R)
        L["label_list"].append(rng.uniform(0, 1, n[i]) < 0.3)
        L["box3d_list"].append(compute_box_3d(C, size, heading))
        L["heading_list"].append(float(heading))
        L["size_list"].append(size)
    return L


def synthetic_lists(kind, F, seed):
    """F frustums in the reference's dtypes (det points float32, refine train points float64)."""
    from frustum_convnet_b200.train_inputs import compute_box_3d
    rng = np.random.default_rng(seed)
    Pm = np.array([[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791], [0.0, 0.0, 1.0, 0.002745884]])
    n = rng.integers(200, 2500, F)
    size = np.array([3.9, 1.6, 1.5]) * rng.uniform(0.85, 1.15, (F, 3))
    C = np.stack([rng.uniform(-15, 15, F), rng.uniform(0.5, 2.0, F), rng.uniform(3, 67, F)], 1)
    heading = rng.uniform(-np.pi, np.pi, F)
    dtype = np.float32 if kind == "det" else np.float64
    L = {"input_list": [(C[i] + rng.normal(0, 1.5, (n[i], 3))).astype(dtype) for i in range(F)],
         "type_list": ["Car"] * F, "box3d_list": [compute_box_3d(C[i], size[i], heading[i]) for i in range(F)],
         "heading_list": [float(h) for h in heading], "size_list": list(size)}
    if kind == "det":
        L["label_list"] = [(rng.uniform(0, 1, k) < 0.3).astype(np.float64) for k in n]
        L["frustum_angle_list"] = [float(-np.arctan2(c[2], c[0])) for c in C]
        L["calib_list"] = [{"P2": Pm.reshape(-1)}] * F
        u = (Pm[0, 0] * C[:, 0] + Pm[0, 2] * C[:, 2] + Pm[0, 3]) / C[:, 2]
        v = (Pm[1, 1] * C[:, 1] + Pm[1, 2] * C[:, 2] + Pm[1, 3]) / C[:, 2]
        L["box2d_list"] = [np.array([a - 40, b - 30, a + 40, b + 30]) for a, b in zip(u, v)]
    else:
        pa = heading + rng.normal(0, 0.2, F)
        psize = size * rng.uniform(0.9, 1.1, (F, 3))
        psize[:, 1] = rng.uniform(1.91, 1.95, F)
        L["pred_box3d_list"] = [compute_box_3d(C[i] + rng.normal(0, 0.3, 3), psize[i], pa[i]) for i in range(F)]
        L["pred_box3d_size_list"] = list(psize)
        L["pred_box3d_angle_list"] = [float(a) for a in pa]
    return L


def reference_path_ms(kind, L, batches, strides, max_depth):
    """Host time per batch of the reference-equivalent path (numpy items, Delaunay labels, collate)."""
    import torch
    from scipy.spatial import Delaunay
    from oracle import train_inputs as oti
    from oracle import train_inputs_sunrgbd as ots
    from frustum_convnet_b200.train_inputs import compute_box_3d

    def in_hull(pc, center, dimension, angle):                      # datasets/data_utils.py:24-34
        return Delaunay(compute_box_3d(center, dimension, angle)).find_simplex(pc) >= 0

    saved = oti.in_box
    oti.in_box = in_hull
    try:
        t0 = time.perf_counter()
        for index, draws in batches:
            out = ots.build(kind, L, index, draws, strides, max_depth)
            out.pop("_margins", None)
            {k: torch.from_numpy(v) for k, v in out.items()}
        return (time.perf_counter() - t0) * 1e3 / len(batches)
    finally:
        oti.in_box = saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frustums", type=int, default=8192)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--ref-batches", type=int, default=10)
    args = ap.parse_args()

    import torch
    from frustum_convnet_b200 import config, synth
    from frustum_convnet_b200.train_engine import TrainStep
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    assert torch.cuda.is_available(), "bench_train_inputs.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = args.batch
    line = {"frustums": args.frustums, "batch": B, "steps": args.steps}
    for kind, strides, N in (("det", CAR, 1024), ("refine", REFINE, 512), ("sunrgbd", SUN, 2048)):
        L = synthetic_sun_lists(args.frustums, seed=3) if kind == "sunrgbd" else synthetic_lists(kind, args.frustums,
                                                                                                 seed=3)
        tb = TrainBatchBuilder(kind, strides, N, max_depth=MAX_DEPTH[kind])
        tb.set_dataset(L["input_list"], L["type_list"], **{k: v for k, v in L.items()
                                                           if k not in ("input_list", "type_list")})
        rng = np.random.RandomState(0)
        order = np.concatenate([rng.permutation(args.frustums) for _ in range(1 + args.steps * B // args.frustums)])
        idx = [order[i * B: (i + 1) * B] for i in range(args.steps)]
        t0 = time.perf_counter()
        draws = [tb.draw(i, rng) for i in idx]
        draw_ms = (time.perf_counter() - t0) * 1e3 / args.steps

        def timed(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for i in range(args.steps):
                fn(i)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / args.steps

        timed(lambda i: tb.build(idx[i], draws[i]))                  # warm-up: module load, buffers
        build_ms = [timed(lambda i: tb.build(idx[i], draws[i])) for _ in range(args.regions)]
        tb.upload(idx[0], draws[0])
        launch_ms = [timed(lambda i: tb.launch()) for _ in range(args.regions)]
        ref_ms = reference_path_ms(kind, L, list(zip(idx, draws))[: args.ref_batches], strides, MAX_DEPTH[kind])
        res = {"build_ms_per_batch": float(np.median(build_ms)), "build_ms_min_max": [min(build_ms), max(build_ms)],
               "launch_ms_per_batch": float(np.median(launch_ms)), "draw_ms_per_batch": draw_ms,
               "reference_ms_per_batch": ref_ms, "reference_batches": args.ref_batches, "npoints": N}
        if kind in ("refine", "sunrgbd"):
            cfg, w = config.load_workload("refine_car" if kind == "refine" else "sunrgbd")
            if kind == "sunrgbd":
                from frustum_convnet_b200.det_base_sunrgbd import PointNetDet
            else:
                from frustum_convnet_b200.det_base import PointNetDet
            sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=7)
            m = PointNetDet(3, num_vec=w["num_vec"])
            m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
            ts = TrainStep(m.to(dev).train(), lr=1e-3, weight_decay=1e-4)
            fixed = {k: v.clone() for k, v in tb.build(idx[0], draws[0]).items()}
            shapes = {tuple(v.shape) for k, v in fixed.items() if k.startswith("center_ref")}

            def step(i, with_build):
                data = tb.build(idx[i], draws[i]) if with_build else fixed
                assert not with_build or {tuple(v.shape) for k, v in data.items() if k.startswith("center_ref")} == shapes
                ts.step(data)

            timed(lambda i: step(i, False))
            timed(lambda i: step(i, True))
            plain, built = [], []
            for _ in range(args.regions):
                plain.append(timed(lambda i: step(i, False)))
                built.append(timed(lambda i: step(i, True)))
            res.update({"train_ms_per_step": float(np.median(plain)),
                        "train_ms_per_step_with_build": float(np.median(built)),
                        "train_extra_ms_per_step": float(np.median(built) - np.median(plain)),
                        "train_plain_min_max": [min(plain), max(plain)], "train_built_min_max": [min(built), max(built)]})
        line[kind] = res
    line["measured_on"] = gpu_identity(dev)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
