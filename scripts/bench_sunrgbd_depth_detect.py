"""Host-to-rows latency of one SunrgbdFrameDetector call from staged clouds against one from depth images: stage()
of (F, P, 6) float32 clouds then a graph replay of detect(), against stage_depth() of uint16 depth and uint8 RGB
images then a graph replay of detect_depth() (the conversion, C ABI section (24), inside the graph).  Each call ends
with a device sync.  The two alternate call by call after a warm-up.  A profiled run of eager detect_depth calls gives
the conversion kernels' device time per call.

    python scripts/bench_sunrgbd_depth_detect.py --frames 1 8 --calls 40
prints one JSON line per frame count, with the card's name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_frame_detect import card  # noqa: E402

H, W = 530, 730
CLASSES = ("bed", "table", "sofa", "chair", "toilet", "desk", "dresser", "night_stand", "bookshelf", "bathtub")


def scene(seed, n_dets):
    """A 530 x 730 depth frame (a ramp from 6 m to 2 m with n_dets boxes in front, 10 % of pixels 0), its RGB image,
    calibration and one detection per box."""
    from oracle.make_golden_sunrgbd_depth import calibs, rot_left3
    rng = np.random.default_rng(seed)
    v, u = np.mgrid[0:H, 0:W]
    d = 2.0 + 4.0 * (1 - v / H) + 0.5 * np.sin(u / 37.0)
    dets = []
    for j in range(n_dets):
        h, w = rng.integers(40, 140, 2)
        y0, x0 = rng.integers(0, H - h), rng.integers(0, W - w)
        d[y0:y0 + h, x0:x0 + w] = rng.uniform(1.0, 3.0)
        dets.append((CLASSES[j % len(CLASSES)], float(np.float32(rng.uniform(0.1, 1.0))),
                     np.array([x0, y0, x0 + w, y0 + h], np.float64)))
    raw = rot_left3(np.clip(np.round(d * 1000), 1, 65535).astype(np.int64))
    raw[rng.random((H, W)) < 0.1] = 0
    rgb = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    R, K = calibs()[seed % 2]
    return raw, rgb, {"Rtilt": R, "K": K}, dets


def conversion_ms(fd, inp, calls):
    """Median device ms per call of the conversion kernels (sd_*), from eager detect_depth calls."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fd.detect_depth(*inp)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    per, cur = [], None
    for e in ev:
        if "sd_count_kernel" in e.name:
            cur = 0.0
            per.append(cur)
        if cur is not None and "sd_" in e.name and "_kernel" in e.name:
            per[-1] += (e.time_range.end - e.time_range.start) / 1e3
    return float(np.median(per)) if per else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--dets", type=int, default=16)
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sunrgbd_depth_detect: needs a CUDA device")
    from train_ref import make_model
    from frustum_convnet_b200 import config
    from frustum_convnet_b200.frame_detect import SunrgbdFrameDetector
    from frustum_convnet_b200.sunrgbd_depth import depth_clouds
    config.load_workload("sunrgbd")
    model = make_model("sunrgbd", 5).eval()
    name, power = card()
    P = H * W
    for F in args.frames:
        frames = [scene(3000 + 10 * F + f, args.dets) for f in range(F)]
        clouds = depth_clouds([f[0] for f in frames], [f[1] for f in frames], [f[2] for f in frames], list(range(F)))
        cloud_frames = [(clouds[f].cpu().numpy(), fr[2], fr[3]) for f, fr in enumerate(frames)]
        fc = SunrgbdFrameDetector(model, frames=F, points=P, dets=args.dets, seed=1)
        fdd = SunrgbdFrameDetector(model, frames=F, points=P, dets=args.dets, seed=1)
        cin, din = fc.inputs(), fdd.inputs_depth(H, W)
        fc.stage(cin, cloud_frames)
        fdd.stage_depth(din, frames)
        fc.detect(*cin)
        fdd.detect_depth(*din)
        torch.cuda.synchronize()
        gc, gd = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(gc):
            oc = fc.detect(*cin)
        with torch.cuda.graph(gd):
            od = fdd.detect_depth(*din)

        def cloud_call():
            fc.stage(cin, cloud_frames)
            gc.replay()
            torch.cuda.synchronize()

        def depth_call():
            fdd.stage_depth(din, frames)
            gd.replay()
            torch.cuda.synchronize()

        for _ in range(args.warmup):
            cloud_call(), depth_call()
        t_c, t_d = [], []
        for _ in range(args.calls):
            for fn, acc in ((cloud_call, t_c), (depth_call, t_d)):
                t0 = time.perf_counter()
                fn()
                acc.append(time.perf_counter() - t0)
        same = bool(torch.equal(oc.seg_offsets, od.seg_offsets) and torch.equal(oc.keep_count, od.keep_count))
        stats = lambda t: {"median_ms": 1e3 * float(np.median(t)), "p10_ms": 1e3 * float(np.percentile(t, 10)),
                           "p90_ms": 1e3 * float(np.percentile(t, 90))}
        print(json.dumps({
            "frames": F, "height": H, "width": W, "points": P, "dets": args.dets, "calls": args.calls,
            "valid_points": [int(len(c)) for c, _, _ in cloud_frames],
            "staged_cloud": dict(stats(t_c), bytes_per_frame=P * 24 + 4),
            "staged_depth": dict(stats(t_d), bytes_per_frame=H * W * (2 + 3) + 8),
            "conversion_device_ms": conversion_ms(fdd, din, min(args.calls, 20)),
            "same_rows": same, "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
