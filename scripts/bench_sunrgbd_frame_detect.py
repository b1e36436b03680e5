"""Cloud-to-boxes latency of one call for the SUN-RGBD model: the offline chain (SunrgbdFrustumExtractor with the
host's np.random cap draw -> TrainBatchBuilder with numpy resampling -> the model -> DetectionCollector.finalize())
against a CUDA-graph replay of SunrgbdFrameDetector.detect followed by FrameDetections.to_dict().  Each call runs from
inputs resident on the device (the clouds as CUDA tensors, the detector's input buffers filled) to the kept rows on
the host.  The two paths alternate call by call after a warm-up; then each runs back to back for the steady-state
frames/s.  A separate profiled run of eager calls gives the device time of the frame path's stages: the count pass,
the cap draw (its resample_choice launch and the rank sort), the write pass and the forward (every kernel between the
batch build and the collector).

    python scripts/bench_sunrgbd_frame_detect.py --frames 1 8 --calls 100
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


def scenes(seed, F, n_dets):
    """F 530 x 730 frames (386 900 grid points plus object points) of sunrgbd_scene_synth.large_frame, n_dets
    detections each: the label boxes, jittered."""
    from oracle import sunrgbd_scene_synth as ss
    from frustum_convnet_b200 import sunrgbd_extract as sx
    rng = np.random.default_rng(seed)
    out = []
    for f in range(F):
        cloud, cal, lines = ss.large_frame(seed * 10 + f, 530, 730, n_dets)
        dets = [(o.classname, float(np.float32(rng.uniform(0.1, 1.0))), o.box2d + rng.uniform(-4, 4, 4))
                for o in (sx.SUNObject3d(ln) for ln in lines)]
        out.append((cloud, cal, dets))
    return out


def offline_call(model, sx, lists, clouds, calibs, strides, N, rng, method):
    from frustum_convnet_b200.detect import DetectionCollector
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    fr = sx.from_rgb_detections(clouds, calibs, *lists, rng=rng)
    if len(fr) == 0:
        return {}
    tb = TrainBatchBuilder.from_frustums(fr, "sunrgbd", strides, N, labels=False)
    idx = np.arange(len(fr))
    data = dict(tb.build(idx, tb.draw(idx, rng)))
    with torch.no_grad():
        out = model(data)
    col = DetectionCollector(fr.id_list, fr.type_list, fr.box2d_list, dataset="SUNRGBD", method=method)
    col.add(out, data, first=0)
    return col.finalize()


def stage_times(fd, inp, calls):
    """Median device ms per call of the count, cap, write and forward stages (torch.profiler, eager calls)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fd.detect(*inp)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    per = {k: [] for k in ("count", "cap", "write", "forward")}
    starts = [i for i, e in enumerate(ev) if "sf_setup_kernel" in e.name]
    for a, b in zip(starts, starts[1:] + [len(ev)]):
        call = ev[a:b]
        t = {k: 0.0 for k in per}
        seen_resample = False
        build = fwd_end = None
        for i, e in enumerate(call):
            us = e.time_range.end - e.time_range.start
            if "sf_points_kernel" in e.name:
                t["write" if "ILb1E" in e.name or "<true>" in e.name else "count"] += us
            elif "resample_choice_kernel" in e.name and not seen_resample:
                t["cap"] += us
                seen_resample = True
            elif "sf_sort_kernel" in e.name:
                t["cap"] += us
            elif "build_train_inputs_kernel" in e.name:
                build = i
            elif "det_candidates_kernel" in e.name and fwd_end is None:
                fwd_end = i
        if build is not None and fwd_end is not None:
            t["forward"] = sum(e.time_range.end - e.time_range.start for e in call[build + 1:fwd_end])
        for k in per:
            per[k].append(t[k] / 1e3)
    return {k + "_ms": float(np.median(v)) for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--dets", type=int, default=16)
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--method", default="top")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sunrgbd_frame_detect: needs a CUDA device")
    from train_ref import make_model
    from frustum_convnet_b200 import config
    from frustum_convnet_b200.frame_detect import SunrgbdFrameDetector
    from frustum_convnet_b200.sunrgbd_extract import SunrgbdFrustumExtractor
    cfg, _ = config.load_workload("sunrgbd")
    model = make_model("sunrgbd", 5).eval()
    name, power = card()
    for F in args.frames:
        frames = scenes(2000 + F, F, args.dets)
        P = max(len(x[0]) for x in frames)
        ids, types, boxes, probs = [], [], [], []
        for f, (_, _, dets) in enumerate(frames):
            for t, p, b in dets:
                ids.append(f), types.append(t), boxes.append(b), probs.append(p)
        clouds = {f: torch.from_numpy(x[0]).cuda() for f, x in enumerate(frames)}
        calibs = {f: x[1] for f, x in enumerate(frames)}
        sx = SunrgbdFrustumExtractor()
        fd = SunrgbdFrameDetector(model, method=args.method, frames=F, points=P, dets=args.dets, seed=1)
        inp = fd.inputs()
        fd.stage(inp, frames)
        fd.detect(*inp)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = fd.detect(*inp)
        rng = np.random.RandomState(0)

        def graph_call():
            g.replay()
            return out.to_dict()

        def off_call():
            return offline_call(model, sx, (ids, types, boxes, probs), clouds, calibs, cfg.DATA.STRIDE,
                                cfg.DATA.NUM_SAMPLES, rng, args.method)

        for _ in range(args.warmup):
            off_call(), graph_call()
        torch.cuda.synchronize()
        t_off, t_graph = [], []
        for _ in range(args.calls):
            for fn, acc in ((off_call, t_off), (graph_call, t_graph)):
                t0 = time.perf_counter()
                fn()
                acc.append(time.perf_counter() - t0)
        thr = {}
        for key, fn in (("offline", off_call), ("graph", graph_call)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.calls):
                fn()
            thr[key] = F * args.calls / (time.perf_counter() - t0)
        status = out.status_bits()
        kept = int(out.valid.sum().item())
        stages = stage_times(fd, inp, min(args.calls, 20))
        stats = lambda t: {"median_ms": 1e3 * float(np.median(t)), "p10_ms": 1e3 * float(np.percentile(t, 10)),
                           "p90_ms": 1e3 * float(np.percentile(t, 90))}
        print(json.dumps({"frames": F, "points": P, "dets": args.dets, "kept": kept, "calls": args.calls,
                          "method": args.method, "offline": stats(t_off), "graph": stats(t_graph),
                          "offline_frames_per_s": thr["offline"], "graph_frames_per_s": thr["graph"],
                          "graph_stages_device": stages, "status": status, "gpu": name, "power_limit": power}),
              flush=True)


if __name__ == "__main__":
    main()
