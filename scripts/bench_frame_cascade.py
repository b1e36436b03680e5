"""Scan-to-refined-boxes latency of one call of the KITTI car cascade (car, then refine_car, synthetic weights of
tests/train_ref.make_model): (a) a CUDA-graph replay of FrameDetector.detect, then the offline handoff
(FrameDetections.collected() -> RefineFrustumExtractor.from_collected -> TrainBatchBuilder.from_frustums -> numpy
resampling -> the refinement model -> DetectionCollector.finalize()) against (b) one CUDA-graph replay of
FrameDetector.detect and FrameRefiner.refine followed by FrameDetections.to_dict().  Each call runs from inputs
resident on the device to the refined rows on the host.  The two paths alternate call by call after a warm-up; then
each runs back to back for the steady-state frames/s.

Both paths must refine the same frustums, so the refiner's capacities are sized to the frames before anything is
timed: J and max_width from the most whitelisted first-stage rows of a frame and the widest enlarged box over
--probe first-stage calls (the first stage draws fresh resampling indices every call, so its rows vary), with a
margin.  --jobs / --max-width fix them instead.  The script refuses to report when any timed graph call dropped a
frustum for a capacity (status bits 4, 8, 32 or 64): the two paths would then not do the same work.

    python scripts/bench_frame_cascade.py --frames 1 8 --calls 200
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

from bench_frame_detect import card, scenes  # noqa: E402


CAPACITY_BITS = 4 | 8 | 32 | 64       # FCN_FRAME_OUT_POINTS, _ROWS, _JOBS, _SECTIONS: the graph path dropped work


def size_refiner(fd, inp, rx, frames_host, calls):
    """J and max_width for the frames in inp: the most Car rows of a frame and the widest enlarged box over `calls`
    first-stage calls, with half again as much of each as margin (a probe sees only some of the first stage's draws)."""
    scans, calibs, hws, ids = frames_host
    most, widest = 1, 0.1
    for _ in range(calls):
        first = fd.detect(*inp)
        most = max([most] + [len(per_class.get("Car", ())) for per_class in first.to_dict().values()])
        rf = rx.from_collected(scans, calibs, hws, ids, first.collected())
        if len(rf):
            widest = max(widest, float(rf.pred_box3d_size[:, 1].max()))
    return most + (most + 1) // 2, 1.5 * widest


def handoff_call(model2, rx, frames_host, first, rng):
    """The offline second stage from a first-stage graph replay's device rows."""
    from frustum_convnet_b200.detect import DetectionCollector
    from frustum_convnet_b200.refine_extract import REFINE_STRIDES
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    scans, calibs, hws, ids = frames_host
    rf = rx.from_collected(scans, calibs, hws, ids, first.collected())
    if len(rf) == 0:
        return {}
    tb = TrainBatchBuilder.from_frustums(rf, "refine", strides=REFINE_STRIDES, npoints=512)
    idx = np.arange(len(rf))
    data = dict(tb.build(idx, tb.draw(idx, rng)))
    with torch.no_grad():
        out = model2(data)
    col = DetectionCollector(rf.id_list, rf.type_list, rf.box2d_list)
    col.add(out, data, first=0)
    return col.finalize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--points", type=int, default=120000)
    ap.add_argument("--dets", type=int, default=8)
    ap.add_argument("--jobs", type=int, default=None, help="FrameRefiner jobs a frame (default: sized by the probe)")
    ap.add_argument("--max-width", type=float, default=None,
                    help="FrameRefiner max_width in metres (default: sized by the probe)")
    ap.add_argument("--probe", type=int, default=50, help="first-stage calls that size J and W")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_cascade: needs a CUDA device")
    from train_ref import make_model
    from frustum_convnet_b200.frame_detect import FrameDetector, FrameRefiner
    from frustum_convnet_b200.refine_extract import RefineFrustumExtractor
    model1, model2 = make_model("car", 5).eval(), make_model("refine_car", 5).eval()
    name, power = card()
    for F in args.frames:
        frames = scenes(1000 + F, F, args.points, args.dets)
        frames_host = ({f: torch.from_numpy(x[0]).cuda() for f, x in enumerate(frames)},
                       {f: x[1] for f, x in enumerate(frames)}, {f: x[2] for f, x in enumerate(frames)},
                       list(range(F)))
        rx = RefineFrustumExtractor(("Car",))
        fd = FrameDetector(model1, ("Car",), frames=F, points=args.points, dets=args.dets, seed=1)
        inp = fd.inputs()
        fd.stage(inp, frames)
        J, width = size_refiner(fd, inp, rx, frames_host, args.probe)
        J = args.jobs if args.jobs is not None else J
        width = args.max_width if args.max_width is not None else width
        fr = FrameRefiner(fd, model2, ("Car",), jobs=J, max_width=width, seed=2)
        fr.refine(inp, fd.detect(*inp))
        torch.cuda.synchronize()
        g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        with torch.cuda.graph(g1):
            first = fd.detect(*inp)
        with torch.cuda.graph(g2):
            out = fr.refine(inp, fd.detect(*inp))
        rng = np.random.RandomState(0)

        def graph_call():
            g2.replay()
            return out.to_dict()

        def handoff():
            g1.replay()
            return handoff_call(model2, rx, frames_host, first, rng)

        for _ in range(args.warmup):
            handoff(), graph_call()
        torch.cuda.synchronize()
        t_off, t_graph, overflow = [], [], 0
        for _ in range(args.calls):
            for fn, acc in ((handoff, t_off), (graph_call, t_graph)):
                t0 = time.perf_counter()
                fn()
                acc.append(time.perf_counter() - t0)
                if fn is graph_call:
                    overflow |= out.status_bits() & CAPACITY_BITS       # read after the timing
        thr = {}
        for key, fn in (("handoff", handoff), ("graph", graph_call)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.calls):
                fn()
            thr[key] = F * args.calls / (time.perf_counter() - t0)
        status = out.status_bits()
        if (overflow | status) & CAPACITY_BITS:
            raise SystemExit("bench_frame_cascade: F = %d: a graph call dropped frustums for a capacity (status bits "
                             "%d, J = %d, W = %s); the two paths did not do the same work, nothing is reported"
                             % (F, (overflow | status) & CAPACITY_BITS, fr.J, fr.T))
        stats = lambda t: {"median_ms": 1e3 * float(np.median(t)), "p10_ms": 1e3 * float(np.percentile(t, 10)),
                           "p90_ms": 1e3 * float(np.percentile(t, 90))}
        print(json.dumps({"frames": F, "points": args.points, "dets": args.dets, "jobs": fr.J, "max_width": round(width, 3), "batch": fr.B,
                          "sections": fr.T, "calls": args.calls, "handoff": stats(t_off), "graph": stats(t_graph),
                          "handoff_frames_per_s": thr["handoff"], "graph_frames_per_s": thr["graph"],
                          "status": status, "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
