"""Wall time of scoring a whole synthetic split through the single-frame path, three ways:
  (a) store:   a CUDA graph of detect + FrameStore.append per call, then one store.collected() and evaluate_collected;
  (b) to_dict: a CUDA graph of detect per call followed by out.to_dict() merged on the host, then evaluate(dict);
  (c) offline: the offline chain per call (extractor, numpy resampling, the model, DetectionCollector.finalize()),
               merged on the host, then evaluate(dict).
Every call stages its frames from host arrays.  Configurations: the KITTI car FrameDetector at F = 1 and 8 with
KittiEvaluator, and SunrgbdFrameDetector at F = 8 with SunrgbdEvaluator.  The split cycles through a pool of distinct
synthetic frames under fresh image ids.  The three ways alternate split by split after a warm-up (median, p10, p90 of
the split times); a separate profiled run of (a) gives the append kernels' device time per call.

    python scripts/bench_frame_split.py --split 512 --reps 5
prints one JSON line per configuration, with the card's name and power limit."""
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

import bench_frame_detect as kitti_bench  # noqa: E402
import bench_sunrgbd_frame_detect as sun_bench  # noqa: E402


def chunks(split, F, pool):
    """[(frames, ids)] of F frames a call: frame i of the split is pool[i % len(pool)] under id i."""
    return [([pool[i % len(pool)] for i in range(s, min(s + F, split))], list(range(s, min(s + F, split))))
            for s in range(0, split, F)]


def kitti_offline(model, cfg):
    from frustum_convnet_b200.frustum_extract import FrustumExtractor
    fe = FrustumExtractor(("Car",))
    fb_args = (cfg.DATA.STRIDE, cfg.DATA.MAX_DEPTH, cfg.DATA.NUM_SAMPLES)
    rng = np.random.RandomState(0)

    def run(frames, ids):
        lists = ([], [], [], [])
        for i, (_, _, _, dets) in zip(ids, frames):
            for t, p, b in dets:
                for dst, v in zip(lists, (i, t, p, b)):
                    dst.append(v)
        return kitti_bench.offline_call(model, fe, fb_args, ({i: x[0] for i, x in zip(ids, frames)},
                                                             {i: x[1] for i, x in zip(ids, frames)},
                                                             {i: x[2] for i, x in zip(ids, frames)}) + lists,
                                        rng, "nms")
    return run


def sun_offline(model, cfg, method):
    from frustum_convnet_b200.sunrgbd_extract import SunrgbdFrustumExtractor
    sx = SunrgbdFrustumExtractor()
    rng = np.random.RandomState(0)

    def run(frames, ids):
        lists = ([], [], [], [])
        for i, (_, _, dets) in zip(ids, frames):
            for t, p, b in dets:
                for dst, v in zip(lists, (i, t, b, p)):
                    dst.append(v)
        return sun_bench.offline_call(model, sx, lists, {i: torch.from_numpy(x[0]).cuda() for i, x in zip(ids, frames)},
                                      {i: x[1] for i, x in zip(ids, frames)}, cfg.DATA.STRIDE, cfg.DATA.NUM_SAMPLES,
                                      rng, method)
    return run


def same_tree(x, y):
    if isinstance(x, dict):
        return x.keys() == y.keys() and all(same_tree(x[k], y[k]) for k in x)
    return bool(np.array_equal(np.asarray(x), np.asarray(y)))


def append_device_ms(fd, store, inp, calls):
    """Median device ms per call of the two append kernels (torch.profiler, eager appends)."""
    from torch.profiler import ProfilerActivity, profile
    out = fd.detect(*inp)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            store.reset()
            store.append(out)
        torch.cuda.synchronize()
    store.reset()
    per = {"plan": [], "copy": []}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for k in per:
            if "fs_%s_kernel" % k in e.name:
                per[k].append((e.time_range.end - e.time_range.start) / 1e3)
    return {k + "_ms": float(np.median(v)) for k, v in per.items()}


def run_config(label, fd, make_ev, offline, split, reps, pool):
    from frustum_convnet_b200.frame_detect import FrameStore
    F = fd.F
    calls = chunks(split, F, pool)
    inp = fd.inputs()
    store = FrameStore(fd, rows=fd.R * len(calls), segments=len(fd.classes) * split)
    fd.stage(inp, calls[0][0])
    store.append(fd.detect(*inp))
    torch.cuda.synchronize()
    g_store, g_plain = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g_store):
        out = fd.detect(*inp)
        store.append(out)
    with torch.cuda.graph(g_plain):
        out_plain = fd.detect(*inp)

    def replay_plain(frames, ids, merged):
        fd.stage(inp, frames)
        g_plain.replay()
        merged.update({i: v for i, v in out_plain.to_dict(ids + [-1] * (F - len(ids))).items() if i >= 0})

    def way_store():
        store.reset()
        for frames, ids in calls:
            fd.stage(inp, frames)
            store.stage_ids(ids)
            g_store.replay()
        return ev.evaluate_collected(store.collected())

    def way_dict():
        merged = {}
        for frames, ids in calls:
            replay_plain(frames, ids, merged)
        return ev.evaluate(merged)

    def way_offline():
        merged = {}
        for frames, ids in calls:
            merged.update(offline(frames, ids))
        return ev.evaluate(merged)

    # the draws are keyed on the stage's call counters: rewound, both graph ways draw alike and must agree bit for bit
    counters = [t for t in (getattr(fd, "call", None), getattr(fd, "cap_call", None)) if t is not None]
    saved = [t.clone() for t in counters]

    def rewind():
        for t, v in zip(counters, saved):
            t.copy_(v)

    merged = {}
    for frames, ids in calls:
        replay_plain(frames, ids, merged)
    ev = make_ev(merged)
    rewind()
    a = way_store()
    rewind()
    b = way_dict()
    got = store.to_dict()
    same = got.keys() == merged.keys() and all(
        list(got[i]) == list(merged[i]) and np.array_equal(got[i][c].view(np.int32), merged[i][c].view(np.int32))
        for i in merged for c in merged[i])
    status = store.status_bits()
    way_offline()
    torch.cuda.synchronize()
    times = {"store": [], "to_dict": [], "offline": []}
    for _ in range(reps):
        for key, fn in (("store", way_store), ("to_dict", way_dict), ("offline", way_offline)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[key].append(time.perf_counter() - t0)
    stats = lambda t: {"median_s": float(np.median(t)), "p10_s": float(np.percentile(t, 10)),
                       "p90_s": float(np.percentile(t, 90)), "frames_per_s": split / float(np.median(t))}
    res = {"config": label, "frames_per_call": F, "split": split, "calls": len(calls), "reps": reps,
           "store_equals_merged_dict": bool(same), "ap_store_equals_dict": same_tree(a.ap, b.ap), "status": status}
    res.update({k: stats(v) for k, v in times.items()})
    res["append_device"] = append_device_ms(fd, store, inp, 50)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--split", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pool", type=int, default=8, help="distinct synthetic frames the split cycles through")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frame_split: needs a CUDA device")
    from det_feed_sets import kitti_set
    from test_gpu_det_eval_feed import kitti_gt
    from train_ref import make_model
    from frustum_convnet_b200 import config
    from frustum_convnet_b200.frame_detect import FrameDetector, SunrgbdFrameDetector
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator, SunrgbdGroundTruth, det_corners
    name, power = kitti_bench.card()

    gts, _ = kitti_set(args.split, seed=5)
    kitti_ev = kitti_gt(list(range(args.split)), gts)
    cfg, _ = config.load_workload("car")
    model = make_model("car", 5).eval()
    pool = kitti_bench.scenes(4000, args.pool, 120000, 8)
    for F in (1, 8):
        fd = FrameDetector(model, ("Car",), frames=F, points=120000, dets=8, seed=1)
        res = run_config("kitti_car", fd, lambda merged: kitti_ev, kitti_offline(model, cfg), args.split,
                         args.reps, pool)
        res.update(gpu=name, power_limit=power)
        print(json.dumps(res), flush=True)

    cfg, _ = config.load_workload("sunrgbd")
    model = make_model("sunrgbd", 5).eval()
    pool = sun_bench.scenes(5000, args.pool, 16)
    P = max(len(x[0]) for x in pool)

    def sun_ev(merged):
        """Ground truth from the frame path's own rows, every other one moved a little, so classes match and miss."""
        rng = np.random.default_rng(0)
        gt = {}
        for i, by_class in merged.items():
            for c, rows in by_class.items():
                r = rows[::2]
                corners, ids = gt.setdefault(c, ([], []))
                corners.append(det_corners(r) + rng.uniform(-0.05, 0.05, (len(r), 1, 3)))
                ids += [i] * len(r)
        return SunrgbdEvaluator(SunrgbdGroundTruth({c: (np.concatenate(v[0]), np.array(v[1]))
                                                    for c, v in gt.items()}))
    fd = SunrgbdFrameDetector(model, method="top", frames=8, points=P, dets=16, seed=1)
    res = run_config("sunrgbd", fd, sun_ev, sun_offline(model, cfg, "top"), args.split, args.reps, pool)
    res.update(gpu=name, power_limit=power)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
