#!/usr/bin/env python
"""Cost of one validation epoch: the reference validate() loop on the drop-in model against the device Validator.

    python scripts/bench_validate.py [--workloads car,people,sunrgbd,refine_car] [--batches 8] [--regions 5]

Per workload: `--batches` resident synthetic batches with labels (seeded weights, B=32, the last batch partial, 17
frustums; refine_car alternates two T pyramids, ref half-extents 0.977 and 1.5 m).  Regions alternate between
  (a) train/train_net_det.py validate() :171-189 on the drop-in model: model(data) in eval mode, the 14 .item()
      calls and AverageMeter/TrainingStates updates on the host;
  (b) Validator.add for each batch, then finalize().
Each region is one epoch, timed with a host clock around a synchronize; reported: median ms per epoch and per batch
of each loop and their ratio.  Prints one JSON line with the card name and its power limit.  Writes nothing to the
tree."""
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
from bench_detect import gpu_identity  # noqa: E402


class _Meter:                         # utils/utils.py:51-67 (host side of the reference loop)
    def __init__(self):
        self.sum, self.count = 0, 1e-14

    def update(self, val, n):
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def _batches(workload, n, B, last_B):
    import torch
    from frustum_convnet_b200 import synth
    out = []
    for i in range(n):
        b = last_B if i == n - 1 else B
        d = synth.make_frustums(workload, b, seed=900 + i, with_labels=True)
        if workload == "refine_car" and i % 2 == 1:          # a second T pyramid
            for s, st in enumerate(synth._PRESETS[workload]["strides"]):
                zc = np.arange(-1.5, 1.5, st) + st / 2.0
                c = np.zeros((b, 3, len(zc)), dtype=np.float64)
                c[:, 2, :] = zc[None, :]
                d["center_ref%d" % (s + 1)] = c.astype(np.float32)
            T2 = d["center_ref2"].shape[2]
            lab = np.random.default_rng(i).integers(-1, 2, (b, T2)).astype(np.int64)
            lab[:, T2 // 2] = 1
            d["cls_label"] = lab
        out.append({k: torch.from_numpy(v).cuda() for k, v in d.items()})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="car,people,sunrgbd,refine_car")
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--last", type=int, default=17)
    ap.add_argument("--regions", type=int, default=5)
    args = ap.parse_args()
    import torch
    from frustum_convnet_b200 import config, synth
    from frustum_convnet_b200.validate import Validator
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"metric": "validation epoch", **gpu_identity(dev), "batches_per_epoch": args.batches,
           "batch": args.batch, "last_batch": args.last, "workloads": {}}
    for wl in args.workloads.split(","):
        cfg, w = config.load_workload(wl)
        if w["arch"].num_scales == 5:
            from frustum_convnet_b200.det_base_sunrgbd import PointNetDet
        else:
            from frustum_convnet_b200.det_base import PointNetDet
        sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=5)
        m = PointNetDet(3, num_vec=w["num_vec"])
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
        m = m.cuda().eval()
        batches = _batches(wl, args.batches, args.batch, args.last)
        val = Validator(m)

        def loop_ref():
            meters = None
            for d in batches:
                with torch.no_grad():
                    losses, metrics = m(d)
                    vals = {k: v.detach().mean().item() for k, v in list(losses.items()) + list(metrics.items())}
                if meters is None:
                    meters = {k: _Meter() for k in vals}
                for k, v in vals.items():
                    meters[k].update(v, d["point_cloud"].shape[0])
            return {k: mt.avg for k, mt in meters.items()}

        def loop_dev():
            val.reset()
            for d in batches:
                val.add(d)
            return val.finalize()

        loop_ref()
        loop_dev()                                   # warm-up: plans, graphs, cuDNN autotune
        times = {"reference_loop": [], "validator": []}
        for _ in range(args.regions):
            for name, fn in (("reference_loop", loop_ref), ("validator", loop_dev)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t0) * 1e3)
        r = {}
        for name, ts in times.items():
            med = float(np.median(ts))
            r[name] = {"ms_per_epoch": round(med, 3), "ms_per_batch": round(med / len(batches), 4),
                       "ms_per_epoch_min_max": [round(min(ts), 3), round(max(ts), 3)]}
        r["speedup"] = round(r["reference_loop"]["ms_per_epoch"] / r["validator"]["ms_per_epoch"], 2)
        res["workloads"][wl] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
