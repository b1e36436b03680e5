#!/usr/bin/env python
"""Device time of one optimizer step over the flat parameter bucket: the fused SGD (`fcn_sgd_step`, momentum 0.9 and
0), the fused Adam (`fcn_adam_step`) and `torch.optim.SGD.step()` (default foreach path, momentum 0.9) over the same
parameters, for the KITTI model (3,316,777 parameters in 79 tensors) and the SUN-RGBD model (6,667,589 in 100).

    python scripts/bench_optimizer_step.py [--launches 200] [--regions 5] [--warmup 50]

Each variant runs `--warmup` steps, then `--regions` regions of `--launches` back-to-back steps between two CUDA
events; the median region gives ms per step.  torch's step is timed the same way, so its time includes the host
issuing its kernels whenever the host is the slower side.  Bytes per step are the arrays each fused kernel reads and
writes per parameter: 20 B for SGD with momentum (parameter, gradient and buffer read, parameter and buffer
written), 12 B without, 28 B for Adam; torch's rate is given for the same 20 B, the least its step must move.
Each variant also reports its working set (the distinct arrays it touches) and whether that fits the H100's 50 MB
L2: on the KITTI bucket the SGD arrays do (3 or 2 x 13.3 MB), so those rates are L2-assisted, and Adam's four (53 MB)
exceed it only slightly; no KITTI rate is stated as a share of HBM bandwidth.  Every SUN-RGBD working set is at
least 53 MB (26.7 MB per array), and those rates are also given as a share of the data sheet's 3.35 TB/s.  Prints
one JSON line with the card name and power limit.  Writes nothing to the tree."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_detect import gpu_identity  # noqa: E402

HBM_PEAK = 3.35e12                    # H100 SXM data sheet, bytes/s
BYTES_PER_PARAM = {"sgd_momentum": 20, "sgd_no_momentum": 12, "adam": 28, "torch_sgd_momentum": 20}
ARRAYS = {"sgd_momentum": 3, "sgd_no_momentum": 2, "adam": 4, "torch_sgd_momentum": 3}     # distinct fp32 arrays
L2_BYTES = 50 * 2 ** 20               # H100 L2
BUCKETS = (("kitti", "car", False), ("sunrgbd", "sunrgbd", True))      # (name, workload, rate vs HBM peak)
LR, MOMENTUM, WD = 1e-3, 0.9, 1e-4


def _model(workload):
    import torch
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload(workload)
    if w["arch"].num_scales == 5:
        from frustum_convnet_b200.det_base_sunrgbd import PointNetDet
    else:
        from frustum_convnet_b200.det_base import PointNetDet
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=7)
    m = PointNetDet(3, num_vec=w["num_vec"])
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()

    import torch
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200.train_engine import FlatParams
    assert torch.cuda.is_available(), "bench_optimizer_step.py needs a CUDA device; there is no CPU fallback"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _lib.load()
    line = {"launches_per_region": args.launches, "regions": args.regions, "lr": LR, "momentum": MOMENTUM,
            "weight_decay": WD}
    for name, workload, vs_hbm in BUCKETS:
        m = _model(workload)
        params = list(m.parameters())
        n, tensors = sum(p.numel() for p in params), len(params)          # counted on the host
        m = m.to(dev)
        flat = FlatParams(m)
        assert flat.numel == n
        g = torch.Generator(device=dev).manual_seed(1)
        flat.grad.copy_(torch.randn(n, generator=g, device=dev) * 1e-3)
        flat.expose_grads(m)
        buf, ea, eas = (torch.zeros_like(flat.param) for _ in range(3))
        P, G, Bf, M, V = (t.data_ptr() for t in (flat.param, flat.grad, buf, ea, eas))
        stream = torch.cuda.current_stream().cuda_stream
        tsgd = torch.optim.SGD(m.parameters(), lr=LR, momentum=MOMENTUM, weight_decay=WD)

        def sgd_momentum():
            _lib.check(lib.fcn_sgd_step(P, G, Bf, n, LR, MOMENTUM, WD, 0, 1.0, stream), "fcn_sgd_step")

        def sgd_no_momentum():
            _lib.check(lib.fcn_sgd_step(P, G, None, n, LR, 0.0, WD, 0, 1.0, stream), "fcn_sgd_step")

        def adam():
            _lib.check(lib.fcn_adam_step(P, G, M, V, n, LR, 0.9, 0.999, 1e-8, WD, 10, 1.0, stream), "fcn_adam_step")

        variants = {"sgd_momentum": sgd_momentum, "sgd_no_momentum": sgd_no_momentum, "adam": adam,
                    "torch_sgd_momentum": tsgd.step}
        res = {"params": n, "tensors": tensors}
        for key, fn in variants.items():
            for _ in range(args.warmup):
                fn()
            times = []
            for _ in range(args.regions):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.launches):
                    fn()
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1) / args.launches)
            ms = float(np.median(times))
            nbytes = BYTES_PER_PARAM[key] * n
            ws = ARRAYS[key] * 4 * n
            r = {"ms": ms, "ms_min_max": [min(times), max(times)], "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6,
                 "working_set_bytes": ws, "fits_l2": ws <= L2_BYTES}
            if vs_hbm:
                r["share_of_hbm_peak"] = nbytes / (ms * 1e-3) / HBM_PEAK
            res[key] = r
        line[name] = res
        del tsgd, flat, m, buf, ea, eas
        torch.cuda.empty_cache()
    line["measured_on"] = gpu_identity(dev)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
