"""Phase timeline of the persistent FCN kernel (csrc/fcn_mega.cu) for one B = 32 forward in isolation.

Runs one forward of each workload to fill the feature maps, then launches fcn_mega with `dbg_clocks` set (every
CTA records 32 clocks per job for its first 64 jobs) and splits each consumer warpgroup's time per job into
  full_wait   clocks waiting for operand stages (`full` barriers), the first stage of the job included,
  mma         the rest of the K loop up to the last retired MMA (MMA issue and execution),
  epilogue    last MMA retired -> tile staged for the store warp (heads: rows decoded and counter published),
and the store warp's time per tile:
  store_issue first staged half received -> last box store issued (the rest of the staging included),
  publish     last box store issued -> stores complete and the counter published,
  store_lag   both warpgroups staged the tile -> counter published,
and reports per layer the scheduler's dependency wait (fetched -> dependencies met), the TMA lane's wait for the
next job descriptor (last box of the previous job -> job taken) and its `empty` waits.  All values are SM clocks,
averaged over the recorded jobs of the layer (a CTA's first job is skipped: it has no previous epilogue).

    python scripts/fcn_mega_timeline.py --out DIR [--workloads car people sunrgbd] [--reps 5]
writes DIR/fcn_mega_timeline.json.  Needs a CUDA device.
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ROWS_PER_JOB = 64           # recorded jobs per CTA (MG_DBG_JOBS)
ROW = 32                    # clocks per recorded job (MG_DBG_ROW)


def timeline(workload, B, reps):
    import torch
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload(workload)
    modname = "det_base_sunrgbd" if w["arch"].num_scales == 5 else "det_base"
    mod = __import__("frustum_convnet_b200." + modname, fromlist=["PointNetDet"])
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=7)
    model = mod.PointNetDet(3, num_vec=w["num_vec"])
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    model = model.cuda().eval()
    model.use_cuda_graph = False
    data = synth.make_frustums(workload, B, seed=1234)
    S = w["arch"].num_scales
    model({k: torch.from_numpy(v).cuda() for k, v in data.items()})
    torch.cuda.synchronize()
    plan = model.engine().plan(B, data["point_cloud"].shape[2],
                               [data["center_ref%d" % (i + 1)].shape[2] for i in range(S)])
    m = plan.mega_args
    assert m is not None, "the persistent FCN kernel is not selected for this workload"
    descs = plan.mega_descs()
    grid = plan.mega_grid
    buf = torch.zeros(grid * ROWS_PER_JOB * ROW, dtype=torch.int64, device="cuda")
    m.dbg_clocks = buf.data_ptr()
    try:
        for _ in range(reps):                      # the last launch is the one read back
            buf.zero_()
            plan._launch_mega(plan.in_centers[1])
        torch.cuda.synchronize()
    finally:
        m.dbg_clocks = None
    rows = buf.cpu().numpy().reshape(grid, ROWS_PER_JOB, ROW)

    per = {}
    for c in range(grid):
        for q in range(1, ROWS_PER_JOB):
            r, pr = rows[c, q], rows[c, q - 1]
            if r[0] == 0 or pr[0] == 0:
                continue
            d = per.setdefault(int(r[14]), dict(jobs=0, full_wait=0.0, mma=0.0, epilogue=0.0, dep_wait=0.0,
                                                desc_wait=0.0, tma_empty_wait=0.0, job=0.0, stored=0,
                                                store_issue=0.0, publish=0.0, store_lag=0.0))
            d["jobs"] += 1
            for wg in range(2):
                o = 6 + 4 * wg
                first, t_full, last_mma, epi = r[o:o + 4]
                prev_epi = pr[o + 3]
                d["full_wait"] += t_full / 2
                d["mma"] += (last_mma - prev_epi - t_full) / 2
                d["epilogue"] += (epi - last_mma) / 2
                d["job"] += (epi - prev_epi) / 2
            d["dep_wait"] += r[3] - r[2]
            d["desc_wait"] += max(0, r[0] - pr[4])
            d["tma_empty_wait"] += r[5]
            if r[22] != 0:                           # store warp (tiles of non-heads layers)
                d["stored"] += 1
                d["store_issue"] += r[21] - r[20]
                d["publish"] += r[22] - r[21]
                d["store_lag"] += r[22] - max(r[9], r[13])
    layers = []
    for li in sorted(per):
        d = per[li]
        n = d.pop("jobs")
        ns = max(1, d.pop("stored"))
        for k in ("store_issue", "publish", "store_lag"):
            d[k] *= n / ns                           # averaged over the stored tiles below
        L = descs[li]
        stages = L.K_pad // 32
        out = {k: round(v / n) for k, v in d.items()}
        out.update(layer=L.name, NT=L.NT, k_stages=stages, jobs_recorded=n,
                   mma_clocks_per_stage=round(d["mma"] / n / stages))
        layers.append(out)
    tot = {k: sum(l[k] * l["jobs_recorded"] for l in layers)
           for k in ("full_wait", "mma", "epilogue", "dep_wait", "desc_wait", "tma_empty_wait", "job")}
    return dict(workload=workload, B=B, grid=grid, jobs=plan.mega_jobs, layers=layers,
                share_of_consumer_time={k: round(tot[k] / tot["job"], 3) for k in ("full_wait", "mma", "epilogue")})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--workloads", nargs="+", default=["car", "people", "sunrgbd"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "the timeline is recorded on the GPU"
    res = dict(gpu=torch.cuda.get_device_name(), runs=[timeline(w, args.batch, args.reps) for w in args.workloads])
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "fcn_mega_timeline.json"), "w") as f:
        json.dump(res, f, indent=1)
    for r in res["runs"]:
        print(r["workload"], "grid", r["grid"], r["share_of_consumer_time"])
        for l in r["layers"]:
            print("  %-16s NT %3d stages %3d jobs %3d | mma/stage %5d full_wait %6d mma %6d epi %5d dep %6d desc %6d"
                  " | store issue %5d publish %5d lag %5d"
                  % (l["layer"], l["NT"], l["k_stages"], l["jobs_recorded"], l["mma_clocks_per_stage"], l["full_wait"],
                     l["mma"], l["epilogue"], l["dep_wait"], l["desc_wait"], l["store_issue"], l["publish"],
                     l["store_lag"]))


if __name__ == "__main__":
    main()
