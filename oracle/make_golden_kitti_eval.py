"""Writes tests/golden/kitti_eval.npz: seeded synthetic label and result files (oracle/kitti_synth.py) and what the
reference's own prebuilt evaluator, train/kitti_eval/evaluate_object_3d_offline, makes of them - every stats_*.txt
vector and the printed AP lines.  Needs the reference tree (oracle/ref_import.REF); the tests read only the fixture.

    python -m oracle.make_golden_kitti_eval               # the fixture
    python -m oracle.make_golden_kitti_eval --time-bench  # the evaluator's wall time on scripts/bench_kitti_eval.py's set

Runs (prefix in the file):
  main   160 images, every class detected; image 5 has no ground truth, image 6 no detections (an empty file);
  noaos  60 images without any Cyclist detection (the class is not evaluated) and one alpha of -10 (no AOS);
  full   60 images where every object also has an exact duplicate detection: the recall of the classes reaches 1,
         so evaluations get all 41 recall-step thresholds (asserted: the high-recall end of getThresholds, its last,
         always-taken score and the last point of the printed AP are pinned).
Every image is drawn again until no overlap lies within 1e-9 of 0.5 or 0.7 and the competing overlaps of each
ground truth are identical or 1e-9 apart, decided in exact arithmetic near each decision (kitti_synth.margins_ok), so
no decision depends on the last bits in which Boost.Geometry's areas and a float64 clip differ.
"""
from __future__ import annotations

import argparse
import glob
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import kitti_eval as ok  # noqa: E402
from oracle import kitti_synth as ks  # noqa: E402
from oracle.ref_import import REF  # noqa: E402

EVALUATOR = os.path.join(REF, "train", "kitti_eval", "evaluate_object_3d_offline")
OUT = os.path.join(ROOT, "tests", "golden", "kitti_eval.npz")


def write_set(tmp, ids, labels, results):
    gt_dir, res_dir = os.path.join(tmp, "label_2"), os.path.join(tmp, "result")
    os.makedirs(gt_dir)
    os.makedirs(os.path.join(res_dir, "data"))
    for i, lab, det in zip(ids, labels, results):
        with open(os.path.join(gt_dir, "%06d.txt" % i), "w") as f:
            f.write("".join(ln + "\n" for ln in lab))
        with open(os.path.join(res_dir, "data", "%06d.txt" % i), "w") as f:
            f.write("".join(ln + "\n" for ln in det))
    return gt_dir, res_dir


def run_evaluator(gt_dir, res_dir):
    """-> (stdout AP lines, {stats file name: (rows, 41)}, wall seconds)."""
    t0 = time.perf_counter()
    p = subprocess.run([EVALUATOR, gt_dir, res_dir], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
                       check=True)
    dt = time.perf_counter() - t0
    lines = [ln.strip() for ln in p.stdout.splitlines() if " AP: " in ln]
    stats = {}
    for path in sorted(glob.glob(os.path.join(res_dir, "stats_*.txt"))):
        rows = [[float(v) for v in ln.split()] for ln in open(path) if ln.strip()]
        stats[os.path.basename(path)[:-4]] = np.asarray(rows, dtype=np.float64)
    return lines, stats, dt


def make_run(name, seed, n, out, **kw):
    labels, results = ks.make_set(seed, n, check_margins=True, **kw)
    if name == "main":
        labels[5], results[6] = [], []
    elif name == "noaos":
        results = [[ln for ln in r if not ln.startswith("Cyclist")] for r in results]
        k = next(i for i, r in enumerate(results) if r)
        t = results[k][0].split(" ")
        t[3] = "-10.0000"
        results[k][0] = " ".join(t)
    ids = np.arange(n, dtype=np.int64) * 3 + 7          # sparse ids, as in a split file
    with tempfile.TemporaryDirectory() as tmp:
        gt_dir, res_dir = write_set(tmp, ids, labels, results)
        lines, stats, _ = run_evaluator(gt_dir, res_dir)
    assert lines, "the evaluator printed no AP line"
    gts = [ks.parse_label_lines(l) for l in labels]
    dets = [ks.parse_result_lines(r) for r in results]
    ref = ok.evaluate(gts, dets)
    assert ref["lines"] == lines, "the oracle disagrees with the evaluator"
    n_thr = max(int(v.max()) for m in ref["n_thresholds"].values() for v in m.values())
    n_dup = sum(1 for g, d in zip(gts, dets) for row in g for r in d
                if all(row[c] == r[c - 2] for c in range(4, 15)))   # x1 .. ry: gt columns 4-14, det 2-12
    print(name, "most thresholds of an evaluation:", n_thr, "| detections identical to a ground truth:", n_dup)
    if name == "full":
        assert n_thr == 41, n_thr
    assert n_dup > 0
    out[name + "_ids"] = ids
    out[name + "_labels"] = np.array(["\n".join(l) for l in labels])
    out[name + "_results"] = np.array(["\n".join(r) for r in results])
    out[name + "_lines"] = np.array(lines)
    out[name + "_stats_names"] = np.array(sorted(stats))
    out[name + "_stats"] = np.stack([stats[k] for k in sorted(stats)])
    print(name, len(ids), "images,", sum(len(l) for l in labels), "GT lines,", sum(len(r) for r in results),
          "detections")
    print("\n".join(lines))


def time_bench():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import bench_kitti_eval as bk
    labels, results = bk.make_bench_set()
    ids = np.arange(len(labels))
    print("%d images, %d GT lines, %d detections" % (len(ids), sum(map(len, labels)), sum(map(len, results))),
          flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        gt_dir, res_dir = write_set(tmp, ids, labels, results)
        lines, _, dt = run_evaluator(gt_dir, res_dir)        # one run: it takes minutes
    print("\n".join(lines))
    print("evaluator wall time: %.1f s" % dt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--time-bench", action="store_true")
    args = ap.parse_args()
    if not os.path.exists(EVALUATOR):
        raise SystemExit("the reference evaluator is missing: %s" % EVALUATOR)
    if args.time_bench:
        time_bench()
        return
    out = {}
    make_run("main", 11, 160, out)
    make_run("noaos", 12, 60, out)
    make_run("full", 13, 60, out, dup_all=True)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
