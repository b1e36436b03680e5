"""Writes tests/golden/refine_extract.npz: what the reference's own, unmodified extract_frustum_data,
extract_frustum_det_data and extract_frustum_data_rgb_detection (kitti/prepare_data_refine.py) pickle for seeded
synthetic scenes (oracle/kitti_refine_synth.py).  Needs the reference tree (oracle/ref_import.REF), cv2 and scipy; the
tests read only the fixture and regenerate the scans from its seeds.

    python -m oracle.make_golden_refine_extract

The scenes are written as data/kitti/training/{velodyne,calib,image_2,label_2} and a result directory in a temporary
directory, and the functions run with prepare_data_refine.ROOT_DIR pointed there.  Stubs: matplotlib (imported,
never called) and ops.pybind11.rbbox_iou.rbbox_iou_3d, which is compiled Boost code: rbbox_iou_3d_shim below, the
oracle's standup pre-filter and float64 clip (oracle/refine_extract.match_iou).  Each frame is drawn again until no
in-image point lies within 1e-9 m of a face of any box the reference tests (every cutting box, perturbed ones
included, and every label box) and no matching IoU lies within 1e-9 of its threshold, so Delaunay and the half-space
test, and the shim and any exact clip, decide alike.

Modes (prefix in the file): gt_train (perturb, augmentX = 5, seeded np.random), gt_val (remove_diff), matched
(remove_diff), det.  The first frame is drawn again until one of its perturbed augmentations has no labelled point
(the training set's drop rule).  Asserted: oracle/refine_extract.py reproduces every pickled list bit for bit."""
from __future__ import annotations

import contextlib
import io
import os
import pickle
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from frustum_convnet_b200 import refine_extract as rx  # noqa: E402
from oracle import kitti_refine_synth as krs  # noqa: E402
from oracle import kitti_scan_synth as ks  # noqa: E402
from oracle import refine_extract as orx  # noqa: E402
from oracle.ref_import import REF  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "refine_extract.npz")
WHITELIST = ("Car",)
TRAIN_SEED = 7
MODES = {"gt_train": dict(mode="gt", perturb=True, augment=5), "gt_val": dict(mode="gt", remove_diff=True),
         "matched": dict(mode="matched", remove_diff=True), "det": dict(mode="det")}


def rbbox_iou_3d_shim(boxes_3d, qboxes_3d, standup_thresh=0.0):
    """Stands in for the reference's Boost rbbox_iou_3d: (1, 7) x (G, 7) -> (1, G)."""
    return orx.match_iou(np.asarray(boxes_3d)[0], list(np.asarray(qboxes_3d)))[None]


def _reference():
    for name in ("matplotlib", "matplotlib.pyplot", "ops", "ops.pybind11", "ops.pybind11.rbbox_iou"):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules.setdefault(name, m)
    sys.modules["ops.pybind11.rbbox_iou"].rbbox_iou_3d = rbbox_iou_3d_shim
    sys.modules["ops.pybind11.rbbox_iou"].bbox_overlaps_2d = None
    for p in (REF, os.path.join(REF, "kitti")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import prepare_data_refine  # noqa: E402
    return prepare_data_refine


def objects(lines):
    return {k: [rx.KittiObject.parse(ln, "%06d.txt:%d" % (k, n + 1)) for n, ln in enumerate(v)]
            for k, v in lines.items()}


def run_reference(frames, labels, results):
    """frames {idx: (scan, calib, (H, W))} -> {mode: {list name: list}}."""
    import cv2
    pdr = _reference()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        split = os.path.join(tmp, "data", "kitti", "training")
        for d in ("velodyne", "calib", "image_2", "label_2"):
            os.makedirs(os.path.join(split, d))
        res = os.path.join(tmp, "results")
        os.makedirs(res)
        for idx, (scan, calib, (h, w)) in frames.items():
            np.ascontiguousarray(scan, dtype=np.float32).tofile(os.path.join(split, "velodyne", "%06d.bin" % idx))
            with open(os.path.join(split, "calib", "%06d.txt" % idx), "w") as f:
                for key in ("P2", "R0_rect", "Tr_velo_to_cam"):
                    f.write("%s: %s\n" % (key, " ".join(repr(float(x)) for x in np.asarray(calib[key]).reshape(-1))))
            cv2.imwrite(os.path.join(split, "image_2", "%06d.png" % idx), np.zeros((h, w, 3), np.uint8))
            with open(os.path.join(split, "label_2", "%06d.txt" % idx), "w") as f:
                f.write("".join(ln + "\n" for ln in labels[idx]))
            with open(os.path.join(res, "%06d.txt" % idx), "w") as f:
                f.write("".join(ln + "\n" for ln in results[idx]))
        ids = os.path.join(tmp, "ids.txt")
        with open(ids, "w") as f:
            f.write("".join("%06d\n" % i for i in frames))
        pdr.ROOT_DIR = tmp
        for part, kw in MODES.items():
            p = os.path.join(tmp, part + ".pickle")
            with contextlib.redirect_stdout(io.StringIO()), np.errstate(all="ignore"):
                if kw["mode"] == "gt":
                    np.random.seed(TRAIN_SEED)
                    pdr.extract_frustum_data(ids, "training", p, perturb_box2d=kw.get("perturb", False),
                                             augmentX=kw.get("augment", 1), type_whitelist=list(WHITELIST),
                                             remove_diff=kw.get("remove_diff", False))
                elif kw["mode"] == "matched":
                    pdr.extract_frustum_det_data(ids, "training", p, res, type_whitelist=list(WHITELIST),
                                                 remove_diff=True)
                else:
                    pdr.extract_frustum_data_rgb_detection(ids, "training", p, res, type_whitelist=list(WHITELIST))
            with open(p, "rb") as f:
                names = orx.LIST_NAMES[kw["mode"]]
                out[part] = {n: pickle.load(f) for n in names}
    return out


def run_oracle(frames, labels, results, part):
    kw = MODES[part]
    scans, calibs, hws = ({k: v[i] for k, v in frames.items()} for i in range(3))
    return orx.extract(kw["mode"], scans, calibs, hws, list(frames), objects(results), objects(labels), WHITELIST,
                       kw.get("remove_diff", False), kw.get("perturb", False), kw.get("augment", 1),
                       np.random.RandomState(TRAIN_SEED))


def _same_value(a, b):
    if isinstance(a, dict):
        return all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in ("P2",))
    if isinstance(a, str) or isinstance(b, str):
        return a == b
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def same(ref, mine):
    for n, r in ref.items():
        if len(r) != len(mine[n]) or not all(_same_value(a, b) for a, b in zip(r, mine[n])):
            print("  list %s differs" % n)
            return False
    return True


def clear(frames, labels, results):
    """No in-image point within BAND of a face of a tested box, no matching IoU within BAND of the threshold."""
    for part, kw in MODES.items():
        jobs, gts = rx.job_table(orx.MODES[kw["mode"]], list(frames), objects(results), objects(labels), WHITELIST,
                                 kw.get("remove_diff", False), kw.get("perturb", False), kw.get("augment", 1),
                                 np.random.RandomState(TRAIN_SEED))
        for jb in jobs:
            pc = orx.fov_points(*frames[jb["frame"]])
            boxes = [jb["cut"]] + [rx.obj_array(o) for o in gts.get(jb["frame"], [])]
            if any(np.any(np.abs(orx.box_margin(pc, b)) < orx.BAND) for b in boxes):
                return False
            if kw["mode"] == "matched":
                ov = orx.match_iou(jb["box"], [rx.obj_array(o) for o in gts[jb["frame"]]])
                if np.any(np.abs(ov - 0.5) < orx.BAND):
                    return False
    return True


def drops_augmentation(one, lab, res):
    """The first frame's perturbed training jobs include one without a labelled point (its draws still count)."""
    (idx,) = one
    L = run_oracle(one, {idx: lab}, {idx: res}, "gt_train")
    jobs, _ = rx.job_table(orx.MODES["gt"], [idx], None, objects({idx: lab}), WHITELIST, False, True, 5,
                           np.random.RandomState(TRAIN_SEED))
    return len(L["id_list"]) < len(jobs)


def main():
    frames, labels, results, seeds = {}, {}, {}, []
    for k, idx in enumerate((1, 4, 9, 10)):
        for attempt in range(50):
            seed = 100 * k + attempt
            scan, calib, hw, lab, res = krs.scene(seed)
            one = {idx: (scan, calib, hw)}
            if clear(one, {idx: lab}, {idx: res}) and (k > 0 or drops_augmentation(one, lab, res)):
                frames[idx], labels[idx], results[idx] = one[idx], lab, res
                seeds.append(seed)
                break
        else:
            raise SystemExit("no clear scene for frame %d" % idx)
    # frame 9 without any whitelisted ground truth (matched mode skips it), frame 10 without result lines
    labels[9] = [ln for ln in labels[9] if not ln.startswith("Car ")]
    results[10] = []
    assert clear(frames, labels, results)
    ref = run_reference(frames, labels, results)
    out = {"frame_ids": np.array(list(frames), np.int64), "seeds": np.array(seeds, np.int64),
           "train_seed": np.array(TRAIN_SEED), "checksum": np.array(ks.checksum([frames[i][0] for i in frames]))}
    for idx in frames:
        out["labels_%d" % idx] = np.array(labels[idx], dtype=str)
        out["results_%d" % idx] = np.array(results[idx], dtype=str)
    for part, lists in ref.items():
        assert same(lists, run_oracle(frames, labels, results, part)), "the oracle disagrees (%s)" % part
        store(out, part, lists)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


def store(out, part, lists):
    for n, v in lists.items():
        if n == "calib_list":
            out["%s_P2" % part] = np.array([np.asarray(c["P2"], np.float64) for c in v]).reshape(-1, 12)
        elif n in ("input_list", "label_list"):
            out["%s_%s" % (part, n)] = np.concatenate(v) if v else np.zeros((0, 4) if n == "input_list" else 0)
            out["%s_counts" % part] = np.array([len(p) for p in v], np.int64)
        else:
            out["%s_%s" % (part, n)] = np.array(v)
    print("%s: %d frustums, %d points" % (part, len(lists["id_list"]), sum(len(p) for p in lists["input_list"])))


if __name__ == "__main__":
    main()
