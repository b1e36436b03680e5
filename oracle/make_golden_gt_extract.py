"""Writes tests/golden/gt_extract.npz: what the reference's own, unmodified extract_frustum_data and
extract_frustum_det_data (kitti/prepare_data.py) pickle for seeded synthetic scenes (oracle/kitti_refine_synth.py).
Needs the reference tree (oracle/ref_import.REF), cv2 and scipy; the tests read only the fixture and regenerate the
scans from its seeds.

    python -m oracle.make_golden_gt_extract

The scenes are written as data/kitti/training/{velodyne,calib,image_2,label_2} plus a 2-D detection file
(read_det_file's 'path type prob xmin ymin xmax ymax' lines, made from the scenes' result lines) in a temporary
directory, and the functions run with prepare_data.ROOT_DIR pointed there.  bbox_overlaps_2d is the reference's own
ops/pybind11/rbbox_iou.py, imported with its compiled modules box_ops_cc and nms stubbed (never called on this path);
matplotlib is stubbed too.  Each frame is drawn again until no in-image point lies within BAND = 1e-9 m of a face of
any whitelisted ground truth's 3-D box (so Delaunay and the half-space test decide alike) or within 1e-7 px of an edge
of any cutting box (so the reference's np.dot projection and the elementwise one cut alike).

Added to the drawn scenes: a Car at the right image border whose perturbed boxes are retried after clipping, a Car
under 25 px tall with a detection on it (dropped on the host in every mode, after its draws), and a frame whose
perturbed training boxes include one without a labelled point (the first frame is drawn again until it has one).

Parts (prefix in the file): {car, people}_{train, val, matched}: whitelists ("Car",) and ("Pedestrian", "Cyclist");
train = perturb, augmentX = 5, np.random.seed(SEED); val = no perturbation; matched = extract_frustum_det_data with
perturb, augmentX = 5, np.random.seed(SEED).  Asserted: oracle/gt_extract.py reproduces every pickled list bit for
bit."""
from __future__ import annotations

import contextlib
import importlib.util
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

from frustum_convnet_b200 import gt_extract as gx  # noqa: E402
from frustum_convnet_b200.frustum_extract import read_rgb_detections  # noqa: E402
from oracle import gt_extract as ogx  # noqa: E402
from oracle import kitti_refine_synth as krs  # noqa: E402
from oracle import kitti_scan_synth as ks  # noqa: E402
from oracle import refine_extract as orx  # noqa: E402
from oracle.ref_import import REF  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "gt_extract.npz")
SEED = 3
FRAMES = (1, 4, 9, 10)
WHITELISTS = {"car": ("Car",), "people": ("Pedestrian", "Cyclist")}
MODES = {"train": dict(mode="gt", perturb=True, augment=5), "val": dict(mode="gt"),
         "matched": dict(mode="matched", perturb=True, augment=5)}
PARTS = tuple("%s_%s" % (w, m) for w in WHITELISTS for m in MODES)
EDGE_BAND = 1e-7
DET_ID = {"Pedestrian": 1, "Car": 2, "Cyclist": 3}


def _reference():
    for name in ("matplotlib", "matplotlib.pyplot", "ops.pybind11.box_ops_cc", "ops.pybind11.nms"):
        sys.modules[name] = types.ModuleType(name)
    for name, path in (("ops", os.path.join(REF, "ops")), ("ops.pybind11", os.path.join(REF, "ops", "pybind11"))):
        m = types.ModuleType(name)
        m.__path__ = [path]
        sys.modules[name] = m
    spec = importlib.util.spec_from_file_location("ops.pybind11.rbbox_iou",
                                                  os.path.join(REF, "ops", "pybind11", "rbbox_iou.py"))
    rbbox_iou = importlib.util.module_from_spec(spec)
    sys.modules["ops.pybind11.rbbox_iou"] = rbbox_iou
    spec.loader.exec_module(rbbox_iou)
    for p in (REF, os.path.join(REF, "kitti")):
        if p not in sys.path:
            sys.path.insert(0, p)
    sys.modules.pop("prepare_data", None)
    import prepare_data  # noqa: E402
    assert prepare_data.bbox_overlaps_2d is rbbox_iou.bbox_overlaps_2d
    return prepare_data


def det_lines(results):
    """{idx: result lines} -> read_det_file lines of the Car / Pedestrian / Cyclist results, frames in order; every
    other Car line names its type by the detector id."""
    out = []
    for idx, lines in results.items():
        for n, ln in enumerate(lines):
            t = ln.split(" ")
            if t[0] not in DET_ID:
                continue
            typ = str(DET_ID[t[0]]) if t[0] == "Car" and n % 2 else t[0]
            out.append("dataset/KITTI/object/training/image_2/%06d.png %s %s %s" % (idx, typ, t[15], " ".join(t[4:8])))
    return out


def objects(labels):
    return krs.objects(labels)


def run_reference(frames, labels, dets):
    """frames {idx: (scan, calib, (H, W))} -> {part: {list name: list}}."""
    import cv2
    pd = _reference()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        split = os.path.join(tmp, "data", "kitti", "training")
        for d in ("velodyne", "calib", "image_2", "label_2"):
            os.makedirs(os.path.join(split, d))
        for idx, (scan, calib, (h, w)) in frames.items():
            np.ascontiguousarray(scan, dtype=np.float32).tofile(os.path.join(split, "velodyne", "%06d.bin" % idx))
            with open(os.path.join(split, "calib", "%06d.txt" % idx), "w") as f:
                for key in ("P2", "R0_rect", "Tr_velo_to_cam"):
                    f.write("%s: %s\n" % (key, " ".join(repr(float(x)) for x in np.asarray(calib[key]).reshape(-1))))
            cv2.imwrite(os.path.join(split, "image_2", "%06d.png" % idx), np.zeros((h, w, 3), np.uint8))
            with open(os.path.join(split, "label_2", "%06d.txt" % idx), "w") as f:
                f.write("".join(ln + "\n" for ln in labels[idx]))
        ids = os.path.join(tmp, "ids.txt")
        with open(ids, "w") as f:
            f.write("".join("%06d\n" % i for i in frames))
        det = os.path.join(tmp, "det.txt")
        with open(det, "w") as f:
            f.write("".join(ln + "\n" for ln in dets))
        pd.ROOT_DIR = tmp
        for part in PARTS:
            wl, kw = WHITELISTS[part.split("_")[0]], MODES[part.split("_")[1]]
            p = os.path.join(tmp, part + ".pickle")
            with contextlib.redirect_stdout(io.StringIO()), np.errstate(all="ignore"):
                np.random.seed(SEED)
                if kw["mode"] == "gt":
                    pd.extract_frustum_data(ids, "training", p, perturb_box2d=kw.get("perturb", False),
                                            augmentX=kw.get("augment", 1), type_whitelist=list(wl))
                else:
                    pd.extract_frustum_det_data(ids, "training", p, det, perturb_box2d=kw.get("perturb", False),
                                                augmentX=kw.get("augment", 1), type_whitelist=list(wl))
            with open(p, "rb") as f:
                out[part] = {n: pickle.load(f) for n in gx.NAMES}
    return out


def run_oracle(frames, labels, dets, part):
    wl, kw = WHITELISTS[part.split("_")[0]], MODES[part.split("_")[1]]
    scans, calibs, hws = ({k: v[i] for k, v in frames.items()} for i in range(3))
    return ogx.extract(kw["mode"], scans, calibs, hws, list(frames), objects(labels), wl, kw.get("perturb", False),
                       kw.get("augment", 1), np.random.RandomState(SEED), read_rgb_detections(dets))


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


def clear(frames, labels, dets):
    """No in-image point within BAND of a face of a whitelisted ground truth's 3-D box, none within EDGE_BAND of an
    edge of a cutting box."""
    gt = objects(labels)
    for part in PARTS:
        wl, kw = WHITELISTS[part.split("_")[0]], MODES[part.split("_")[1]]
        pcs = {k: ogx.fov_points(*frames[k]) for k in frames}
        for k in frames:
            for o in gt[k]:
                if o.type in wl and np.any(np.abs(orx.box_margin(pcs[k][0], gx.obj_array(o))) < orx.BAND):
                    return False
        jobs = ogx.jobs_of(kw["mode"], list(frames), gt, wl, {k: v[2] for k, v in frames.items()},
                           kw.get("perturb", False), kw.get("augment", 1), np.random.RandomState(SEED),
                           read_rgb_detections(dets))
        for jb in jobs:
            _, u, v = pcs[jb["frame"]]
            b = jb["cut"]
            if min(np.abs(u[:, None] - b[[0, 2]]).min(initial=1.0), np.abs(v[:, None] - b[[1, 3]]).min(initial=1.0)) \
                    < EDGE_BAND:
                return False
    return True


def drops_augmentation(frames, labels):
    """The car training jobs include one without a labelled point (its draws still count)."""
    L = run_oracle(frames, labels, [], "car_train")
    jobs = ogx.jobs_of("gt", list(frames), objects(labels), WHITELISTS["car"], {k: v[2] for k, v in frames.items()},
                       True, 5, np.random.RandomState(SEED))
    return len(L["id_list"]) < len(jobs)


def _label(typ, box2d, h, w, l, t, ry):
    return krs._line(typ, 0.0, 0, box2d, h, w, l, t, ry)


def main():
    frames, labels, results, seeds = {}, {}, {}, []
    for k, idx in enumerate(FRAMES):
        for attempt in range(50):
            seed = 500 + 100 * k + attempt
            scan, calib, hw, lab, res = krs.scene(seed)
            if k == 0:
                H, W = hw
                lab = lab + [_label("Car", [W - 1 - 0.05, 150.0, W - 1 + 20.0, 200.0], 1.5, 1.6, 3.9,
                                    [14.0, 1.65, 16.0], 0.1),                       # retried after clipping
                             _label("Car", [400.0, 180.0, 430.0, 200.0], 1.5, 1.6, 3.9, [-8.0, 1.65, 40.0], 0.2)]
                res = res + [krs._line("Car", -1, -1, [400.0, 180.0, 430.0, 200.0], 1.5, 1.6, 3.9,
                                       [-8.0, 1.65, 40.0], 0.2, 0.9)]              # matches the < 25 px Car
            one = {idx: (scan, calib, hw)}
            d = det_lines({idx: res})
            if clear(one, {idx: lab}, d) and (k > 0 or drops_augmentation(one, {idx: lab})):
                frames[idx], labels[idx], results[idx] = one[idx], lab, res
                seeds.append(seed)
                break
        else:
            raise SystemExit("no clear scene for frame %d" % idx)
    # frame 9 without any whitelisted Car ground truth (matched car mode skips it), frame 10 without detections
    labels[9] = [ln for ln in labels[9] if not ln.startswith("Car ")]
    results[10] = []
    dets = det_lines(results)
    assert clear(frames, labels, dets)
    ref = run_reference(frames, labels, dets)
    out = {"frame_ids": np.array(list(frames), np.int64), "seeds": np.array(seeds, np.int64),
           "train_seed": np.array(SEED), "checksum": np.array(ks.checksum([frames[i][0] for i in frames])),
           "dets": np.array(dets, dtype=str)}
    for idx in frames:
        out["labels_%d" % idx] = np.array(labels[idx], dtype=str)
    for part, lists in ref.items():
        assert same(lists, run_oracle(frames, labels, dets, part)), "the oracle disagrees (%s)" % part
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
