"""Writes tests/golden/frustum_extract.npz: what the reference's own, unmodified extract_frustum_data_rgb_detection
(kitti/prepare_data.py:462-568) pickles for seeded synthetic scenes (oracle/kitti_scan_synth.py).  Needs the reference
tree (oracle/ref_import.REF) and cv2; the tests read only the fixture and regenerate the scans from its seeds.

    python -m oracle.make_golden_frustum_extract

The scenes are written as a data/kitti/training/{velodyne,calib,image_2} tree in a temporary directory (calib values
printed with repr, so they read back as the same float64; blank PNGs of the image size) and the function runs with
prepare_data.ROOT_DIR pointed there.  matplotlib, matplotlib.pyplot and ops.pybind11.rbbox_iou are only imported by the
reference's modules, never called on this path: they are stubbed in sys.modules.

Parts (prefix in the file):
  exact  kitti_scan_synth.exact_scene with a Car whitelist: points on every box and image edge, decided identically by
         any rounding order (drawn again until the box meant to be empty is);
  real   one ~20k-point frame per image of the first 40 lines of the reference's rgb_detection_val.txt (the lines are
         stored verbatim as `val_lines`), whitelist Car, Pedestrian, Cyclist; each frame is drawn again until no u, v
         lies within 1e-9 px of an edge and the oracle's float32 points equal the pickle's.
Asserted for both: oracle/frustum_extract.py reproduces every pickled list bit for bit."""
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

from oracle import frustum_extract as ofx  # noqa: E402
from oracle import kitti_scan_synth as ks  # noqa: E402
from oracle.ref_import import REF  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "frustum_extract.npz")
VAL = os.path.join(REF, "kitti", "rgb_detections", "rgb_detection_val.txt")


def _reference():
    for name in ("matplotlib", "matplotlib.pyplot", "ops", "ops.pybind11", "ops.pybind11.rbbox_iou"):
        m = types.ModuleType(name)
        m.__path__ = []
        sys.modules.setdefault(name, m)
    sys.modules["ops.pybind11.rbbox_iou"].bbox_overlaps_2d = None
    for p in (REF, os.path.join(REF, "kitti")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import prepare_data  # noqa: E402
    return prepare_data


def run_reference(frames, lines, whitelist):
    """frames {idx: (scan, calib, (H, W))}, detection lines -> the seven pickled lists."""
    import cv2
    pd = _reference()
    with tempfile.TemporaryDirectory() as tmp:
        split = os.path.join(tmp, "data", "kitti", "training")
        for d in ("velodyne", "calib", "image_2"):
            os.makedirs(os.path.join(split, d))
        for idx, (scan, calib, (h, w)) in frames.items():
            np.ascontiguousarray(scan, dtype=np.float32).tofile(os.path.join(split, "velodyne", "%06d.bin" % idx))
            with open(os.path.join(split, "calib", "%06d.txt" % idx), "w") as f:
                for key in ("P2", "R0_rect", "Tr_velo_to_cam"):
                    f.write("%s: %s\n" % (key, " ".join(repr(float(x)) for x in np.asarray(calib[key]).reshape(-1))))
            cv2.imwrite(os.path.join(split, "image_2", "%06d.png" % idx), np.zeros((h, w, 3), np.uint8))
        det = os.path.join(tmp, "det.txt")
        with open(det, "w") as f:
            f.write("".join(ln + "\n" for ln in lines))
        out = os.path.join(tmp, "out.pickle")
        pd.ROOT_DIR = tmp
        with contextlib.redirect_stdout(io.StringIO()):
            pd.extract_frustum_data_rgb_detection(det, "training", out, type_whitelist=list(whitelist))
        with open(out, "rb") as f:
            lists = [pickle.load(f) for _ in range(7)]
    return lists


def read_det_lines(lines):
    pd = _reference()
    with tempfile.TemporaryDirectory() as tmp:
        p = os.path.join(tmp, "det.txt")
        with open(p, "w") as f:
            f.write("".join(ln + "\n" for ln in lines))
        return pd.read_det_file(p)          # id, type, box2d, prob


def oracle_lists(frames, lines, whitelist):
    ids, types_, boxes, probs = read_det_lines(lines)
    return ofx.extract({k: v[0] for k, v in frames.items()}, {k: v[1] for k, v in frames.items()},
                       {k: v[2] for k, v in frames.items()}, ids, types_, probs, boxes, whitelist)


def same(ref, mine):
    """Every pickled list bit for bit (points, order, ids, types, probabilities, boxes, angles, calib P2)."""
    r_id, r_box, r_in, r_type, r_ang, r_prob, r_cal = ref
    m_id, m_box, m_in, m_type, m_ang, m_prob, m_cal = mine
    if r_id != m_id or r_type != m_type or r_prob != m_prob or len(r_in) != len(m_in):
        return False
    for a, b in zip(r_in, m_in):
        if a.dtype != np.float32 or a.shape != b.shape or a.tobytes() != b.tobytes():
            return False
    for a, b in zip(r_box, m_box):
        if np.asarray(a).tobytes() != np.asarray(b, dtype=np.float64).tobytes():
            return False
    if np.asarray(r_ang, np.float64).tobytes() != np.asarray(m_ang, np.float64).tobytes():
        return False
    return all(np.asarray(a["P2"]).tobytes() == np.asarray(b["P2"], np.float64).tobytes() for a, b in zip(r_cal, m_cal))


def store(out, part, lists, lines, whitelist, frames):
    r_id, r_box, r_in, r_type, r_ang, r_prob, r_cal = lists
    out[part + "_lines"] = np.array(lines)
    out[part + "_whitelist"] = np.array(whitelist)
    out[part + "_frame_ids"] = np.array(sorted(frames), dtype=np.int64)
    out[part + "_checksum"] = np.array(ks.checksum([frames[i][0] for i in sorted(frames)]))
    out[part + "_ids"] = np.array(r_id, dtype=np.int64)
    out[part + "_types"] = np.array(r_type)
    out[part + "_probs"] = np.array(r_prob, dtype=np.float64)
    out[part + "_boxes"] = np.array(r_box, dtype=np.float64).reshape(-1, 4)
    out[part + "_counts"] = np.array([len(p) for p in r_in], dtype=np.int64)
    out[part + "_points"] = np.concatenate(r_in).astype(np.float32) if r_in else np.zeros((0, 4), np.float32)
    out[part + "_angles"] = np.array(r_ang, dtype=np.float64)
    out[part + "_P2"] = np.array([np.asarray(c["P2"], np.float64) for c in r_cal]).reshape(-1, 12)
    print("%s: %d lines, %d frames, %d kept, %d points" % (part, len(lines), len(frames), len(r_id),
                                                           sum(len(p) for p in r_in)))


def main():
    out = {}
    val_lines = [ln.rstrip("\n") for ln in open(VAL)][:40]
    out["val_lines"] = np.array(val_lines)
    v_id, v_type, v_box, v_prob = read_det_lines(val_lines)
    out["val_ids"], out["val_types"] = np.array(v_id, dtype=np.int64), np.array(v_type)
    out["val_probs"], out["val_boxes"] = np.array(v_prob, dtype=np.float64), np.array(v_box, dtype=np.float64)

    wl = ("Car",)
    for seed in range(1, 100):
        frames, lines = ks.exact_scene(seed)
        lists = run_reference(frames, lines, wl)
        _, u, v = ofx.project(frames[5][0], frames[5][1])
        fov = ofx.in_image(frames[5][0], u, v, ks.H, ks.W)
        if np.any(fov & (u >= 300) & (u < 360) & (v >= 5) & (v < 40)):
            continue                               # the empty box caught a clutter point: draw again
        assert same(lists, oracle_lists(frames, lines, wl)), "the oracle disagrees with the reference (exact part)"
        out["exact_seed"] = np.array(seed)
        store(out, "exact", lists, lines, wl, frames)
        break
    else:
        raise SystemExit("no exact scene without a point in its empty box")

    wl = ("Car", "Pedestrian", "Cyclist")
    groups = {}
    for ln in val_lines:
        groups.setdefault(ks.det_id(ln), []).append(ln)
    frames, seeds = {}, {}
    for j, (idx, own) in enumerate(groups.items()):
        for attempt in range(100):
            seed = 1000 + 100 * j + attempt
            scan, calib, hw = ks.realistic_scene(seed, own)
            _, u, v = ofx.project(scan, calib)
            if not ks.edges_clear(u, v, hw, [ks.parse_line(ln)[2] for ln in own]):
                continue
            single = {idx: (scan, calib, hw)}
            if not same(run_reference(single, own, wl), oracle_lists(single, own, wl)):
                print("frame %d seed %d: the float32 points of np.dot and the elementwise order differ" % (idx, seed))
                continue
            frames[idx], seeds[idx] = single[idx], seed
            break
        else:
            raise SystemExit("no clean realistic scene for image %d" % idx)
    lists = run_reference(frames, val_lines, wl)
    assert same(lists, oracle_lists(frames, val_lines, wl)), "the oracle disagrees with the reference (real part)"
    out["real_seeds"] = np.array([seeds[i] for i in sorted(frames)], dtype=np.int64)
    store(out, "real", lists, val_lines, wl, frames)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
