"""Writes tests/golden/sunrgbd_extract.npz: what the reference's own, unmodified extract_frustum_data and
extract_frustum_data_from_rgb_detection (sunrgbd/prepare_data.py) pickle for seeded synthetic frames
(oracle/sunrgbd_scene_synth.py).  Needs the reference tree (oracle/ref_import.REF), cv2, PIL and scipy; the tests read
only the fixture and regenerate the clouds from its seeds.

    python -m oracle.make_golden_sunrgbd_extract

The frames are written as mysunrgbd/training/{calib,label,pc} (pc/%06d.mat via scipy.io.savemat, key 'x') in a
temporary directory, with an index file and a detection file ('data_idx type prob xmin ymin xmax ymax').  Parts, each
after np.random.seed(SEED), with the generator's next random() recorded after the call:
  train      extract_frustum_data, perturb_box2d=True, augmentX=5 (--gen_train);
  val        extract_frustum_data, unperturbed, augmentX=1 (--gen_val);
  det        extract_frustum_data_from_rgb_detection (--gen_val_rgb_detection);
  det_valid  the same with valid_id_list=VALID.
Each frame is drawn again (next seed) until no point lies within 1e-9 m of a face of a whitelisted label box or within
1e-7 px of an edge of a cutting box, and the set covers every rule (covers() below).  Asserted:
oracle/sunrgbd_extract.py reproduces every key bit for bit and leaves the generator in the same state.  The fixture
keeps the small lists, the per-frustum counts and SHA-256 digests of the points and labels."""
from __future__ import annotations

import contextlib
import hashlib
import importlib.util
import io
import os
import pickle
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from frustum_convnet_b200 import sunrgbd_extract as sx  # noqa: E402
from oracle import sunrgbd_extract as osx  # noqa: E402
from oracle import sunrgbd_scene_synth as sss  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "sunrgbd_extract.npz")
SEED = 7
H, W = 120, 160
TINY = {"half": (0.02, 0.02, 0.02)}
SPECS = {
    1: [("chair", 0.3, 0.35, 42.0, 44.0, 200, {}),          # about 2048 points: capped in some augmentations only
        ("table", 0.65, 0.5, 70.0, 70.0, 8, TINY),          # > 2048 points, 8 labelled: < 5 among the chosen
        ("desk", 0.25, 0.8, 30.0, 22.0, 3, TINY),           # <= 2048 points, 3 labelled: dropped
        ("sofa", 0.85, 0.2, 20.0, 20.0, 30, {"zero_h": True}),   # zero extent: skipped, no choice
        ("lamp", 0.5, 0.15, 20.0, 20.0, 30, {}),            # not whitelisted
        ("bed", 0.45, 0.7, 55.0, 50.0, 600, {})],
    2: [("chair", 0.4, 0.4, 50.0, 45.0, 300, {}), ("bed", 0.75, 0.6, 35.0, 30.0, 400, {})],
    3: [("toilet", 0.5, 0.5, 40.0, 40.0, 150, {}), ("lamp", 0.2, 0.2, 30.0, 30.0, 40, {})],
}
VALID = [1, 3]
PARTS = ("train", "val", "det", "det_valid")


def frames_of(seeds):
    return {idx: sss.frame(seed, H, W, SPECS[idx]) for idx, seed in seeds.items()}


def det_lines(labels, seed):
    """Detections jittered off the label boxes, frames 1, 2, 1, 3 (frame 1 again after frame 2), plus a 1.5 px chair
    box (fewer than 5 points) in frame 2."""
    rng = np.random.default_rng(seed)
    out = []

    def add(idx, objs):
        for o in objs:
            b = o.box2d + rng.uniform(-3, 3, 4)
            out.append("%d %s %r %r %r %r %r" % (idx, o.classname, float(rng.uniform(0.1, 1)), *map(float, b)))
    add(1, labels[1][:3])
    add(2, labels[2])
    c = labels[2][0].box2d
    out.append("2 chair 0.5 %r %r %r %r" % tuple(float(x) for x in (c[0] + 5.0, c[1] + 5.0, c[0] + 6.5, c[1] + 6.5)))
    add(1, labels[1][3:])
    add(3, labels[3])
    return out


def parse_dets(lines):
    with tempfile.TemporaryDirectory() as tmp:
        p = os.path.join(tmp, "det.txt")
        with open(p, "w") as f:
            f.write("".join(ln + "\n" for ln in lines))
        return sx.read_det_file(p)


def labels_of(frames):
    return {idx: [sx.SUNObject3d(ln, "%d:%d" % (idx, k + 1)) for k, ln in enumerate(fr[2])]
            for idx, fr in frames.items()}


def run_oracle(frames, dets, part, rng):
    points = {k: v[0] for k, v in frames.items()}
    calibs = {k: v[1] for k, v in frames.items()}
    labels = labels_of(frames)
    ids = list(frames)
    if part == "train":
        return osx.from_ground_truth(points, calibs, ids, labels, perturb=True, augment=5, rng=rng)
    if part == "val":
        return osx.from_ground_truth(points, calibs, ids, labels, rng=rng)
    return osx.from_rgb_detections(points, calibs, *parse_dets(dets), valid_ids=VALID if part == "det_valid" else None,
                                   rng=rng)


def clear(frames, dets):
    """No point within BAND of a face of a whitelisted label box, none within EDGE_BAND of a cutting box's edge."""
    labels = labels_of(frames)
    for idx, (pc, cal, _) in frames.items():
        cam = osx.camera_points(pc)
        for o in labels[idx]:
            if o.classname in sx.TYPE_WHITELIST and not sx.zero_extent(o) and \
                    np.abs(osx.box_margin(cam, o)).min() < osx.BAND:
                return False
    for part in PARTS:
        boxes = []
        rng = np.random.RandomState(SEED)
        L, trace = run_oracle(frames, dets, part, rng)
        rng = np.random.RandomState(SEED)
        # the cutting boxes of every job, drawn again in the same order (the trace holds the frames)
        if part == "train":
            for idx in frames:
                for o in labels_of(frames)[idx]:
                    if o.classname in sx.TYPE_WHITELIST:
                        for _ in range(5):
                            boxes.append((idx, sx.random_shift_box2d(o.box2d, rng)))
                            t = trace[len(boxes) - 1]
                            if t["choice"]:
                                rng.choice(t["n"], sx.CAP, replace=False)
        elif part == "val":
            boxes = [(idx, o.box2d) for idx in frames for o in labels[idx] if o.classname in sx.TYPE_WHITELIST]
        else:
            ids, types, bx, _ = parse_dets(dets)
            boxes = [(i, b) for i, t, b in zip(ids, types, bx) if t in sx.TYPE_WHITELIST]
        for idx, b in boxes:
            uv = osx.image_coords(frames[idx][0], frames[idx][1])
            if min(np.abs(uv[:, 0:1] - b[[0, 2]]).min(), np.abs(uv[:, 1:2] - b[[1, 3]]).min()) < osx.EDGE_BAND:
                return False
    return True


def covers(frames, dets):
    """The set exercises every rule: capped and uncapped frustums within one object's augmentations, a job dropped
    after its choice, one dropped with n <= 2048, a skipped zero-extent box, a detection with < 5 points."""
    _, tr = run_oracle(frames, dets, "train", np.random.RandomState(SEED))
    _, tv = run_oracle(frames, dets, "val", np.random.RandomState(SEED))
    _, td = run_oracle(frames, dets, "det", np.random.RandomState(SEED))
    mixed = any(len({t["n"] > sx.CAP for t in tr[k:k + 5]}) == 2 for k in range(0, len(tr), 5))
    after_choice = any(t["choice"] and t["in_box"] >= 5 and t["chosen"] < 5 for t in tr + tv)
    small = any(not t["skipped"] and t["n"] <= sx.CAP and not t["kept"] for t in tr + tv)
    skipped = any(t["skipped"] for t in tr)
    few = any(t["n"] < 5 for t in td)
    return mixed and after_choice and small and skipped and few


def _reference():
    from oracle.ref_import import REF
    sys.path.insert(0, os.path.join(REF, "sunrgbd"))
    spec = importlib.util.spec_from_file_location("sunrgbd_prepare_data", os.path.join(REF, "sunrgbd",
                                                                                       "prepare_data.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def run_reference(frames, dets):
    """-> {part: (the pickled dict, the generator's next random())}."""
    import scipy.io
    pd = _reference()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "mysunrgbd")
        split = os.path.join(root, "training")
        for d in ("calib", "label", "pc"):
            os.makedirs(os.path.join(split, d))
        for idx, (pc, cal, lines) in frames.items():
            scipy.io.savemat(os.path.join(split, "pc", "%06d.mat" % idx), {"x": pc})
            with open(os.path.join(split, "calib", "%06d.txt" % idx), "w") as f:
                for key in ("Rtilt", "K"):
                    f.write(" ".join(repr(float(x)) for x in cal[key].reshape(-1, order="F")) + "\n")
            with open(os.path.join(split, "label", "%06d.txt" % idx), "w") as f:
                f.write("".join(ln + "\n" for ln in lines))
        ids = os.path.join(tmp, "ids.txt")
        with open(ids, "w") as f:
            f.write("".join("%d\n" % i for i in frames))
        det = os.path.join(tmp, "det.txt")
        with open(det, "w") as f:
            f.write("".join(ln + "\n" for ln in dets))
        wl = set(sx.TYPE_WHITELIST)
        for part in PARTS:
            p = os.path.join(tmp, part + ".pickle")
            with contextlib.redirect_stdout(io.StringIO()), np.errstate(all="ignore"):
                np.random.seed(SEED)
                if part == "train":
                    pd.extract_frustum_data(root, ids, "training", p, wl, perturb_box2d=True, augmentX=5)
                elif part == "val":
                    pd.extract_frustum_data(root, ids, "training", p, wl, perturb_box2d=False, augmentX=1)
                else:
                    pd.extract_frustum_data_from_rgb_detection(root, det, "training", p, wl,
                                                               valid_id_list=VALID if part == "det_valid" else None)
                nxt = np.random.random()
            with open(p, "rb") as f:
                out[part] = (pickle.load(f), nxt)
    return out


def same(ref, mine):
    for k, r in ref.items():
        m = mine[k]
        if len(r) != len(m):
            print("  key %s: %d vs %d" % (k, len(r), len(m)))
            return False
        for a, b in zip(r, m):
            if isinstance(a, str):
                ok = a == b
            else:
                a, b = np.asarray(a), np.asarray(b)
                ok = a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
            if not ok:
                print("  key %s differs" % k)
                return False
    return True


def digest(arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def checksum(frames):
    return digest([frames[k][0] for k in sorted(frames)])


def store(out, part, d, nxt):
    for k, v in d.items():
        if k == "input":
            out[part + "_counts"] = np.array([len(p) for p in v], np.int64)
            out[part + "_input_sha256"] = np.array(digest(v))
        elif k == "label":
            out[part + "_label_sha256"] = np.array(digest(v))
        else:
            out[part + "_" + k] = np.array(v)
    out[part + "_next_random"] = np.array(nxt)
    print("%s: %d frustums, %d points" % (part, len(d["id"]), sum(len(p) for p in d["input"])))


def main():
    seeds = {idx: 100 * idx for idx in SPECS}
    for attempt in range(200):
        frames = frames_of(seeds)
        dets = det_lines(labels_of(frames), SEED + attempt)
        if covers(frames, dets) and clear(frames, dets):
            break
        seeds = {idx: s + 1 for idx, s in seeds.items()}
    else:
        raise SystemExit("no clear scene covering every rule")
    ref = run_reference(frames, dets)
    out = {"frame_ids": np.array(list(frames), np.int64), "seeds": np.array([seeds[i] for i in frames], np.int64),
           "seed": np.array(SEED), "checksum": np.array(checksum(frames)), "dets": np.array(dets, dtype=str),
           "det_seed": np.array(SEED + attempt), "valid": np.array(VALID, np.int64)}
    for idx, (pc, cal, lines) in frames.items():
        out["labels_%d" % idx] = np.array(lines, dtype=str)
        out["Rtilt_%d" % idx], out["K_%d" % idx] = cal["Rtilt"], cal["K"]
    for part, (d, nxt) in ref.items():
        rng = np.random.RandomState(SEED)
        mine, _ = run_oracle(frames, dets, part, rng)
        assert same(d, mine), "the oracle disagrees (%s)" % part
        assert rng.random() == nxt, "the oracle leaves the generator elsewhere (%s)" % part
        store(out, part, d, nxt)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
