"""CPU: the SUN-RGBD frustum extractor's host side (frustum_convnet_b200/sunrgbd_extract.py) and its numpy oracle
(oracle/sunrgbd_extract.py) against the reference's own pickles (tests/golden/sunrgbd_extract.npz, written by
oracle/make_golden_sunrgbd_extract.py): the oracle, the readers, the label-box record against the flipped corners, the
round driver against the sequential oracle, the dgemm order the device projection restates, the C ABI entries'
argument checks (on the host, before any CUDA call) and the ctypes struct layout."""
import ctypes
import hashlib
import os
from fractions import Fraction

import numpy as np
import pytest

from conftest import GOLDEN_DIR

GOLDEN = os.path.join(GOLDEN_DIR, "sunrgbd_extract.npz")
PARTS = ("train", "val", "det", "det_valid")


def scenes():
    """-> (npz, points {idx}, calibs {idx}, labels {idx: [SUNObject3d]}, detection lists)."""
    from frustum_convnet_b200 import sunrgbd_extract as sx
    from oracle import make_golden_sunrgbd_extract as mg
    z = np.load(GOLDEN)
    seeds = dict(zip(z["frame_ids"].tolist(), z["seeds"].tolist()))
    frames = mg.frames_of(seeds)
    assert mg.checksum(frames) == str(z["checksum"]), "the scene generator drifted from the fixture"
    points = {k: v[0] for k, v in frames.items()}
    calibs = {k: v[1] for k, v in frames.items()}
    labels = {k: [sx.SUNObject3d(str(ln), "%d:%d" % (k, n + 1)) for n, ln in enumerate(z["labels_%d" % k])]
              for k in frames}
    return z, points, calibs, labels, mg.parse_dets([str(s) for s in z["dets"]])


def oracle_part(part, z, points, calibs, labels, dets, rng):
    from oracle import sunrgbd_extract as osx
    ids = z["frame_ids"].tolist()
    if part == "train":
        return osx.from_ground_truth(points, calibs, ids, labels, perturb=True, augment=5, rng=rng)
    if part == "val":
        return osx.from_ground_truth(points, calibs, ids, labels, rng=rng)
    return osx.from_rgb_detections(points, calibs, *dets, valid_ids=z["valid"].tolist() if part == "det_valid"
                                   else None, rng=rng)


def sha(arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def check_dict(z, part, d):
    """d: the reference's dict (the oracle's, an unpickled file's, or built from a SunrgbdFrustums)."""
    p = part + "_"
    assert [len(x) for x in d["input"]] == z[p + "counts"].tolist()
    assert all(x.dtype == np.float32 and x.shape[1] == 6 for x in d["input"])
    assert sha(d["input"]) == str(z[p + "input_sha256"])
    if "label" in d:
        assert all(x.dtype == bool for x in d["label"])
        assert sha(d["label"]) == str(z[p + "label_sha256"])
    for k, v in d.items():
        if k in ("input", "label"):
            continue
        want = z[p + k]
        got = np.array(v)
        assert got.dtype == want.dtype and got.shape == want.shape and got.tobytes() == want.tobytes(), k


@pytest.mark.parametrize("part", PARTS)
def test_oracle_reproduces_the_reference_pickle(part):
    z, *sc = scenes()
    rng = np.random.RandomState(int(z["seed"]))
    d, _ = oracle_part(part, z, *sc, rng)
    assert len(d["id"]) > 0
    check_dict(z, part, d)
    assert rng.random() == float(z[part + "_next_random"])


def test_readers_restate_the_references(tmp_path):
    from frustum_convnet_b200 import sunrgbd_extract as sx
    z, points, calibs, labels, dets = scenes()
    for idx in z["frame_ids"].tolist():
        p = tmp_path / ("%06d.txt" % idx)
        with open(p, "w") as f:
            for key in ("Rtilt", "K"):
                f.write(" ".join(repr(float(x)) for x in z["%s_%d" % (key, idx)].reshape(-1, order="F")) + "\n")
        c = sx.read_calib(str(p))
        for key in ("Rtilt", "K"):
            assert c[key].tobytes() == z["%s_%d" % (key, idx)].tobytes()
            assert not c[key].flags.c_contiguous         # order='F', as SUNRGBD_Calibration reshapes
        for o, line in zip(labels[idx], z["labels_%d" % idx]):
            t = [float(x) for x in str(line).split(" ")[1:]]
            assert o.xmax == t[0] + t[2] and o.ymax == t[1] + t[3]
            assert o.heading_angle == -1 * np.arctan2(t[15], t[14])
            assert (o.w, o.l, o.h) == (t[7], t[8], t[9])
    ids, types, boxes, probs = dets
    assert ids == [int(str(s).split(" ")[0]) for s in z["dets"]]
    assert ids.index(2) < len(ids) - 1 - ids[::-1].index(1)           # frame 1 reappears after frame 2
    assert "lamp" in types and all(b.dtype == np.float64 for b in boxes)


def test_box_record_matches_the_flipped_corners():
    """box_record's half-space test puts the flipped compute_box_3d corners on the faces, their centre inside and
    points just outside every face outside, for any heading (both signs of sin and cos)."""
    from frustum_convnet_b200 import sunrgbd_extract as sx
    from oracle import sunrgbd_extract as osx
    from oracle import sunrgbd_scene_synth as sss
    rng = np.random.default_rng(3)
    for t in np.linspace(-np.pi, np.pi, 13):
        l, w, h = rng.uniform(0.2, 1.0, 3)
        obj = sx.SUNObject3d(sss.label_line("bed", [0, 0, 10, 10], rng.uniform(-2, 2, 3), w, l, h, t))
        corners = sx.box3d_corners(obj)
        r = sx.box_record(obj)
        c = corners.mean(0)
        assert np.allclose(c, r["center"], atol=1e-12)
        d = corners - r["center"]
        lx = r["cs"] * d[:, 0] - r["sn"] * d[:, 2]
        lz = r["sn"] * d[:, 0] + r["cs"] * d[:, 2]
        assert np.allclose(np.abs(lx), r["half"][0], atol=1e-12)
        assert np.allclose(np.abs(d[:, 1]), r["half"][1], atol=1e-12)
        assert np.allclose(np.abs(lz), r["half"][2], atol=1e-12)
        inner = c + (corners - c) * 0.999
        outer = c + (corners - c) * 1.001
        assert osx.in_box(inner, obj).all() and not osx.in_box(outer, obj).any()
        # the faces: the centre moved 1.001 half extents along each corner-to-corner axis is outside
        for a, b in ((0, 1), (0, 3), (0, 4)):
            axis = corners[b] - corners[a]
            assert not osx.in_box((c + 0.5005 * axis)[None], obj).any()
            assert osx.in_box((c + 0.4995 * axis)[None], obj).all()


def _slots(labels, ids, perturb):
    from frustum_convnet_b200 import sunrgbd_extract as sx
    return [dict(frame=i, box=o.box2d, skip=sx.zero_extent(o)) for i in ids for o in labels[i]
            if o.classname in sx.TYPE_WHITELIST for _ in range(5 if perturb else 1)]


@pytest.mark.parametrize("window", [1, 2, 7, 1024])
def test_round_driver_replays_the_sequential_stream(window):
    """replay with the oracle's counts in place of the device: the same cutting boxes, counts, choices and final
    generator state as the sequential oracle, at every window."""
    from frustum_convnet_b200 import sunrgbd_extract as sx
    from oracle import sunrgbd_extract as osx
    z, points, calibs, labels, dets = scenes()
    ids = z["frame_ids"].tolist()
    for perturb in (True, False):
        slots = _slots(labels, ids, perturb)
        seq = np.random.RandomState(11)
        _, trace = osx.from_ground_truth(points, calibs, ids, labels, perturb=perturb, augment=5 if perturb else 1,
                                         rng=seq)
        rng = np.random.RandomState(11)
        calls = []
        count = osx.counter(points, calibs, slots)
        cuts, n, choices, rounds = sx.replay(slots, perturb, rng, lambda b, e, c: calls.append(e - b) or
                                             count(b, e, c), window)
        assert rng.random() == seq.random()
        assert [t["n"] if not t["skipped"] else -1 for t in trace] == n.tolist()
        assert sorted(choices) == [k for k, t in enumerate(trace) if t["choice"]]
        assert rounds == len(calls) and max(calls) <= (window if perturb else len(slots))
        # the choices themselves: drawn again from a sequential replay
        rs = np.random.RandomState(11)
        for k, s in enumerate(slots):
            box = sx.random_shift_box2d(s["box"], rs) if perturb else s["box"]
            assert np.array_equal(box, cuts[k])
            if k in choices:
                assert np.array_equal(rs.choice(int(n[k]), sx.CAP, replace=False), choices[k])


def test_the_fixture_covers_every_rule():
    from frustum_convnet_b200 import sunrgbd_extract as sx
    from oracle import make_golden_sunrgbd_extract as mg
    z = np.load(GOLDEN)
    frames = mg.frames_of(dict(zip(z["frame_ids"].tolist(), z["seeds"].tolist())))
    assert mg.covers(frames, [str(s) for s in z["dets"]])
    K = [z["K_%d" % i] for i in z["frame_ids"].tolist()]
    assert all(k[0, 0] != k[1, 1] for k in K)
    assert all(not np.allclose(z["Rtilt_%d" % i], np.eye(3)) for i in z["frame_ids"].tolist())
    assert "lamp" in " ".join(str(s) for s in z["labels_1"]) and sx.CAP == 2048


def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def test_numpy_dot_accumulates_as_dot_fma():
    """The device projection restates each np.dot as the first product rounded, then one FMA per further term
    (dot_fma of csrc/input_builder.cuh); numpy's float64 dot of these shapes does exactly that."""
    from frustum_convnet_b200 import sunrgbd_extract as sx
    z, points, calibs, labels, dets = scenes()
    pc = points[1][:400]
    R, K = calibs[1]["Rtilt"], calibs[1]["K"]
    d = np.transpose(np.dot(np.transpose(R), np.transpose(pc[:, 0:3])))
    cam = sx.flip_axis_to_camera(d)
    uvw = np.dot(cam, np.transpose(K))
    p = pc[:, :3].astype(np.float64)
    for i in range(len(pc)):
        for k in range(3):
            want = _fma(R[2, k], p[i, 2], _fma(R[1, k], p[i, 1], float(Fraction(R[0, k]) * Fraction(p[i, 0]))))
            assert d[i, k] == want
            want = _fma(cam[i, 2], K[k, 2], _fma(cam[i, 1], K[k, 1], float(Fraction(cam[i, 0]) * Fraction(K[k, 0]))))
            assert uvw[i, k] == want
    uv = sx.project_upright_depth_to_image(pc, R, K)
    assert np.array_equal(uv[:, 0], uvw[:, 0] / uvw[:, 2]) and np.array_equal(uv[:, 1], uvw[:, 1] / uvw[:, 2])


def test_errors_are_raised():
    from frustum_convnet_b200 import sunrgbd_extract as sx
    with pytest.raises(ValueError, match="3 x 3"):
        sx.calib_mats({"Rtilt": np.eye(3), "K": np.eye(4)})
    with pytest.raises(ValueError, match="3 x 3"):
        sx.calib_mats({"Rtilt": np.full((3, 3), np.nan), "K": np.eye(3)})
    with pytest.raises(RuntimeError):
        sx.SunrgbdFrustumExtractor(device="cpu")


def test_cabi_rejects_bad_arguments():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    a = _lib.SunrgbdExtractArgs()
    names = ("fcn_sunrgbd_extract_project", "fcn_sunrgbd_extract_count", "fcn_sunrgbd_extract_select",
             "fcn_sunrgbd_extract_write")
    for name in names:
        assert getattr(lib, name)(None, None) == -1
        assert getattr(lib, name)(ctypes.byref(a), None) == 0            # zero frames: nothing to do
    assert lib.fcn_sunrgbd_extract_workspace_bytes(None) == -1
    assert lib.fcn_sunrgbd_extract_workspace_bytes(ctypes.byref(a)) == 0
    a.num_frames, a.num_jobs = 1, 1
    assert lib.fcn_sunrgbd_extract_count(ctypes.byref(a), None) == -1     # NULL device pointers
    a.scan_offsets = a.frames = a.jobs = 256
    assert lib.fcn_sunrgbd_extract_workspace_bytes(ctypes.byref(a)) == -1  # NULL host offsets
    assert b"host_scan_offsets" in lib.fcn_last_error()
    so = np.array([0, 3], np.int32)
    a.host_scan_offsets = so.ctypes.data
    assert lib.fcn_sunrgbd_extract_workspace_bytes(ctypes.byref(a)) == -1  # offsets end past num_points
    assert b"scan offsets" in lib.fcn_last_error()
    a.num_points, a.scans = 3, 2
    assert lib.fcn_sunrgbd_extract_workspace_bytes(ctypes.byref(a)) == -1  # scans not float-aligned
    assert b"aligned" in lib.fcn_last_error()
    a.scans = 256
    a.labelled = 1
    assert lib.fcn_sunrgbd_extract_workspace_bytes(ctypes.byref(a)) == -1  # labelled without label boxes
    a.labelled = 2
    assert lib.fcn_sunrgbd_extract_workspace_bytes(ctypes.byref(a)) == -1
    assert b"labelled" in lib.fcn_last_error()
    a.labelled, a.num_choices = 0, 2
    assert lib.fcn_sunrgbd_extract_workspace_bytes(ctypes.byref(a)) == -1  # more draws than jobs
    a.num_choices, a.num_labels = 0, -1
    assert lib.fcn_sunrgbd_extract_count(ctypes.byref(a), None) == -1


class FakeTensor:
    def __init__(self, a):
        self.a = a

    def cpu(self):
        return self

    def numpy(self):
        return self.a


@pytest.mark.parametrize("part", ["train", "det"])
def test_to_pickle_round_trip(part, tmp_path):
    """to_pickle writes the reference's dict (its keys, bool labels): reading it back as provider_sample_sunrgbd does
    gives the fixture's lists."""
    import pickle
    from frustum_convnet_b200 import sunrgbd_extract as sx
    z, *sc = scenes()
    d, _ = oracle_part(part, z, *sc, np.random.RandomState(int(z["seed"])))
    names = dict(sx.GT_KEYS if part == "train" else sx.DET_KEYS)
    lists = {n: d[k] for k, n in names.items() if n is not None}
    fr = sx.SunrgbdFrustums(FakeTensor(np.concatenate(d["input"])), None,
                            FakeTensor(np.concatenate(d["label"]).astype(np.uint8)) if "label" in d else None,
                            np.array([len(p) for p in d["input"]]), np.arange(len(d["id"])), lists)
    p = tmp_path / "f.pickle"
    fr.to_pickle(str(p))
    with open(p, "rb") as f:
        back = pickle.load(f)
    assert list(back) == [k for k, _ in (sx.GT_KEYS if part == "train" else sx.DET_KEYS)]
    check_dict(z, part, back)
