"""CPU: the refinement extractor's host side (frustum_convnet_b200/refine_extract.py) and its numpy oracle
(oracle/refine_extract.py) against the reference's own pickles (tests/golden/refine_extract.npz, written by
oracle/make_golden_refine_extract.py), the perturbation replay, the detection records, the C ABI entries' argument
checks (on the host, before any CUDA call), the ctypes struct layout and the pickle round trip.

The inside-box test is a float64 half-space test where the reference triangulates the corners with scipy's Delaunay;
the fixture's scenes keep every point more than BAND = 1e-9 m from every face of every box they test, where the two
cannot disagree."""
import ctypes
import os
import pickle

import numpy as np
import pytest

from conftest import GOLDEN_DIR

GOLDEN = os.path.join(GOLDEN_DIR, "refine_extract.npz")
PARTS = ("gt_train", "gt_val", "matched", "det")


def _scenes():
    from oracle import kitti_refine_synth as krs
    z = np.load(GOLDEN)
    return z, krs.fixture_scenes(z)


def _oracle(part, z, scenes):
    from oracle import kitti_refine_synth as krs
    from oracle import make_golden_refine_extract as mg
    from oracle import refine_extract as orx
    scans, calibs, hws, labels, results = scenes
    kw = mg.MODES[part]
    return orx.extract(kw["mode"], scans, calibs, hws, z["frame_ids"].tolist(), krs.objects(results),
                       krs.objects(labels), mg.WHITELIST, kw.get("remove_diff", False), kw.get("perturb", False),
                       kw.get("augment", 1), np.random.RandomState(int(z["train_seed"])))


def check_lists(z, part, L, points=None, labels=None):
    """L: {list name: list} (the oracle's, or a RefineFrustums' attributes); points / labels default to L's."""
    if points is None:
        points = np.concatenate(L["input_list"]) if L["input_list"] else np.zeros((0, 4), np.float32)
    assert L["id_list"] == z[part + "_id_list"].tolist()
    assert L["type_list"] == z[part + "_type_list"].tolist()
    assert [len(p) for p in L["input_list"]] == z[part + "_counts"].tolist() if "input_list" in L else True
    assert np.asarray(points, np.float32).tobytes() == z[part + "_input_list"].astype(np.float32).tobytes()
    for n in ("frustum_angle_list", "box2d_list", "pred_box3d_list", "pred_box3d_size_list", "pred_box3d_angle_list",
              "box3d_list", "heading_list", "size_list", "prob_list"):
        if part + "_" + n in z.files:
            mine = np.array(L[n], dtype=np.float64).reshape(z[part + "_" + n].shape)
            assert mine.tobytes() == z[part + "_" + n].astype(np.float64).tobytes(), n
    assert np.array([np.asarray(c["P2"]) for c in L["calib_list"]]).reshape(-1, 12).tobytes() == \
        z[part + "_P2"].tobytes()
    if part != "det":
        lab = np.concatenate(L["label_list"]) if labels is None else labels
        assert np.asarray(lab, np.float64).tobytes() == z[part + "_label_list"].astype(np.float64).tobytes()


@pytest.mark.parametrize("part", PARTS)
def test_oracle_reproduces_the_reference_pickle(part):
    z, scenes = _scenes()
    check_lists(z, part, _oracle(part, z, scenes))


def test_fixture_covers_every_rule():
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200 import refine_extract as rx
    from oracle import kitti_refine_synth as krs
    from oracle import refine_extract as orx
    z, (scans, calibs, hws, labels, results) = _scenes()
    ids = z["frame_ids"].tolist()
    assert len(z["gt_train_id_list"]) > 5 * 4 and len(z["gt_val_id_list"]) > 0
    assert len(z["matched_id_list"]) > 0 and len(z["det_id_list"]) > 0
    assert 9 not in z["matched_id_list"].tolist()                     # no whitelisted ground truth
    assert 10 not in z["det_id_list"].tolist()                        # empty result file
    assert any(ln.startswith("car ") for i in ids for ln in z["labels_%d" % i])
    gt, dets = krs.objects(labels), krs.objects(results)
    # training: a perturbed augmentation without a labelled point is dropped
    jobs, _ = rx.job_table(_lib.REFINE_GT, ids, None, gt, ("Car",), perturb=True, augment=5,
                           rng=np.random.RandomState(int(z["train_seed"])))
    assert len(z["gt_train_id_list"]) < len(jobs)
    # detections: a whitelisted line with a 2-D box under 5 px tall (not clipped) is dropped
    assert any(o.type == "Car" and o.ymax - o.ymin < 5 for i in ids for o in dets[i])
    # matched: a detection below the IoU threshold is dropped, one above it is kept
    jobs, gts = rx.job_table(_lib.REFINE_MATCHED, ids, dets, gt, ("Car",), remove_diff=True)
    best = [orx.match_iou(j["box"], [rx.obj_array(o) for o in gts[j["frame"]]]).max() for j in jobs]
    assert min(best) < 0.5 <= max(best)


class _Counting:
    def __init__(self, seed):
        self.rs, self.n = np.random.RandomState(seed), 0

    def random(self):
        self.n += 1
        return self.rs.random()


def test_perturbation_replays_the_reference_chain():
    """Seven draws an attempt in the order l, h, w, cx, cy, cz, angle; the chain restarts per object; the draws of a
    dropped augmentation are consumed all the same (the fixture's gt_train pins the resulting boxes)."""
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200 import refine_extract as rx
    from oracle import kitti_refine_synth as krs
    z, (scans, calibs, hws, labels, results) = _scenes()
    rng = _Counting(3)
    jobs, gts = rx.job_table(_lib.REFINE_GT, z["frame_ids"].tolist(), None, krs.objects(labels), ("Car",),
                             perturb=True, augment=5, rng=rng)
    n_obj = sum(len(v) for v in gts.values())
    assert len(jobs) == 5 * n_obj and rng.n == 7 * 5 * n_obj            # no retry at these sizes
    rs = np.random.RandomState(3)
    a = rx.obj_array(jobs[0]["obj"])
    enl = a.copy()
    enl[3:6] *= rx.RATIO
    u = rs.random(7)
    expect = np.array([enl[0] + enl[3] * 0.05 * (u[3] * 2 - 1), enl[1] + enl[5] * 0.05 * (u[4] * 2 - 1),
                       enl[2] + enl[4] * 0.05 * (u[5] * 2 - 1), enl[3] + enl[3] * 0.05 * (u[0] * 2 - 1),
                       enl[4] + enl[4] * 0.05 * (u[2] * 2 - 1), enl[5] + enl[5] * 0.05 * (u[1] * 2 - 1),
                       ((enl[6] + np.pi) + 0.05 * (u[6] * 2 - 1) * np.pi) % (2 * np.pi) - np.pi])
    assert jobs[0]["cut"].tobytes() == expect.tobytes()
    # a chain: the second augmentation perturbs the first one's box
    assert not np.array_equal(jobs[1]["cut"], jobs[0]["cut"])


def test_perturbation_retries_non_positive_extents():
    from frustum_convnet_b200 import refine_extract as rx

    class Seq:
        def __init__(self, v):
            self.v, self.i = v, 0

        def random(self):
            self.i += 1
            return self.v[self.i - 1]

    # r = 25 makes l1 = l + 25 l (2u - 1) <= 0 for u = 0: the first attempt is drawn again
    s = Seq([0.0] + [0.5] * 6 + [0.5] * 7)
    b = rx.random_shift_rotate_box3d(np.array([1.0, 2.0, 3.0, 4.0, 2.0, 1.5, 0.5]), 25.0, s)
    assert s.i == 14 and b[3] == 4.0


def test_detection_records_equal_parsed_result_text():
    """objects_from_detections gives what Object3d reads back from write_detection_results' text."""
    from frustum_convnet_b200 import refine_extract as rx
    from frustum_convnet_b200.kitti_eval import compute_alpha
    rng = np.random.default_rng(5)
    dets = {7: {"Car": rng.normal(0, 10, (4, 12)).astype(np.float32),
                "Pedestrian": rng.normal(0, 10, (2, 12)).astype(np.float32)}}
    for rows in dets[7].values():
        rows[:, 7:10] = np.abs(rows[:, 7:10]) + 0.5
    got = rx.objects_from_detections(dets)[7]
    lines = []
    for cls, rows in dets[7].items():
        for r in rows:
            alpha = compute_alpha(r[4], r[6], r[10])
            s = cls + " -1 -1 " + "%.4f " % alpha + "%.4f %.4f %.4f %.4f " % tuple(r[:4])
            s += "%.4f %.4f %.4f %.4f %.4f %.4f %.4f %f" % (r[7], r[8], r[9], r[4], r[5], r[6], r[10], r[11])
            lines.append(rx.KittiObject.parse(s))
    assert len(got) == len(lines)
    for a, b in zip(got, lines):
        assert (a.type, a.truncation, a.occlusion, a.alpha, a.h, a.w, a.l, a.t, a.ry, a.score) == \
            (b.type, b.truncation, b.occlusion, b.alpha, b.h, b.w, b.l, b.t, b.ry, b.score)
        assert a.box2d.tobytes() == b.box2d.tobytes()


def test_read_result_dir(tmp_path):
    from frustum_convnet_b200 import refine_extract as rx
    (tmp_path / "000003.txt").write_text("Car -1 -1 0.1 1 2 30 40 1.5 1.6 3.9 1 1.6 20 0.2 0.9\n")
    (tmp_path / "000004.txt").write_text("")
    d = rx.read_result_dir(str(tmp_path), [3, 4])
    assert len(d[3]) == 1 and d[4] == [] and d[3][0].score == 0.9 and d[3][0].t == (1.0, 1.6, 20.0)
    with pytest.raises(FileNotFoundError):
        rx.read_result_dir(str(tmp_path), [5])


def test_whitelist_is_exact_case_and_non_positive_extent_raises():
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200 import refine_extract as rx
    o = [rx.KittiObject.parse("car 0 0 0 1 2 30 40 1.5 1.6 3.9 1 1.6 20 0.2", "a:1"),
         rx.KittiObject.parse("Car 0 0 0 1 2 30 40 1.5 1.6 3.9 1 1.6 20 0.2", "a:2")]
    jobs, _ = rx.job_table(_lib.REFINE_GT, [0], None, {0: o}, ("Car",))
    assert [j["obj"].line for j in jobs] == ["a:2"]
    bad = [rx.KittiObject.parse("Car 0 0 0 1 2 30 40 1.5 0 3.9 1 1.6 20 0.2", "b:1")]
    with pytest.raises(ValueError, match="b:1"):
        rx.job_table(_lib.REFINE_DET, [0], {0: bad}, None, ("Car",))


def test_cabi_rejects_bad_arguments():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    a = _lib.RefineExtractArgs()
    assert lib.fcn_refine_extract_count(None, None) == -1
    assert lib.fcn_refine_extract_workspace_bytes(None) == -1
    assert lib.fcn_refine_extract_count(ctypes.byref(a), None) == 0           # zero frames: nothing to do
    assert lib.fcn_refine_extract_write(ctypes.byref(a), None) == 0
    assert lib.fcn_refine_extract_workspace_bytes(ctypes.byref(a)) == 0
    a.mode = 3
    assert lib.fcn_refine_extract_count(ctypes.byref(a), None) == -1
    a.mode, a.num_frames, a.num_jobs = _lib.REFINE_DET, 1, 1
    assert lib.fcn_refine_extract_count(ctypes.byref(a), None) == -1          # NULL host offsets
    so = np.array([0, 0], np.int32)
    a.host_scan_offsets = so.ctypes.data
    assert lib.fcn_refine_extract_count(ctypes.byref(a), None) == -1          # NULL device pointers
    a.mode = _lib.REFINE_MATCHED
    assert lib.fcn_refine_extract_workspace_bytes(ctypes.byref(a)) == -1
    a.num_jobs = -1
    assert lib.fcn_refine_extract_count(ctypes.byref(a), None) == -1


class _FakeTensor:
    def __init__(self, a):
        self.a = a

    def cpu(self):
        return self

    def numpy(self):
        return self.a


@pytest.mark.parametrize("part", ["gt_val", "det"])
def test_to_pickle_round_trip(part, tmp_path):
    """to_pickle writes the reference function's lists in its order: reading them back as the reference's provider
    does (provider_sample_refine.py:85-117) gives the fixture's lists."""
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200 import refine_extract as rx
    z, scenes = _scenes()
    L = _oracle(part, z, scenes)
    pts = np.concatenate(L["input_list"])
    mode = _lib.REFINE_DET if part == "det" else _lib.REFINE_GT
    lab = None if part == "det" else _FakeTensor(np.concatenate(L["label_list"]).astype(np.uint8))
    fr = rx.RefineFrustums(mode, _FakeTensor(pts), None, lab, np.array([len(p) for p in L["input_list"]]),
                           np.arange(len(L["id_list"])), {n: v for n, v in L.items() if n not in ("input_list",
                                                                                                  "label_list")})
    p = tmp_path / "f.pickle"
    fr.to_pickle(str(p))
    names = rx._DET_NAMES if part == "det" else rx._GT_NAMES
    with open(p, "rb") as f:
        back = {n: pickle.load(f) for n in names}
    check_lists(z, part, back)
