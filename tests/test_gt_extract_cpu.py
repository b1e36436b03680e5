"""CPU: the first-stage ground-truth extractor's host side (frustum_convnet_b200/gt_extract.py) and its numpy oracle
(oracle/gt_extract.py) against the reference's own pickles (tests/golden/gt_extract.npz, written by
oracle/make_golden_gt_extract.py), the random_shift_box2d replay, the errors, the C ABI entries' argument checks (on
the host, before any CUDA call), the ctypes struct layout and the pickle round trip.

The label test is a float64 half-space test where the reference triangulates the corners with scipy's Delaunay; the
fixture's scenes keep every point more than 1e-9 m from every face of every whitelisted box, where the two cannot
disagree."""
import ctypes
import os
import pickle

import numpy as np
import pytest

from conftest import GOLDEN_DIR

GOLDEN = os.path.join(GOLDEN_DIR, "gt_extract.npz")
PARTS = ("car_train", "car_val", "car_matched", "people_train", "people_val", "people_matched")


def scenes():
    from oracle import kitti_refine_synth as krs
    z = np.load(GOLDEN)
    ids = z["frame_ids"].tolist()
    scans, calibs, hws = {}, {}, {}
    for idx, seed in zip(ids, z["seeds"].tolist()):
        scans[idx], calibs[idx], hws[idx] = krs.scene(seed)[:3]
    from oracle import kitti_scan_synth as ks
    assert ks.checksum([scans[i] for i in ids]) == str(z["checksum"]), "the scene generator drifted from the fixture"
    labels = {i: [str(s) for s in z["labels_%d" % i]] for i in ids}
    return z, scans, calibs, hws, labels, [str(s) for s in z["dets"]]


def part_args(part):
    """part -> (whitelist, mode, perturb, augment)."""
    from oracle import make_golden_gt_extract as mg
    w, m = part.split("_")
    kw = mg.MODES[m]
    return mg.WHITELISTS[w], kw["mode"], kw.get("perturb", False), kw.get("augment", 1)


def oracle_lists(part, z, scans, calibs, hws, labels, dets):
    from frustum_convnet_b200.frustum_extract import read_rgb_detections
    from oracle import gt_extract as ogx
    from oracle import kitti_refine_synth as krs
    wl, mode, perturb, augment = part_args(part)
    return ogx.extract(mode, scans, calibs, hws, z["frame_ids"].tolist(), krs.objects(labels), wl, perturb, augment,
                       np.random.RandomState(int(z["train_seed"])), read_rgb_detections(dets))


def check_lists(z, part, L, points=None, labels=None):
    """L: {list name: list} (the oracle's, an unpickled file's, or a GtFrustums' attributes)."""
    if points is None:
        points = np.concatenate(L["input_list"]) if L["input_list"] else np.zeros((0, 4), np.float32)
    assert L["id_list"] == z[part + "_id_list"].tolist()
    assert L["type_list"] == z[part + "_type_list"].tolist()
    if "input_list" in L:
        assert [len(p) for p in L["input_list"]] == z[part + "_counts"].tolist()
        assert all(p.dtype == np.float32 for p in L["input_list"])
    assert np.asarray(points).tobytes() == z[part + "_input_list"].astype(np.float32).tobytes()
    for n in ("box2d_list", "box3d_list", "heading_list", "size_list", "frustum_angle_list", "gt_box2d_list"):
        mine = np.array(L[n], dtype=np.float64).reshape(z[part + "_" + n].shape)
        assert mine.tobytes() == z[part + "_" + n].astype(np.float64).tobytes(), n
    assert np.array([np.asarray(c["P2"]) for c in L["calib_list"]]).reshape(-1, 12).tobytes() == \
        z[part + "_P2"].tobytes()
    lab = np.concatenate(L["label_list"]) if labels is None else labels
    assert np.asarray(lab, np.float64).tobytes() == z[part + "_label_list"].astype(np.float64).tobytes()


@pytest.mark.parametrize("part", PARTS)
def test_oracle_reproduces_the_reference_pickle(part):
    z, *sc = scenes()
    L = oracle_lists(part, z, *sc)
    assert len(L["id_list"]) > 0
    check_lists(z, part, L)


class Counting:
    """np.random stand-in that counts its random() draws."""

    def __init__(self, seed):
        self.rs, self.n = np.random.RandomState(seed), 0

    def random(self):
        self.n += 1
        return self.rs.random()


def test_fixture_covers_every_rule():
    from frustum_convnet_b200 import gt_extract as gx
    from frustum_convnet_b200.frustum_extract import read_rgb_detections
    from oracle import kitti_refine_synth as krs
    z, scans, calibs, hws, labels, dets = scenes()
    ids, gt = z["frame_ids"].tolist(), krs.objects(labels)
    car = [o for i in ids for o in gt[i] if o.type == "Car"]
    # a Car under 25 px tall: its jobs are dropped on the host, in every mode
    small = [o for o in car if o.box2d[3] - o.box2d[1] < gx.MIN_HEIGHT]
    assert small
    rng = Counting(int(z["train_seed"]))
    jobs = gx.job_table(ids, gt, ("Car",), hws, True, 5, rng)
    assert len(jobs) == 5 * (len(car) - len(small))
    # a box at the image border: some perturbation attempt is drawn again after clipping
    assert rng.n > 4 * 5 * len(car)
    # an augmentation without a labelled point is dropped on the device
    assert len(z["car_train_id_list"]) < len(jobs)
    # matched: frame 9 has no whitelisted Car (skipped), frame 10 no detection; one detection below the threshold
    assert 9 not in z["car_matched_id_list"].tolist() and 10 not in z["car_matched_id_list"].tolist()
    table = gx.detection_table(*read_rgb_detections(dets))
    best = []
    for i in ids:
        g = [o for o in gt[i] if o.type == "Car"]
        for _, t, b in table.get(i, []):
            if t == "Car" and g:
                best.append(gx.bbox_overlaps_2d(b.reshape(-1, 4), np.stack([o.box2d for o in g]))[0].max())
    assert min(best) < 0.5 <= max(best)
    assert any(t.split(" ")[1] == "2" for t in dets) and any(t.split(" ")[1] == "Car" for t in dets)
    for part in PARTS:
        assert len(z[part + "_id_list"]) > 0, part


def test_perturbation_replays_random_shift_box2d():
    """Four draws an attempt in the order cx, cy, h, w; the box clipped to the image and drawn again while degenerate;
    the draws of a box dropped for its height are consumed all the same.  The fixture's car_train box2d_list pins the
    boxes the reference drew."""
    from frustum_convnet_b200 import gt_extract as gx
    from oracle import kitti_refine_synth as krs
    z, scans, calibs, hws, labels, dets = scenes()
    ids, gt = z["frame_ids"].tolist(), krs.objects(labels)
    rng = Counting(4)
    jobs = gx.job_table(ids, gt, ("Car",), hws, True, 5, rng)
    rs = np.random.RandomState(4)
    n_draws, k = 0, 0
    for i in ids:
        H, W = hws[i]
        for o in [o for o in gt[i] if o.type == "Car"]:
            xmin, ymin, xmax, ymax = o.box2d
            w, h, cx, cy = xmax - xmin, ymax - ymin, (xmin + xmax) / 2.0, (ymin + ymax) / 2.0
            for _ in range(5):
                while True:
                    u = rs.random(4)
                    n_draws += 4
                    cx2, cy2 = cx + w * 0.1 * (u[0] * 2 - 1), cy + h * 0.1 * (u[1] * 2 - 1)
                    h2, w2 = h * (1 + u[2] * 2 * 0.1 - 0.1), w * (1 + u[3] * 2 * 0.1 - 0.1)
                    b = np.array([cx2 - w2 / 2.0, cy2 - h2 / 2.0, cx2 + w2 / 2.0, cy2 + h2 / 2.0])
                    b[[0, 2]] = np.clip(b[[0, 2]], 0, W - 1)
                    b[[1, 3]] = np.clip(b[[1, 3]], 0, H - 1)
                    if b[0] < b[2] and b[1] < b[3]:
                        break
                if h >= 25:
                    assert jobs[k]["cut"].tobytes() == b.tobytes() and jobs[k]["obj"] is o
                    k += 1
    assert k == len(jobs) and rng.n == n_draws


def test_errors_are_raised():
    from frustum_convnet_b200 import gt_extract as gx
    from frustum_convnet_b200.refine_extract import KittiObject
    ok = KittiObject.parse("Car 0 0 0 10 20 110 120 1.5 1.6 3.9 1 1.6 20 0.2", "a:1")
    flat = KittiObject.parse("Car 0 0 0 110 20 110 120 1.5 1.6 3.9 1 1.6 20 0.2", "a:2")
    hw = {0: (375, 1242)}
    gx.job_table([0], {0: [ok, flat]}, ("Car",), hw)                       # unperturbed: the reference cuts as given
    with pytest.raises(ValueError, match="a:2"):
        gx.job_table([0], {0: [ok, flat]}, ("Car",), hw, perturb=True, augment=2)
    nan = KittiObject.parse("Car 0 0 0 10 20 nan 120 1.5 1.6 3.9 1 1.6 20 0.2", "a:3")
    with pytest.raises(ValueError, match="a:3"):
        gx.job_table([0], {0: [nan]}, ("Car",), hw)
    gx.job_table([0], {0: [nan]}, ("Pedestrian",), hw)                     # not whitelisted: not read
    zero = KittiObject.parse("Car 0 0 0 10 20 110 120 1.5 0 3.9 1 1.6 20 0.2", "a:4")
    with pytest.raises(ValueError, match="a:4"):
        gx.job_table([0], {0: [zero]}, ("Car",), hw)
    x = gx.GtFrustumExtractor(device="cuda:0")
    with pytest.raises(ValueError, match="same length"):
        x.from_matched_detections({}, {}, hw, [0], [0, 0], ["Car"], [0.9], [np.zeros(4)], {0: [ok]})
    dets = gx.detection_table([0], ["Car"], [0.9], [np.array([10.0, 20.0, np.inf, 120.0])])
    with pytest.raises(ValueError, match="detection line 0"):
        gx.job_table([0], {0: [ok]}, ("Car",), hw, dets=dets, thresh=0.5)
    degenerate = gx.detection_table([0], ["Car"], [0.9], [np.array([10.0, 20.0, 10.0, 120.0])])
    g0 = KittiObject.parse("Car 0 0 0 10 20 10 120 1.5 1.6 3.9 1 1.6 20 0.2", "a:5")
    # bbox_overlaps_2d of two zero-area boxes is NaN, numpy's max: matched, as in the reference; then perturbed
    with pytest.raises(ValueError, match="detection line 0"):
        gx.job_table([0], {0: [g0]}, ("Car",), hw, perturb=True, dets=degenerate, thresh=0.5)
    with pytest.raises(RuntimeError):
        gx.GtFrustumExtractor(device="cpu")


def test_matching_takes_numpys_first_maximum():
    from frustum_convnet_b200 import gt_extract as gx
    from frustum_convnet_b200.refine_extract import KittiObject
    g = [KittiObject.parse("Car 0 0 0 10 20 110 120 1.5 1.6 3.9 1 1.6 20 0.2", "g:1"),
         KittiObject.parse("Car 0 0 0 10 20 110 120 1.5 1.6 3.9 2 1.6 20 0.2", "g:2"),
         KittiObject.parse("Car 0 0 0 300 20 400 120 1.5 1.6 3.9 3 1.6 20 0.2", "g:3")]
    dets = gx.detection_table([0, 0, 0], ["Car", "Pedestrian", "Car"], [0.9, 0.8, 0.7],
                              [np.array([10.0, 20.0, 110.0, 120.0]), np.array([10.0, 20.0, 110.0, 120.0]),
                               np.array([600.0, 20.0, 700.0, 120.0])])
    jobs = gx.job_table([0], {0: g}, ("Car",), {0: (375, 1242)}, dets=dets, thresh=0.5)
    assert [(j["det"], j["obj"].line) for j in jobs] == [(0, "g:1")]


def test_cabi_rejects_bad_arguments():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    a = _lib.GtExtractArgs()
    assert lib.fcn_gt_extract_count(None, None) == -1
    assert lib.fcn_gt_extract_workspace_bytes(None) == -1
    assert lib.fcn_gt_extract_count(ctypes.byref(a), None) == 0               # zero frames: nothing to do
    assert lib.fcn_gt_extract_write(ctypes.byref(a), None) == 0
    assert lib.fcn_gt_extract_workspace_bytes(ctypes.byref(a)) == 0
    a.num_frames, a.num_jobs = 1, 1
    assert lib.fcn_gt_extract_count(ctypes.byref(a), None) == -1              # NULL device pointers
    a.scan_offsets = a.frames = a.jobs = 256
    assert lib.fcn_gt_extract_workspace_bytes(ctypes.byref(a)) == -1          # NULL host offsets
    assert b"host_scan_offsets" in lib.fcn_last_error()
    so = np.array([0, 3], np.int32)
    a.host_scan_offsets = so.ctypes.data
    assert lib.fcn_gt_extract_workspace_bytes(ctypes.byref(a)) == -1          # offsets end past num_points
    assert b"scan offsets" in lib.fcn_last_error()
    a.num_points, a.scans = 3, 8
    assert lib.fcn_gt_extract_workspace_bytes(ctypes.byref(a)) == -1          # scans not 16-byte aligned
    assert b"aligned" in lib.fcn_last_error()
    a.num_labels = -1
    assert lib.fcn_gt_extract_count(ctypes.byref(a), None) == -1


class FakeTensor:
    def __init__(self, a):
        self.a = a

    def cpu(self):
        return self

    def numpy(self):
        return self.a


@pytest.mark.parametrize("part", ["car_train", "people_matched"])
def test_to_pickle_round_trip(part, tmp_path):
    """to_pickle writes the reference function's lists in its order: reading them back as the reference's provider
    does (provider_sample.py:96-108) gives the fixture's lists."""
    from frustum_convnet_b200 import gt_extract as gx
    z, *sc = scenes()
    L = oracle_lists(part, z, *sc)
    fr = gx.GtFrustums(FakeTensor(np.concatenate(L["input_list"])), None,
                       FakeTensor(np.concatenate(L["label_list"]).astype(np.uint8)),
                       np.array([len(p) for p in L["input_list"]]), np.arange(len(L["id_list"])), L)
    p = tmp_path / "f.pickle"
    fr.to_pickle(str(p))
    with open(p, "rb") as f:
        back = {n: pickle.load(f) for n in gx.NAMES}
    check_lists(z, part, back)
