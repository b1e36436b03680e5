"""CPU: the SUN-RGBD kind of the training-batch builder (C ABI section 11, FCN_TRAIN_SUNRGBD).  The numpy restatement
(oracle/train_inputs_sunrgbd.py) reproduces what the reference's own provider_sample_sunrgbd ``__getitem__`` +
default_collate produced (tests/golden/train_inputs_sunrgbd.npz, oracle/make_golden_train_inputs_sunrgbd.py),
``draw_items(..., height=True)`` replays the reference's four draws per item, the fixture covers the cases the device
builder is checked on, and the C ABI and the host builder validate the new kind's arguments."""
import ctypes
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR

BAND = 1e-9        # refs this close to a box face may be labelled differently by Delaunay and the half-space test
FLOAT_KEYS = ("point_cloud", "rot_angle", "center_ref1", "center_ref2", "center_ref3", "center_ref4", "center_ref5",
              "box3d_center", "box3d_heading", "box3d_size", "one_hot", "rgb_prob")
SUN = (0.1, 0.2, 0.4, 0.8, 1.6)


def load_fixture():
    return dict(np.load(os.path.join(GOLDEN_DIR, "train_inputs_sunrgbd.npz")))


def fixture_lists(g, labels=True):
    """The provider's lists as the fixture stores them (inverse of make_golden_train_inputs_sunrgbd._store_lists);
    labels=False leaves out what the from_rgb_detection provider does not read."""
    counts = g["counts"]
    off = np.concatenate([[0], np.cumsum(counts)])
    F = len(counts)
    L = {"input_list": [g["points"][off[i]: off[i + 1]] for i in range(F)],
         "type_list": [str(t) for t in g["type_list"]],
         "box2d_list": list(g["box2d_list"]),
         "frustum_angle_list": list(g["frustum_angle_list"]),
         "calib_K_list": list(g["calib_K_list"]), "calib_R_list": list(g["calib_R_list"]),
         "prob_list": [float(p) for p in g["prob_list"]]}
    if labels:
        L["label_list"] = [g["label_list"][off[i]: off[i + 1]] for i in range(F)]
        L["box3d_list"] = list(g["box3d_list"])
        L["heading_list"] = [float(h) for h in g["heading_list"]]
        L["size_list"] = list(g["size_list"])
    return L


def fixture_batches(g):
    """-> [(mode 'train' | 'val' | 'rgb', index, draws, reference batch)]"""
    out = []
    for k in range(int(g["n_batches"])):
        p = "b%d_" % k
        draws = {n: g[p + n] for n in ("choice", "flip_u", "shift_n", "height_u")}
        ref = {n[len(p) + 4:]: v for n, v in g.items() if n.startswith(p + "ref_")}
        out.append((str(g[p + "mode"]), g[p + "index"], draws, ref))
    return out


def oracle_batch(g, mode, index, draws):
    from oracle import train_inputs_sunrgbd as ots
    aug = mode == "train"
    return ots.build("sunrgbd", fixture_lists(g, mode != "rgb"), index, draws, tuple(g["strides"]),
                     float(g["max_depth"]), random_flip=aug, random_shift=aug, labels=mode != "rgb")


def compare(got, ref, margins=None, exact=True):
    """Float keys bit-equal (exact) or within one float32 ulp; int keys exact; cls_label exact outside the face band.
    -> (float values compared, float values bit-identical)."""
    total = same = 0
    for k, r in ref.items():
        if k not in got:
            raise AssertionError("missing key " + k)
        v = np.asarray(got[k])
        assert v.shape == r.shape and v.dtype == r.dtype, (k, v.shape, r.shape, v.dtype, r.dtype)
        if k in FLOAT_KEYS:
            if exact:
                assert np.array_equal(v, r), k
            ulp = np.spacing(np.abs(r).astype(np.float32)).astype(np.float64)
            assert (np.abs(v.astype(np.float64) - r.astype(np.float64)) <= ulp).all(), k
            total, same = total + r.size, same + int((v == r).sum())
        elif k == "cls_label":
            keep = np.ones(r.shape, bool) if margins is None else (np.abs(margins) > BAND).all(0)
            assert np.array_equal(v[keep], r[keep]), k
        else:
            assert np.array_equal(v, r), k
    return total, same


def test_oracle_reproduces_the_reference_provider():
    g = load_fixture()
    for mode, index, draws, ref in fixture_batches(g):
        out = oracle_batch(g, mode, index, draws)
        margins = out.pop("_margins", None)
        assert set(out) == set(ref), (set(out) ^ set(ref))
        assert set(ref) - set(FLOAT_KEYS) <= {"cls_label", "seg_label", "size_class"}
        compare(out, ref, margins, exact=True)
        if margins is not None:
            assert (np.abs(margins) <= BAND).sum() == 0, "refs within %g m of a face" % BAND


def test_draws_replay_the_recorded_reference_draws():
    from frustum_convnet_b200.train_inputs import draw_items
    g = load_fixture()
    N = int(g["npoints"])
    for k, (mode, index, draws, ref) in enumerate(fixture_batches(g)):
        aug = mode == "train"
        np.random.seed(int(g["b%d_seed" % k]))
        d = draw_items(g["counts"], index, N, aug, aug, height=True)
        assert set(d) == set(draws)
        for n in draws:
            assert np.array_equal(d[n], draws[n]), (k, n)
        rs = np.random.RandomState(int(g["b%d_seed" % k]))             # a RandomState is the same stream
        d = draw_items(g["counts"], index, N, aug, aug, rs, height=True)
        for n in draws:
            assert np.array_equal(d[n], draws[n]), (k, n)
    # without height=True the draws (and their keys) are the detection provider's
    np.random.seed(0)
    assert set(draw_items(g["counts"], [1, 2], N, True, True)) == {"choice", "flip_u", "shift_n"}


def test_fixture_covers_the_cases():
    from frustum_convnet_b200.train_inputs import frustum_table
    g = load_fixture()
    counts, N = g["counts"], int(g["npoints"])
    assert N == 2048 and tuple(g["strides"]) == SUN and float(g["max_depth"]) == 8.0
    assert 1 in counts and (counts < N).any() and (counts > N).any() and (counts == N).any()
    assert g["points"].dtype == np.float32 and g["points"].shape[1] == 6
    assert g["box2d_list"].dtype == np.float32 and g["label_list"].dtype == bool
    K, R = g["calib_K_list"], g["calib_R_list"]
    assert (K[:, 0, 0] != K[:, 1, 1]).all()
    assert all(np.abs(r - np.eye(3)).max() > 1e-2 and np.allclose(r @ r.T, np.eye(3)) for r in R)
    b = g["box2d_list"]
    c32 = (b[:, 0] + b[:, 2]) / 2.
    c64 = (b[:, 0].astype(np.float64) + b[:, 2].astype(np.float64)) / 2.
    assert c32.dtype == np.float32 and (c32 != c64).any()
    # the host keeps the float32 centre (the record is float64, the value the float32 one)
    L = fixture_lists(g)
    fr = frustum_table("sunrgbd", SUN, 8.0, True, list(g["classes"]), L["type_list"],
                       **{k: v for k, v in L.items() if k not in ("input_list", "type_list")})
    assert np.array_equal(fr["cx"], c32.astype(np.float64)) and not np.array_equal(fr["cx"], c64)
    assert [list(t[:5]) for t in fr["T"]] == [[80, 40, 20, 10, 5]] * len(counts)
    assert len(set(L["type_list"])) >= 6
    seen, fallback, near = set(), 0, 0
    for mode, index, draws, ref in fixture_batches(g):
        seen.add(mode)
        if mode == "rgb":
            assert "rgb_prob" in ref and "cls_label" not in ref and "seg_label" not in ref
            assert ref["one_hot"].shape == (len(index), 10)
            continue
        if mode == "val":
            assert not draws["flip_u"].any() and not draws["shift_n"].any() and not draws["height_u"].any()
        out = oracle_batch(g, mode, index, draws)
        m = out["_margins"]
        fallback += int((m[0] < 0).all(1).sum())
        near += int((np.abs(m) < 1e-6).any(0).any(1).sum())
        assert ref["cls_label"].shape == (len(index), 40)
        if mode != "train":
            continue
        for b, i in enumerate(index):
            l, w = L["size_list"][i][:2]
            dist = np.sqrt(l ** 2 + w ** 2)
            sh = draws["shift_n"][b] * dist * 0.2
            seen |= {"+d"} if sh > 0.5 * dist else ({"-d"} if sh < -0.5 * dist else set())
            cz = ref["box3d_center"][b, 2]
            seen |= {"0"} if abs(cz) < 1e-5 else ({"max"} if abs(cz - 8.0) < 1e-5 else set())
        seen |= {"flip"} if (draws["flip_u"] > 0.5).any() else set()
        seen |= {"noflip"} if (draws["flip_u"] <= 0.5).any() else set()
        seen |= {"h+"} if (draws["height_u"] > 0.5).any() else set()
        seen |= {"h-"} if (draws["height_u"] < 0.5).any() else set()
    assert seen == {"train", "val", "rgb", "+d", "-d", "0", "max", "flip", "noflip", "h+", "h-"}, seen
    assert fallback >= 1 and near >= 4


def _sun_args(labels=1):
    from frustum_convnet_b200 import _lib
    a = _lib.TrainInputArgs()
    a.kind, a.labels, a.rtc, a.B, a.N, a.num_scales, a.num_frustums = _lib.TRAIN_SUNRGBD, labels, 1, 2, 2048, 5, 3
    a.num_classes, a.max_depth, a.random_flip, a.random_shift = 10, 8.0, labels, labels
    buf = np.zeros(64, dtype=np.float32)
    for s in range(5):
        a.stride[s], a.centers[s] = SUN[s], buf.ctypes.data
    for k in ("points", "point_offsets", "frustums", "index", "choice", "point_cloud", "rot_angle", "seg",
              "cls_label", "box3d_center", "box3d_heading", "box3d_size", "size_class", "seg_label", "flip_u",
              "shift_n", "height_u", "rgb_prob"):
        setattr(a, k, buf.ctypes.data)
    return a, buf


def test_argument_validation_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()

    def rejects(a, what):
        return lib.fcn_build_train_inputs(ctypes.byref(a), None) == -1 and what in lib.fcn_last_error()

    a, buf = _sun_args()
    a.num_scales = 4
    assert rejects(a, b"5 scales")
    a.num_scales, a.max_depth = 5, 0.0
    assert rejects(a, b"max_depth")
    a.max_depth, a.rtc = 8.0, 0
    assert rejects(a, b"RTC")
    a.rtc, a.extra_feat = 1, 1
    assert rejects(a, b"EXTRA_FEAT")
    a.extra_feat, a.labels = 0, 2
    assert rejects(a, b"labels")
    a.labels = 1
    for k, what in (("seg", b"seg"), ("seg_label", b"seg"), ("height_u", b"height_u"), ("shift_n", b"draw"),
                    ("cls_label", b"label")):
        a, buf = _sun_args()
        setattr(a, k, None)
        assert rejects(a, what), k
    a, buf = _sun_args()
    a.random_shift, a.height_u = 0, None                                # no shift: height_u is not read
    a.B = 0
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == 0
    # from_rgb_detection: no labels, no seg, but rgb_prob
    a, buf = _sun_args(labels=0)
    a.rgb_prob = None
    assert rejects(a, b"rgb_prob")
    a.rgb_prob = buf.ctypes.data
    for k in ("seg", "seg_label", "cls_label", "height_u", "flip_u", "shift_n"):
        setattr(a, k, None)
    a.B = 0
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == 0
    # the other kinds' checks still hold for the new kind's neighbours
    a, buf = _sun_args()
    a.kind = 3
    assert rejects(a, b"kind")


def _lists(labels=True):
    return fixture_lists(load_fixture(), labels)


def test_builder_validates_on_the_host():
    from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES, TrainBatchBuilder
    for strides in ((0.1, 0.2, 0.4, 0.8), (0.1, 0.2, 0.4, 0.8, 1.6, 3.2)):
        with pytest.raises(ValueError, match="5 strides"):
            TrainBatchBuilder("sunrgbd", strides, 2048)
    with pytest.raises(RuntimeError):
        TrainBatchBuilder("sunrgbd", SUN, 2048, device="cpu")
    with pytest.raises(ValueError):
        TrainBatchBuilder("sunrgbd", SUN, 2048, with_extra_feat=True)
    # constructing touches no device: the defaults are the SUN-RGBD cfg's
    tb = TrainBatchBuilder("sunrgbd", SUN, 2048)
    assert tb.V == len(SUNRGBD_CLASSES) == 10 and tb.max_depth == 8.0 and tb._has_seg
    assert not TrainBatchBuilder("sunrgbd", SUN, 2048, labels=False)._has_seg
    assert TrainBatchBuilder("det", (0.25, 0.5, 1.0, 2.0), 1024).max_depth == 70.0
    L = _lists()
    for missing in ("calib_K_list", "calib_R_list", "box2d_list", "label_list"):
        tb = TrainBatchBuilder("sunrgbd", SUN, 2048)
        with pytest.raises(ValueError, match=missing):
            tb.set_dataset(L["input_list"], L["type_list"], SUNRGBD_CLASSES,
                           **{k: v for k, v in L.items() if k not in ("input_list", "type_list", missing)})
    R = _lists(labels=False)
    tb = TrainBatchBuilder("sunrgbd", SUN, 2048, labels=False)
    with pytest.raises(ValueError, match="prob_list"):
        tb.set_dataset(R["input_list"], R["type_list"], SUNRGBD_CLASSES,
                       **{k: v for k, v in R.items() if k not in ("input_list", "type_list", "prob_list")})


def test_from_dataset_reads_the_sunrgbd_lists():
    """from_dataset on an object shaped like the SUN-RGBD provider (no category_info): the class list defaults to
    SUN-RGBD's, and the frustum records hold K, Rtilt and the float32 box centre."""
    from frustum_convnet_b200 import train_inputs as ti

    class Provider:
        pass

    g = load_fixture()
    ds = Provider()
    for k, v in fixture_lists(g).items():
        setattr(ds, k, v)
    ds.npoints, ds.random_flip, ds.random_shift, ds.one_hot, ds.from_rgb_detection = 2048, True, True, True, False
    seen = {}

    def set_dataset(self, input_list, type_list, classes, **lists):
        seen.update(classes=classes, **lists)

    orig = ti.TrainBatchBuilder.set_dataset
    ti.TrainBatchBuilder.set_dataset = set_dataset
    try:
        tb = ti.TrainBatchBuilder.from_dataset(ds, "sunrgbd", SUN)
    finally:
        ti.TrainBatchBuilder.set_dataset = orig
    assert seen["classes"] == list(ti.SUNRGBD_CLASSES) and tb.V == 10 and tb.max_depth == 8.0
    assert seen["calib_K_list"] is ds.calib_K_list and seen["calib_R_list"] is ds.calib_R_list
    assert tb.random_flip and tb.random_shift and tb.labels
