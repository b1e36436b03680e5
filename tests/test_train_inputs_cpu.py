"""CPU: the numpy restatement of the providers' training branches (oracle/train_inputs.py) reproduces what the
reference's own ``__getitem__`` + collate produced (tests/golden/train_inputs_{det,refine}.npz,
oracle/make_golden_train_inputs.py), ``draw_items`` replays the reference's draws, the fixtures cover the cases the
device builder is checked on, and the C ABI of section (11) validates its arguments."""
import ctypes
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR

BAND = 1e-9        # refs this close to a box face may be labelled differently by Delaunay and the half-space test
FLOAT_KEYS = ("point_cloud", "rot_angle", "center_ref1", "center_ref2", "center_ref3", "center_ref4", "box3d_center",
              "box3d_heading", "box3d_size", "one_hot", "ref_center", "rgb_prob")
INT_KEYS = ("seg_label", "size_class")


def load_fixture(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, "train_inputs_%s.npz" % name)))


def fixture_lists(g, prefix=""):
    """The provider's lists as the fixture stores them (inverse of make_golden_train_inputs._store_lists)."""
    counts = g[prefix + "counts"]
    off = np.concatenate([[0], np.cumsum(counts)])
    L = {"input_list": [g[prefix + "points"][off[i]: off[i + 1]] for i in range(len(counts))]}
    for k, v in g.items():
        if not k.startswith(prefix) or k in (prefix + "counts", prefix + "points"):
            continue
        name = k[len(prefix):]
        if name == "label_list":
            L[name] = [v[off[i]: off[i + 1]] for i in range(len(counts))]
        elif name == "calib_list":
            L[name] = [{"P2": p} for p in v]
        elif name == "type_list":
            L[name] = [str(t) for t in v]
        elif name.endswith("_list") and name not in L:
            L[name] = [x if np.ndim(x) else float(x) for x in v]
    return L


def fixture_batches(g):
    """-> [(kind, lists prefix, strides, index, draws, reference batch)]"""
    out = []
    for k in range(int(g["n_batches"])):
        p = "b%d_" % k
        draws = {n: g[p + n] for n in ("choice", "flip_u", "shift_n")}
        ref = {n[len(p) + 4:]: v for n, v in g.items() if n.startswith(p + "ref_")}
        if p + "kind" in g:
            kind, prefix, strides = "refine", str(g[p + "kind"]) + "_", tuple(g["strides"])
        else:
            kind, prefix, strides = "det", "", tuple(g[p + "strides"])
        out.append((kind, prefix, strides, g[p + "index"], draws, ref))
    return out


def oracle_batch(g, kind, prefix, strides, index, draws):
    from oracle import train_inputs as oti
    return oti.build(kind, fixture_lists(g, prefix), index, draws, strides, float(g.get("max_depth", 70.0)),
                     labels=prefix != "rgb_")


def compare(got, ref, margins=None, exact=True):
    """Float keys bit-equal (exact) or within one float32 ulp with >= 99.9 % bit-identical; int keys exact; cls_label
    exact outside the face band.  -> (values compared, values bit-identical)."""
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


@pytest.mark.parametrize("name", ["det", "refine"])
def test_oracle_reproduces_the_reference_providers(name):
    g = load_fixture(name)
    for kind, prefix, strides, index, draws, ref in fixture_batches(g):
        out = oracle_batch(g, kind, prefix, strides, index, draws)
        margins = out.pop("_margins", None)
        assert set(out) == set(ref), (set(out) ^ set(ref))
        compare(out, ref, margins, exact=True)
        if margins is not None:
            band = (np.abs(margins) <= BAND).any(0)
            assert band.sum() == 0, "refs within %g m of a face" % BAND


@pytest.mark.parametrize("name", ["det", "refine"])
def test_padded_columns_repeat_the_edge(name):
    g = load_fixture(name)
    from frustum_convnet_b200.train_inputs import frustum_table
    for kind, prefix, strides, index, draws, ref in fixture_batches(g):
        if kind != "refine":
            continue
        L = fixture_lists(g, prefix)
        labels = prefix == "train_"
        T = frustum_table("refine", strides, 70.0, labels, list(g["classes"]), L["type_list"],
                          **{k: v for k, v in L.items() if k not in ("input_list", "type_list", "label_list")})["T"]
        for s in range(4):
            c = ref["center_ref%d" % (s + 1)]
            for b, i in enumerate(index):
                t = T[i, s]
                assert (c[b, :, t:] == c[b, :, t - 1: t]).all()
                if s == 1 and labels:
                    assert (ref["cls_label"][b, t:] == ref["cls_label"][b, t - 1]).all()


def test_refine_T_is_the_length_of_numpy_arange():
    from frustum_convnet_b200.train_inputs import frustum_table
    g = load_fixture("refine")
    strides = tuple(g["strides"])
    seen = []
    for prefix in ("train_", "rgb_"):
        L = fixture_lists(g, prefix)
        fr = frustum_table("refine", strides, 70.0, prefix == "train_", list(g["classes"]), L["type_list"],
                           **{k: v for k, v in L.items() if k not in ("input_list", "type_list", "label_list")})
        for i, (pb, size) in enumerate(zip(L["pred_box3d_list"], L["pred_box3d_size_list"])):
            w = size[1]
            for s, st in enumerate(strides):
                assert fr["T"][i, s] == len(np.arange(-w / 2, w / 2, st)), (prefix, i, s)
                # numpy's arange fills start + i * ((start + s) - start)
                z = fr["z_start"][i] + np.arange(fr["T"][i, s]) * fr["z_step"][i, s]
                assert np.array_equal(z, np.arange(fr["z_start"][i], -fr["z_start"][i], st))
            seen.append(tuple(fr["T"][i, :4]))
    assert any(len(set(t)) == 4 for t in seen)
    assert len({t[0] for t in seen}) >= 4


def test_draws_replay_the_recorded_reference_draws():
    from frustum_convnet_b200.train_inputs import draw_items
    for name in ("det", "refine"):
        g = load_fixture(name)
        for k, (kind, prefix, strides, index, draws, ref) in enumerate(fixture_batches(g)):
            aug = prefix != "rgb_"
            np.random.seed(int(g["b%d_seed" % k]))
            d = draw_items(g[prefix + "counts"], index, int(g["npoints"]), aug, aug)
            for n in draws:
                assert np.array_equal(d[n], draws[n]), (name, k, n)
            rs = np.random.RandomState(int(g["b%d_seed" % k]))          # a RandomState is the same stream
            assert np.array_equal(draw_items(g[prefix + "counts"], index, int(g["npoints"]), aug, aug, rs)["choice"],
                                  draws["choice"])


def test_fixtures_cover_the_cases():
    g = load_fixture("det")
    counts, N = g["counts"], int(g["npoints"])
    assert 1 in counts and (counts < N).any() and (counts > N).any() and (counts == N).any()
    assert {tuple(g["b%d_strides" % k]) for k in range(int(g["n_batches"]))} == {(0.25, 0.5, 1.0, 2.0),
                                                                                 (0.1, 0.2, 0.4, 0.8)}
    clips = set()
    fallback = near = 0
    for k, (kind, prefix, strides, index, draws, ref) in enumerate(fixture_batches(g)):
        L = fixture_lists(g)
        for b, i in enumerate(index):
            l, w = L["size_list"][i][:2]
            dist = np.sqrt(l ** 2 + w ** 2)
            sh = draws["shift_n"][b] * dist * 0.2
            clips |= {"+d"} if sh > 0.5 * dist else ({"-d"} if sh < -0.5 * dist else set())
            out = oracle_batch(g, kind, prefix, strides, index[b: b + 1], {n: v[b: b + 1] for n, v in draws.items()})
            m = out["_margins"][:, 0]
            fallback += int((m[0] < 0).all())
            near += int((np.abs(m) < 1e-6).any())
            cz = ref["box3d_center"][b, 2]
            clips |= {"0"} if abs(cz) < 1e-5 else ({"max"} if abs(cz - g["max_depth"]) < 1e-5 else set())
        clips |= {"flip"} if (draws["flip_u"] > 0.5).any() else set()
        clips |= {"noflip"} if (draws["flip_u"] <= 0.5).any() else set()
    assert clips == {"+d", "-d", "0", "max", "flip", "noflip"}, clips
    assert fallback >= 1 and near >= 4
    idx0 = g["b0_index"]
    assert len(set(idx0.tolist())) < len(idx0) and not (np.diff(idx0) >= 0).all()      # repeated and unsorted
    r = load_fixture("refine")
    s1 = float(r["strides"][0])
    rclips = set()
    for k, (kind, prefix, strides, index, draws, ref) in enumerate(fixture_batches(r)):
        if prefix != "train_":
            assert "rgb_prob" in ref and "cls_label" not in ref
            continue
        L = fixture_lists(r, prefix)
        for b, i in enumerate(index):
            l, w = L["size_list"][i][:2]
            sh = draws["shift_n"][b] * np.sqrt(l ** 2 + w ** 2) * 0.1
            rclips |= {"+"} if sh > 2 * s1 else ({"-"} if sh < -2 * s1 else set())
        widths = {c: ref[c].shape[-1] for c in ("center_ref1", "center_ref2", "center_ref3", "center_ref4")}
        assert len(widths) == 4
    assert rclips == {"+", "-"}
    assert r["train_points"].dtype == np.float64 and r["rgb_points"].dtype == np.float32
    assert g["points"].dtype == np.float32


def test_argument_validation_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    assert lib.fcn_build_train_inputs(None, None) == -1 and b"NULL" in lib.fcn_last_error()
    a = _lib.TrainInputArgs()
    a.kind, a.labels, a.rtc, a.B, a.N, a.num_scales, a.num_frustums = 7, 1, 1, 2, 512, 4, 3
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == -1 and b"kind" in lib.fcn_last_error()
    a.kind, a.labels = _lib.TRAIN_DET, 0
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == -1 and b"fcn_build_inputs" in lib.fcn_last_error()
    a.kind, a.labels, a.rtc = _lib.TRAIN_REFINE, 1, 0
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == -1 and b"RTC" in lib.fcn_last_error()
    a.rtc, a.extra_feat = 1, 1
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == -1 and b"EXTRA_FEAT" in lib.fcn_last_error()
    a.extra_feat, a.N = 0, 0
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == -1 and b"sizes" in lib.fcn_last_error()
    a.N, a.num_scales = 512, 9
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == -1 and b"num_scales" in lib.fcn_last_error()
    a.num_scales = 4
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == -1 and b"scale" in lib.fcn_last_error()
    buf = np.zeros(64, dtype=np.float32)
    for s in range(4):
        a.stride[s], a.centers[s] = 0.1 * 2 ** s, buf.ctypes.data
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == -1 and b"NULL" in lib.fcn_last_error()
    a.B = 0
    assert lib.fcn_build_train_inputs(ctypes.byref(a), None) == 0           # empty batch: nothing to launch


def test_builder_validates_on_the_host():
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    with pytest.raises(RuntimeError):
        TrainBatchBuilder("det", (0.25, 0.5, 1.0, 2.0), 1024, device="cpu")
    with pytest.raises(ValueError):
        TrainBatchBuilder("refine", (0.1, 0.2, 0.4, 0.8), 512, rtc=False)
    with pytest.raises(ValueError):
        TrainBatchBuilder("refine", (0.1, 0.2, 0.4, 0.8), 512, with_extra_feat=True)
    with pytest.raises(ValueError):
        TrainBatchBuilder("det", (0.25, 0.5, 1.0, 2.0), 1024, labels=False)
    with pytest.raises(ValueError):
        TrainBatchBuilder("sunrgbd", (0.1, 0.2, 0.4, 0.8), 1024)
