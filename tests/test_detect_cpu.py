"""CPU: the numpy restatement of the per-image detection step (oracle/detect.py) reproduces what the reference's own
``test()`` handed to ``write_detection_results`` (tests/golden/detect_*.npz, oracle/make_golden_detect.py), and the
C ABI of section (10) validates its arguments without a GPU."""
import ctypes
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR


def load_fixture(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, "detect_%s.npz" % name)))


def fixture_runs(g):
    """-> [(method, use_ref, use_rgb, {(idx, cls): rows})] with the dict order kept."""
    out = []
    for r, spec in enumerate(g["runs"]):
        method, use_ref, use_rgb = str(spec).split(",")
        rows, pos, res = g["run%d_rows" % r], 0, {}
        for i, c, n in zip(g["run%d_key_idx" % r], g["run%d_key_cls" % r], g["run%d_counts" % r]):
            res[(int(i), str(c))] = rows[pos: pos + n]
            pos += n
        out.append((method, use_ref == "1", use_rgb == "1", res))
    return out


def oracle_result(g, dataset, method, use_ref, use_rgb, trace=None):
    from oracle import detect as od
    from oracle.make_golden_detect import batches
    det = od.collect(batches(g, use_ref, use_rgb), [int(i) for i in g["id_list"]], [str(t) for t in g["type_list"]],
                     list(g["box2d"]), dataset, method, trace=trace)
    res, keeps = od.nms_results(det, float(g["thresh"]), dataset, method)
    return {(i, c): res[i][c] for i in res for c in res[i]}, keeps


@pytest.mark.parametrize("name,dataset", [("kitti", "KITTI"), ("sunrgbd", "SUNRGBD")])
def test_oracle_reproduces_the_reference_test_loop(name, dataset):
    g = load_fixture(name)
    for method, use_ref, use_rgb, want in fixture_runs(g):
        got, _ = oracle_result(g, dataset, method, use_ref, use_rgb)
        assert list(got) == list(want), (method, use_ref, use_rgb)           # dict order, zero-row lists included
        for k in want:
            assert got[k].shape == want[k].reshape(-1, 12).shape, k
            np.testing.assert_allclose(got[k], want[k].reshape(-1, 12), rtol=1e-6, atol=1e-6, err_msg=str(k))


def test_fixture_covers_the_cases():
    """The cases the device path is checked on exist in the fixtures."""
    for name, dataset in (("kitti", "KITTI"), ("sunrgbd", "SUNRGBD")):
        g = load_fixture(name)
        runs = fixture_runs(g)
        assert {r[0] for r in runs} == {"nms", "top"} and {r[1] for r in runs} == {True, False}
        assert {r[2] for r in runs} == {True, False}
        nms = runs[0][3]
        assert any(len(v) == 0 for v in nms.values())                      # a list whose rows were all dropped
        assert max(len(v) for v in nms.values()) == 300                     # top_k truncation
        assert len({c for _, c in nms}) == 3
        trace = []
        _, keeps = oracle_result(g, dataset, "nms", True, True, trace)
        assert max(len(k) for k in keeps.values()) == 300
        per_list = {}
        for f, t, kept in trace:
            key = (int(g["id_list"][f]), str(g["type_list"][f]))
            per_list[key] = per_list.get(key, 0) + kept
        assert max(per_list.values()) > 512                                 # a list longer than 512 rows
        assert any(not k for _, _, k in trace)                              # tiny boxes dropped
        p = g["cls_probs"]
        assert (p[..., 0] == p[..., 1]).any()                               # exact ties
        assert ((p[..., 0] >= p[..., 1]).all(1)).any()                      # an all-background frustum
        ids = g["id_list"]
        assert len(np.unique(np.nonzero(ids == 7)[0] // int(g["batch_size"]))) >= 2   # non-adjacent batches


def test_argument_validation_without_gpu():
    from frustum_convnet_b200 import _lib
    assert ctypes.sizeof(_lib.DetRecord) == 48            # the collector's (capacity, 12) int32 record rows
    lib = _lib.load()
    a = _lib.DetCandidateArgs()
    assert lib.fcn_det_candidates(None, None) == -1
    a.B, a.T2, a.NS, a.num_frustums, a.capacity = 2, 0, 3, 4, 10
    assert lib.fcn_det_candidates(ctypes.byref(a), None) == -1 and b"T2" in lib.fcn_last_error()
    a.T2, a.dataset = 140, 2
    assert lib.fcn_det_candidates(ctypes.byref(a), None) == -1 and b"dataset" in lib.fcn_last_error()
    a.dataset, a.method = 0, 5
    assert lib.fcn_det_candidates(ctypes.byref(a), None) == -1 and b"method" in lib.fcn_last_error()
    a.method, a.first = 0, 3
    assert lib.fcn_det_candidates(ctypes.byref(a), None) == -1 and b"segment table" in lib.fcn_last_error()
    a.first = 0
    assert lib.fcn_det_candidates(ctypes.byref(a), None) == -1 and b"NULL" in lib.fcn_last_error()
    a.B = 0
    assert lib.fcn_det_candidates(ctypes.byref(a), None) == 0                 # empty batch: nothing to launch
    assert lib.fcn_det_workspace_bytes(-1, 3) == -1
    f = _lib.DetFinalizeArgs()
    f.num_segments, f.capacity, f.top_k = 3, 10, 0
    assert lib.fcn_det_prepare(ctypes.byref(f), None) == -1 and b"top_k" in lib.fcn_last_error()
    f.top_k = 300
    assert lib.fcn_det_prepare(ctypes.byref(f), None) == -1 and b"NULL" in lib.fcn_last_error()
    buf = np.zeros(64, dtype=np.int64)
    for k in ("counter", "info", "seg_offsets", "keep_count", "workspace", "records", "rows", "box2d"):
        setattr(f, k, buf.ctypes.data)
    f.n_counted = 11                                                          # more rows than the capacity
    assert lib.fcn_det_select(ctypes.byref(f), None) == -1
    assert b"capacity >= 11" in lib.fcn_last_error()


def test_collector_rejects_cpu_tensors():
    import torch
    from frustum_convnet_b200.detect import DetectionCollector
    with pytest.raises(RuntimeError):
        DetectionCollector([1], ["Car"], [np.zeros(4)], device="cpu")
