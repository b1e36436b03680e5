"""CPU: the float64 loss reference (tests/loss_ref.py) against the reference's own train branch
(tests/golden/det_loss_edges.npz, oracle/make_golden_det_loss.py), and the argument validation of fcn_det_loss.

Fixture bar: the discrete decisions (heading class, heading residual label, predicted heading and size classes,
accuracies) match exactly; losses and d(total)/d(logits) agree to float32 accuracy: the fixture is the reference's
own float32 arithmetic, so the per-element bound is the one the kernel is held to (tests/test_gpu_det_loss.py),
16u |g64| + 4u mag, and each loss term 64u |L| + 4u mag_rows / n; the total adds the terms' bounds with the loss
weights to its own 64u |total|."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

import loss_ref as lr
from conftest import GOLDEN_DIR

CASES = {"nh12_ns3": (12, 3), "nh12_ns1": (12, 1), "nh12_ns10": (12, 10), "nh32_ns32": (32, 32), "nh9_ns3": (9, 3)}
KEYS = ["cls", "reg", "cls_label", "center_ref2", "box3d_center", "box3d_heading", "box3d_size", "size_class",
        "mean_size"]
U = lr.U


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN_DIR, "det_loss_edges.npz")))


def _ref(g, name, NH, NS):
    c = {k: g["%s/%s" % (name, k)] for k in KEYS}
    return c, lr.det_loss_ref(*(torch.from_numpy(c[k]) for k in KEYS), tuple(g["weights"].astype(np.float64)), NH,
                              NS, iou_thresh=float(g["iou_thresh"]))


@pytest.mark.parametrize("name", list(CASES))
def test_loss_ref_matches_reference_train_branch(golden, name):
    NH, NS = CASES[name]
    g = {k.split("/", 1)[1]: v for k, v in golden.items() if k.startswith(name + "/")}
    c, r = _ref(golden, name, NH, NS)
    # discrete decisions, exactly
    assert np.array_equal(r.hc.numpy(), g["hc"])
    assert np.array_equal(r.hres_lab.numpy().view(np.int32), g["hres_lab"].view(np.int32))
    ok_h, ok_s = ~r.amb_h.numpy(), ~r.amb_s.numpy()
    assert np.array_equal(r.h_arg.numpy()[ok_h], g["h_arg"][ok_h])
    assert np.array_equal(r.s_arg.numpy()[ok_s], g["s_arg"][ok_s])
    M = r.metrics.numpy()
    den = np.array([max(r.nkeep, 1), max(r.nfg, 1), max(r.nfg, 1)])   # the reference scales by 1/n in float32
    assert np.array_equal(np.rint(M[:3] * den), np.rint(g["metrics"][:3].astype(np.float64) * den))
    assert np.all(np.abs(M[3:] - g["metrics"][3:]) <= 1e-5)
    # exact score ties are part of the case, and the reference takes their first maximum
    o = c["reg"][r.fg_rows.numpy()]
    hs = o[:, 3:3 + NH]
    tie = (hs == hs.max(-1, keepdims=True)).sum(-1) > 1
    assert tie.any() and np.array_equal(g["h_arg"][tie], hs[tie].argmax(-1))
    if name == "nh12_ns3":
        # the GT heading edges are on frustums with foreground rows, so the decisions above include them
        B, T2 = c["center_ref2"].shape[0], c["center_ref2"].shape[2]
        with_fg = np.unique(r.fg_rows.numpy() // T2)
        kinds = lr.heading_kinds(c["box3d_heading"][with_fg], NH)
        assert kinds >= set(lr.HEADING_KINDS) - {"random", "near-pi"}, sorted(kinds)
    # values to float32 accuracy
    L = r.losses.numpy()
    n = max(r.nfg, 1)
    den = np.array([n, r.nfg + lr.EPS14] + [n] * 6)
    mag = np.concatenate([[0.0], r.mag_loss_rows.numpy()])
    tol = 64 * U * np.abs(L) + 4 * U * mag / den
    w_box, w_hr, w_sr, w_c = golden["weights"].astype(np.float64)
    tol[0] += tol[1] + w_box * (tol[2] + tol[3] + tol[5] + w_hr * tol[4] + w_sr * tol[6] + w_c * tol[7])
    assert np.all(np.abs(g["losses"] - L) <= tol), (g["losses"], L, tol)
    for nm, got, ref, mag in (("dcls", g["dcls"], r.dcls, r.mag_dcls), ("dreg", g["dreg"], r.dreg, r.mag_dreg)):
        err = (torch.from_numpy(got).double() - ref).abs()
        bound = 16 * U * ref.abs() + 4 * U * mag
        bad = ~(err <= bound)
        assert not bool(bad.any()), (nm, int(bad.sum()), float((err / bound.clamp(min=1e-300)).max()))


def test_corner_tie_sends_the_gradient_to_the_gt_box():
    """dg == df exactly (zero-size predicted box at the centre of a GT box of zero width): the gradient of the
    length residual is the GT box's, -4 gD / |corner| * mean_size_l, where torch.min's half split gives 0."""
    NH, NS = 12, 1
    reg = np.zeros((1, 3 + 2 * NH + 4 * NS), np.float32)
    reg[0, 3 + 2 * NH + NS:] = -1.0
    args = [np.array([[0.0, 1.0]], np.float32), reg, np.array([[1]], np.int64), np.zeros((1, 3, 1), np.float32),
            np.zeros((1, 3), np.float32), np.zeros(1, np.float32), np.array([[2.0, 0.0, 0.5]], np.float32),
            np.zeros(1, np.int64), np.array([[1.5, 1.0, 1.0]], np.float32)]
    t = [torch.from_numpy(a) for a in args]
    w = (2.3, 17.0, 13.0, 5.5)
    r = lr.det_loss_ref(*t, w, NH, NS)
    r0 = lr.det_loss_ref(*t, w[:3] + (0.0,), NH, NS)
    assert float(r.dg[0]) == float(r.df[0]) and bool(r.use_g[0])
    col = 3 + 2 * NH + NS
    corner = float(r.dreg[0, col] - r0.dreg[0, col])
    assert abs(corner - (-4 * w[0] * w[3] / 8 / math.sqrt(1.0625) * 1.5)) <= 1e-12


def test_float32_composition_matches_the_reference_expressions():
    """loss_ref.total_f32 and loss_ref.accuracy_f32, which the GPU tests hold the kernels' total and accuracies to bit
    for bit, against the reference's own expressions evaluated by torch on float32 tensors: the total of
    det_base.py:468-474 on 0-dim tensors with Python-float weights, and get_accuracy's
    correct.float().sum(0, keepdim=True).mul_(1.0 / n), for random means, weights and counts with n up to 4096."""
    rng = np.random.default_rng(17)
    f32 = np.float32
    once = 0
    for i in range(3000):
        means = (10.0 ** rng.uniform(-4, 4, 7)).astype(f32)
        means[rng.random(7) < 0.1] = 0
        weights = [float(w) for w in rng.uniform(0, 30, 4)]
        if i % 5 < 4:
            weights[i % 5] = (0.0, 1.0, 2.0, 20.0)[i // 5 % 4]     # zero, integral and power-of-two weights too
        cls_loss, center_loss, heading_class_loss, heading_res_norm_loss, size_class_loss, size_res_norm_loss, \
            corners_loss = (torch.tensor(m) for m in means)
        BOX_LOSS_WEIGHT, HEAD_REG_WEIGHT, SIZE_REG_WEIGHT, CORNER_LOSS_WEIGHT = weights
        loss = cls_loss + \
            BOX_LOSS_WEIGHT * (center_loss +
                               heading_class_loss + size_class_loss +
                               HEAD_REG_WEIGHT * heading_res_norm_loss +
                               SIZE_REG_WEIGHT * size_res_norm_loss +
                               CORNER_LOSS_WEIGHT * corners_loss)
        assert loss.dtype == torch.float32
        got = lr.total_f32(means, weights)
        assert loss.numpy().view(np.int32) == got.view(np.int32), (i, means, weights, float(loss), got)
        m, (w_box, w_hr, w_sr, w_c) = means.astype(np.float64), weights
        exact = m[0] + w_box * (m[1] + m[2] + m[4] + w_hr * m[3] + w_sr * m[5] + w_c * m[6])
        once += f32(exact) != got
    assert once > 300, once          # a total rounded once (or through FMAs) is not the reference's
    div = 0
    for i in range(3000):
        n = int(rng.integers(1, 4097)) if i >= 3 else (6, 7, 10)[i]
        c = int(rng.integers(0, n + 1)) if i >= 3 else (5, 3, 9)[i]
        correct = torch.zeros(1, n, dtype=torch.bool)
        correct[0, :c] = True
        ref = correct[:1].view(-1).float().sum(0, keepdim=True).mul_(1.0 / n)
        got = lr.accuracy_f32(c, n)
        assert ref.numpy()[0].view(np.int32) == got.view(np.int32), (c, n, float(ref[0]), got)
        div += f32(f32(c) / f32(n)) != got
        if i < 3:
            assert f32(f32(c) / f32(n)) != got, (c, n)      # 5/6, 3/7, 9/10: c / n is not the reference's value
    assert div > 300, div


def test_no_foreground_reference_is_defined():
    c = lr.make_case(3, 20, 12, 3, seed=2)
    c["cls_label"][c["cls_label"] == 1] = 0
    r = lr.det_loss_ref(*(torch.from_numpy(c[k]) for k in KEYS), (2.3, 17.0, 13.0, 5.5), 12, 3)
    assert r.nfg == 0 and bool(torch.isfinite(r.losses).all()) and float(r.losses[1]) > 1e12
    assert bool((r.dreg == 0).all()) and (r.losses[2:] == 0).all()


# ============================================================================ argument validation
def _args(**over):
    from frustum_convnet_b200 import _lib
    a = _lib.LossArgs()
    a.B, a.T2, a.NH, a.NS, a.with_iou = 2, 4, 12, 3, 1
    for f in ("cls", "reg", "center_ref2", "cls_label", "size_class", "box3d_center", "box3d_heading", "box3d_size",
              "mean_size", "dcls", "dreg", "out", "scratch"):
        setattr(a, f, 0x1000)                       # never dereferenced: validation fails first
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("field,value", [("NH", 0), ("NH", 33), ("NS", 0), ("NS", 33), ("B", 0), ("T2", 0)])
def test_bad_sizes_rejected(field, value):
    from frustum_convnet_b200 import _lib
    a = _args(**{field: value})
    assert _lib.load().fcn_det_loss(C.byref(a), None) != 0
    assert "bad sizes" in _lib.load().fcn_last_error().decode()


@pytest.mark.parametrize("field", ["cls", "reg", "center_ref2", "cls_label", "size_class", "box3d_center",
                                   "box3d_heading", "box3d_size", "mean_size", "dcls", "dreg", "out", "scratch"])
def test_null_pointers_rejected(field):
    from frustum_convnet_b200 import _lib
    a = _args(**{field: None})
    assert _lib.load().fcn_det_loss(C.byref(a), None) != 0
    assert "NULL" in _lib.load().fcn_last_error().decode()


def test_null_args_rejected():
    from frustum_convnet_b200 import _lib
    assert _lib.load().fcn_det_loss(None, None) != 0
