"""GPU: the fused detection loss (csrc/loss.cu, fcn_det_loss) through its C ABI against the float64 reference of
tests/loss_ref.py computed from the call's own inputs, at the shapes, weights, labels and branch points where a
hand-derived gradient goes wrong.

Bounds (u = 2^-24; ``mag_*`` are the absolute-value companions of tests/loss_ref.py, float64 magnitudes of the
terms the kernel rounds, each built so that the kernel's error is at most a few u times it):
  * gradients, per element:  |g - g64| <= 16u |g64| + 4u mag.  A row computes its gradient from a handful of
    fp32 operations (expf / logf / sqrtf / cosf / sinf within 2 ulp, products, divisions, sums of at most 32
    softmax terms, the eight corner terms); the companion carries the magnitude of every operand that can cancel
    (1 - pt, (cgt - ref) - ctr, (sgt - ex) / ex - sr, P - G), with its amplification (1 / |P - G| for a corner's
    unit vector, 1 / (pt + 1e-14) for the focal term), the fp32 rounding of the heading label, and that of the two
    angles the kernel computes: the decoded angle and the flipped heading hgt + pi (the GT heading is exact).
    Where a row's gradient terms cancel (a corner gradient summing to ~0 over the eight corners), the bound is
    relative to the terms, not to their small sum;
  * losses: each term is a sum over rows of non-negative values reduced by warp shuffles, shared and global fp32
    atomics in any order (<= 5 + 4 + ceil(N/128) additions on a path): |L - L64| <= u ((ceil(N/128) + 16) L64
    + 4 mag_rows) / n  + 4 ulp(L), n = nfg (num_fg + 1e-14 for the focal term); the total adds its terms with the
    weights and 8u |total|, and is bit-equal to the reference's float32 composition of the kernel's own seven means
    (loss_ref.total_f32: Python's evaluation order, every product and sum rounded on its own);
  * accuracies: the count c = rint(acc * n) exact (first maximum on exact ties), and the value bit-equal to the
    reference's float32 c * float32(1 / n) (loss_ref.accuracy_f32); IoU means 1e-4 against oracle/box_iou.py on the
    same boxes.
A row whose flip choice |dg - df| is within rounding may take either box and must match one of the two float64
gradients; a row whose arg-max has two scores within rounding (not equal) may take either class.  The number of such
rows is printed; the crafted cases keep them rare.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import loss_ref as lr

pytestmark = pytest.mark.gpu
U = lr.U
KEYS = ["cls", "reg", "cls_label", "center_ref2", "box3d_center", "box3d_heading", "box3d_size", "size_class",
        "mean_size"]
WEIGHTS = (2.3, 17.0, 13.0, 5.5)      # distinct, none a power of two: a swapped weight changes the result
SENTINEL = 12345.678


def _lib():
    from frustum_convnet_b200 import _lib
    return _lib


class Call:
    """Device buffers of one fcn_det_loss call: dcls / dreg filled with NaN, one sentinel row past B*T2."""

    def __init__(self, case, NH, NS, weights=WEIGHTS, with_iou=1, iou_thresh=0.7):
        self.case, self.NH, self.NS, self.weights = case, NH, NS, weights
        self.t = {k: torch.from_numpy(np.ascontiguousarray(case[k])).cuda() for k in KEYS}
        B, _, T2 = case["center_ref2"].shape
        self.N, self.W = B * T2, 3 + 2 * NH + 4 * NS
        self.dcls = torch.full((self.N + 1, 2), math.nan, device="cuda")
        self.dreg = torch.full((self.N + 1, self.W), math.nan, device="cuda")
        self.dcls[self.N] = SENTINEL
        self.dreg[self.N] = SENTINEL
        self.out = torch.full((16,), math.nan, device="cuda")
        self.scratch = torch.full((2 + 13,), math.nan, device="cuda")
        a = _lib().LossArgs()
        a.B, a.T2, a.NH, a.NS, a.with_iou = B, T2, NH, NS, with_iou
        for k, f in (("cls", "cls"), ("reg", "reg"), ("center_ref2", "center_ref2"), ("cls_label", "cls_label"),
                     ("size_class", "size_class"), ("box3d_center", "box3d_center"),
                     ("box3d_heading", "box3d_heading"), ("box3d_size", "box3d_size"), ("mean_size", "mean_size")):
            setattr(a, f, self.t[k].data_ptr())
        a.w_box, a.w_head_reg, a.w_size_reg, a.w_corner = weights
        a.iou_thresh = iou_thresh
        a.dcls, a.dreg, a.out, a.scratch = (self.dcls.data_ptr(), self.dreg.data_ptr(), self.out.data_ptr(),
                                            self.scratch.data_ptr())
        self.args = a

    def run(self, stream=None):
        s = stream if stream is not None else torch.cuda.current_stream()
        _lib().call("fcn_det_loss", C.byref(self.args), s.cuda_stream)
        s.synchronize()
        return self.out.clone(), self.dcls[:self.N].clone(), self.dreg[:self.N].clone()

    def ref(self, **kw):
        a = self.args
        return lr.det_loss_ref(*(torch.from_numpy(np.ascontiguousarray(self.case[k])) for k in KEYS), self.weights,
                               self.NH, self.NS, iou_thresh=a.iou_thresh, with_iou=bool(a.with_iou), **kw)


def _ulp(x):
    return np.spacing(np.float32(abs(x))).astype(np.float64)


def _loss_tol(ref, N, weights):
    nb = -(-N // 128)
    L = ref.losses.numpy()
    tol = np.zeros(8)
    den = [ref.nfg + lr.EPS14] + [max(ref.nfg, 1)] * 6
    mag = ref.mag_loss_rows.numpy()
    for k in range(7):
        tol[k + 1] = U * ((nb + 16) * L[k + 1] * den[k] + 4 * mag[k]) / den[k] + 4 * _ulp(L[k + 1])
    w_box, w_hr, w_sr, w_c = weights
    tol[0] = (tol[1] + w_box * (tol[2] + tol[3] + tol[5] + w_hr * tol[4] + w_sr * tol[6] + w_c * tol[7])
              + 8 * U * abs(L[0]) + 4 * _ulp(L[0]))
    return tol


def _grad_within(got, g64, mag, what, rows=None):
    got = got.double().cpu()
    tol = 16 * U * g64.abs() + 4 * U * mag
    err = (got - g64).abs()
    ok = err <= tol
    if rows is not None:
        ok = ok | ~rows[:, None]
    if not bool(ok.all()):
        i = int((~ok).reshape(-1).nonzero()[0])
        r, c = divmod(i, got.shape[1])
        raise AssertionError("%s: %d elements out of bound; first (row %d, col %d): got %r expected %r tol %r" % (
            what, int((~ok).sum()), r, c, float(got[r, c]), float(g64[r, c]), float(tol[r, c])))
    ratio = float((err / tol.clamp(min=1e-300))[ok].max()) if err.numel() else 0.0
    return ratio


def check_values(out, ref, N, weights, with_iou, iou_thresh):
    """A kernel's 14 values of one batch (float32 out[0..13]) against the reference of the same inputs."""
    out = np.asarray(out, np.float32)
    o64 = out.astype(np.float64)
    L = ref.losses.numpy()
    tol = _loss_tol(ref, N, weights)
    bad = np.abs(o64[:8] - L) > tol
    assert not bad.any(), ("losses", o64[:8], L, tol)
    # the total: the reference's float32 composition of the kernel's own means, bit for bit
    total = lr.total_f32(out[1:8], weights)
    assert out[0].view(np.int32) == total.view(np.int32), ("total", out[0], total)
    # accuracies: the reference's float32 correct * (1 / n) of an exact count, and the count exact up to rows whose
    # arg-max is within rounding
    n_amb = [int(ref.amb_cls.sum()), int(ref.amb_h.sum()), int(ref.amb_s.sum())]
    den = [max(ref.nkeep, 1), max(ref.nfg, 1), max(ref.nfg, 1)]
    M = ref.metrics.numpy()
    for k in range(3):
        c, c_ref = np.rint(o64[8 + k] * den[k]), np.rint(M[k] * den[k])
        acc = lr.accuracy_f32(c, den[k])
        assert out[8 + k].view(np.int32) == acc.view(np.int32), ("accuracy", k, out[8 + k], acc)
        assert abs(c - c_ref) <= n_amb[k], ("accuracy", k, c, c_ref, n_amb[k])
    if with_iou:
        amb_iou = int(ref.amb_h.sum() + ref.amb_s.sum())
        assert np.all(np.abs(o64[11:13] - M[3:5]) <= 1e-4 + amb_iou / den[1]), ("IoU", o64[11:14], M[3:])
        near = int((np.abs(ref.iou[:, 1] - iou_thresh) <= 1e-4).sum()) + amb_iou
        assert abs(o64[13] - M[5]) <= near / den[1] + 1e-6, ("IoU >= thresh", o64[13], M[5])
    else:
        assert np.isnan(o64[11:14]).all()
    return n_amb


def check(call, out, dcls, dreg, ref=None):
    """Kernel output of one call vs loss_ref; returns the reference."""
    ref = ref if ref is not None else call.ref()
    out = out.cpu().numpy()
    n_amb = check_values(out[:14], ref, call.N, call.weights, call.args.with_iou, call.args.iou_thresh)
    assert out[14] == ref.nfg and out[15] == ref.nkeep
    # gradients: every row written, each element within its bound
    assert bool(torch.isfinite(dcls).all()) and bool(torch.isfinite(dreg).all()), "a row was not written"
    r1 = _grad_within(dcls, ref.dcls, ref.mag_dcls, "dcls")
    amb = torch.zeros(call.N, dtype=torch.bool)
    amb[ref.fg_rows] = ref.amb_flip
    r2 = _grad_within(dreg, ref.dreg, ref.mag_dreg, "dreg", rows=~amb)
    if bool(amb.any()):
        got = dreg.double().cpu()[amb]
        tol = 16 * U * ref.dreg[amb].abs() + 4 * U * ref.mag_dreg[amb]
        ok_g = ((got - ref.dreg[amb]).abs() <= tol).all(-1)
        ok_f = ((got - ref.dreg_alt[amb]).abs() <= 16 * U * ref.dreg_alt[amb].abs() + 4 * U * ref.mag_dreg[amb]).all(-1)
        assert bool((ok_g | ok_f).all()), "a flip-ambiguous row matches neither box"
    lab = torch.from_numpy(call.case["cls_label"]).reshape(-1)
    assert bool((dcls.cpu()[lab == -1] == 0).all()) and bool((dreg.cpu()[lab != 1] == 0).all())
    assert bool((call.dcls[call.N] == SENTINEL).all()) and bool((call.dreg[call.N] == SENTINEL).all()), "row N written"
    print("rows %d fg %d | ambiguous: flip %d, arg-max cls/head/size %s | worst error/bound dcls %.2f dreg %.2f" % (
        call.N, ref.nfg, int(amb.sum()), n_amb, r1, r2))
    return ref


# ============================================================================ shapes, sizes, weights
@pytest.mark.parametrize("NH,NS", [(12, 1), (12, 3), (12, 10), (32, 32)])
def test_head_shapes(NH, NS):
    call = Call(lr.make_case(6, 53, NH, NS, seed=NH * 100 + NS), NH, NS)
    out, dcls, dreg = call.run()
    ref = check(call, out, dcls, dreg)
    if NS == 1:
        # one size cluster: the size cross-entropy and its gradient are exactly 0
        assert float(out[5]) == 0.0
        assert bool((dreg[:, 3 + 2 * NH] == 0).all())
    assert int((~ref.use_g).sum()) > 0 and int(ref.use_g.sum()) > 0, "rows of both boxes"


@pytest.mark.parametrize("B,T2", [(1, 1), (1, 31), (1, 127), (4, 32), (3, 43), (32, 280)])
def test_row_counts(B, T2):
    case = lr.make_case(B, T2, 12, 3, seed=B * 1000 + T2)
    if B * T2 == 1:
        case["cls_label"][:] = 1                                   # the single row is foreground
    call = Call(case, 12, 3)
    out, dcls, dreg = call.run()
    check(call, out, dcls, dreg)


@pytest.mark.parametrize("zero", [None, 0, 1, 2, 3])
def test_loss_weights(zero):
    w = list(WEIGHTS)
    if zero is not None:
        w[zero] = 0.0
    call = Call(lr.make_case(4, 61, 12, 3, seed=77), 12, 3, weights=tuple(w))
    out, dcls, dreg = call.run()
    check(call, out, dcls, dreg)


# ============================================================================ labels
def test_single_foreground_row():
    case = lr.make_case(3, 40, 12, 10, seed=5)
    lab = case["cls_label"]
    lab[lab == 1] = 0
    lab[2, 17] = 1
    call = Call(case, 12, 10)
    out, dcls, dreg = call.run()
    ref = check(call, out, dcls, dreg)
    assert ref.nfg == 1


@pytest.mark.parametrize("labels", ["no_fg", "all_ignored"])
def test_batch_without_foreground(labels):
    """No foreground row: the reference asserts; the kernel returns defined output.  The focal sum is divided by
    0 + 1e-14 (finite, large), every box term, accuracy over foreground rows and IoU is 0, out[14] == 0, dreg is 0
    everywhere and dcls is the focal gradient scaled by 1e14.  With every row ignored, all outputs are 0."""
    case = lr.make_case(4, 30, 12, 3, seed=9)
    lab = case["cls_label"]
    lab[lab == 1] = 0 if labels == "no_fg" else -1
    if labels == "all_ignored":
        lab[:] = -1
    call = Call(case, 12, 3)
    out, dcls, dreg = call.run()
    o = out.double().cpu().numpy()
    assert o[14] == 0 and o[15] == (0 if labels == "all_ignored" else int((lab != -1).sum()))
    assert np.isfinite(o).all()
    assert (o[2:8] == 0).all() and (o[9:14] == 0).all()
    assert bool((dreg == 0).all()) and bool(torch.isfinite(dcls).all())
    if labels == "all_ignored":
        assert (o[:14] == 0).all() and bool((dcls == 0).all())
    else:
        assert o[1] > 1e12 and o[0] == o[1]
    check(call, out, dcls, dreg)


# ============================================================================ branch points
def corner_tie_case():
    """One foreground row with dg == df exactly: a zero-size predicted box at the centre of a GT box of zero width,
    heading 0 (NH = 12, NS = 1)."""
    case = {"cls": np.array([[0.0, 1.0]], np.float32), "cls_label": np.array([[1]], np.int64),
            "center_ref2": np.zeros((1, 3, 1), np.float32), "box3d_center": np.zeros((1, 3), np.float32),
            "box3d_heading": np.zeros(1, np.float32), "box3d_size": np.array([[2.0, 0.0, 0.5]], np.float32),
            "size_class": np.zeros(1, np.int64), "mean_size": np.array([[1.5, 1.0, 1.0]], np.float32)}
    NH, NS = 12, 1
    reg = np.zeros((1, 3 + 2 * NH + 4 * NS), np.float32)
    reg[0, 3 + 2 * NH + NS:] = -1.0                            # predicted size 0
    case["reg"] = reg
    return case, NH, NS


def test_corner_tie_goes_to_gt_box():
    """dg == df exactly (a zero-size predicted box at the centre of a GT box of zero width, heading 0): the
    whole corner gradient goes to the GT side, so the length residual gets -4 gD / |corner| where torch.min's
    half split would give 0."""
    case, NH, NS = corner_tie_case()
    call = Call(case, NH, NS)
    out, dcls, dreg = call.run()
    ref = check(call, out, dcls, dreg)
    assert float(ref.dg[0]) == float(ref.df[0]) and bool(ref.use_g[0])
    col_l = 3 + 2 * NH + NS
    # corner part of the length gradient: -4 gD / |corner| * mean_size_l with gD = w_box * w_corner / 8
    w_box, _, _, w_c = WEIGHTS
    expect_corner = -4 * (w_box * w_c / 8) / math.sqrt(1.0 + 0.0625) * 1.5
    ref0 = lr.det_loss_ref(*(torch.from_numpy(case[k]) for k in KEYS), WEIGHTS[:3] + (0.0,), NH, NS)
    size_part = float(ref0.dreg[0, col_l])
    assert abs(float(ref.dreg[0, col_l]) - size_part - expect_corner) <= 1e-12 * abs(expect_corner)
    assert abs(float(dreg[0, col_l]) - size_part - expect_corner) <= 1e-5 * abs(expect_corner)


@pytest.mark.parametrize("gap", [0.0, 30.0, -30.0, 100.0, -100.0])
def test_focal_saturation(gap):
    case = lr.make_case(2, 64, 12, 3, seed=int(abs(gap)) + 3)
    case["cls"][:, 1] = case["cls"][:, 0] + np.float32(gap)
    call = Call(case, 12, 3)
    out, dcls, dreg = call.run()
    check(call, out, dcls, dreg)


def test_branch_coverage_of_crafted_case():
    """The crafted inputs reach both sides of every branch point (so the comparisons above are not vacuous)."""
    B, T2 = 16, 40
    case = lr.make_case(B, T2, 12, 3, seed=21)
    call = Call(case, 12, 3)
    out, dcls, dreg = call.run()
    ref = check(call, out, dcls, dreg)
    d_c, d_s, e, D = ref.d_c.numpy(), ref.d_s.numpy(), ref.e_h.numpy(), ref.D.numpy()
    assert (d_c < 3).any() and (d_c > 3).any() and (np.abs(d_c - 3) < 1e-5).any()
    assert (d_s < 1).any() and (d_s > 1).any() and (d_s < 1e-6).any()
    assert (np.abs(e) < 1).any() and (e > 1).any() and (e < -1).any()
    assert (D < 1).any() and (D > 1).any()
    assert (~ref.use_g).any() and ref.use_g.any()
    ang = ref.ang.numpy()
    assert (np.abs(ang - np.pi) < 0.3).any() and (np.abs(ang + np.pi) < 0.3).any()
    pt = ref.pt.numpy()
    assert (pt > 1 - 1e-12).any() and (pt < 1e-12).any() and (pt == 0.5).any()
    hc = ref.hc.numpy()
    assert (hc == 0).any() and (hc == 11).any()
    # every GT heading kind sits on a frustum with foreground rows
    with_fg = np.unique(ref.fg_rows.numpy() // T2)
    kinds = lr.heading_kinds(case["box3d_heading"][with_fg], 12)
    assert kinds >= set(lr.HEADING_KINDS) - {"random", "near-pi"}, sorted(kinds)


@pytest.mark.parametrize("NH", [9, 11, 12, 13, 32])
def test_heading_bin_boundaries(NH):
    """GT headings on every bin boundary of NH bins and one ulp to each side.  The bin width is 2 pi / NH rounded
    once from double, as in the model; float32(2 pi) / NH is 1 ulp off for NH = 9, 11, 13 and moves a quarter of
    these headings into the neighbouring class.  Just above the last boundary, where the model's own class index
    runs past the last bin, the kernel takes the last bin."""
    B, T2 = 3 * NH, 4
    case = lr.make_case(B, T2, NH, 3, seed=NH)
    rng = np.random.default_rng(NH)
    case["box3d_heading"] = np.array([lr._heading_of_kind(kind, k, NH, rng) for k in range(NH)
                                      for kind in ("boundary", "boundary+ulp", "boundary-ulp")], np.float32)
    case["cls_label"][:] = 1
    call = Call(case, NH, 3)
    out, dcls, dreg = call.run()
    ref = check(call, out, dcls, dreg)
    assert set(ref.hc.numpy()) == set(range(NH))


# ============================================================================ metrics
def near_gt_case():
    """6 x 40 rows (NH = 12, NS = 3) whose foreground rows predict boxes near their GT box, with predicted heading
    and size classes that differ from the labels on part of the rows."""
    case = lr.make_case(6, 40, 12, 3, seed=31)
    NH, NS = 12, 3
    rng = np.random.default_rng(1)
    reg, lab = case["reg"], case["cls_label"].reshape(-1)
    hc, hres, _ = lr.angle_encode_f32(torch.from_numpy(case["box3d_heading"]), NH)
    for r in np.nonzero(lab == 1)[0]:
        b, t = divmod(int(r), 40)
        reg[r, :3] = case["box3d_center"][b] - case["center_ref2"][b, :, t] + rng.normal(0, 0.1, 3)
        hs = reg[r, 3:3 + NH]
        k = int(hc[b]) if r % 3 else (int(hc[b]) + 1) % NH
        hs[k] = hs.max() + 2
        reg[r, 3 + NH:3 + 2 * NH] = hres[b] + rng.normal(0, 0.05, NH)
        ss = reg[r, 3 + 2 * NH:3 + 2 * NH + NS]
        ss[int(case["size_class"][b]) if r % 4 else (int(case["size_class"][b]) + 1) % NS] = ss.max() + 2
        ms = case["mean_size"]
        reg[r, 3 + 2 * NH + NS:] = ((case["box3d_size"][b] - ms) / ms).reshape(-1) + rng.normal(0, 0.05, 3 * NS)
    return case, NH, NS


def test_without_iou_gives_nan():
    call = Call(lr.make_case(3, 33, 12, 3, seed=4), 12, 3, with_iou=0)
    out, dcls, dreg = call.run()
    check(call, out, dcls, dreg)


def test_iou_against_oracle_near_gt():
    """Predicted boxes near their GT box (non-trivial IoU) with predicted classes that differ from the labels on
    part of the rows: the IoU metrics use the PREDICTED heading and size classes."""
    case, NH, NS = near_gt_case()
    call = Call(case, NH, NS, iou_thresh=0.5)
    out, dcls, dreg = call.run()
    ref = check(call, out, dcls, dreg)
    assert 0.2 < float(out[12]) < 0.95 and 0.0 < float(out[13]) < 1.0
    assert (ref.h_arg != ref.hc).any() and (ref.s_arg != torch.from_numpy(case["size_class"])[ref.fg_rows // 40]).any()


# ============================================================================ contract
def test_deterministic_gradients_and_scratch_reuse():
    """dcls / dreg do not depend on the fp32 atomics: bit-identical across calls and streams.  The losses do; they
    agree within the reordering bound.  A second call on the same scratch starts from clean accumulators."""
    call = Call(lr.make_case(32, 280, 12, 3, seed=8), 12, 3)
    o1, c1, r1 = call.run()
    o2, c2, r2 = call.run()
    s = torch.cuda.Stream()
    o3, c3, r3 = call.run(s)
    for c, r in ((c2, r2), (c3, r3)):
        assert torch.equal(c.view(torch.int32), c1.view(torch.int32))
        assert torch.equal(r.view(torch.int32), r1.view(torch.int32))
    ref = check(call, o1, c1, r1)
    tol = torch.from_numpy(_loss_tol(ref, call.N, WEIGHTS))
    for o in (o2, o3):
        assert bool(((o[:8].double().cpu() - o1[:8].double().cpu()).abs() <= 2 * tol).all())
        assert torch.equal(o[8:11], o1[8:11]) and torch.equal(o[14:], o1[14:])
