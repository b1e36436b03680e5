"""GPU: the validation kernel (csrc/validate.cu, fcn_val_batch) called directly through its C ABI on the crafted cases
of tests/loss_ref.py, against the float64 reference computed from each call's own inputs, at the edges that
tests/test_gpu_det_loss.py pins for the training loss: head shapes NH/NS from 1/1 to 32/32, every GT heading kind and
every bin boundary +- 1 ulp, 1 to 2^18 rows (one CTA slot to about 2 000 of them), labels with -1, one, no and only
ignored rows, each loss weight 0, focal saturation, exact arg-max and corner ties, flipped-box rows, and the logits in
a pitched buffer whose pad rows and columns hold NaN.

Bars (u = 2^-24), those of test_gpu_det_loss.check_values:
  * losses out[1..7] within test_gpu_det_loss._loss_tol: its ceil(N/128) + 16 additions cover the xor butterfly,
    the four warps in order and the serial sum over the CTA slots;
  * total out[0] bit-equal to loss_ref.total_f32 of the kernel's own out[1..7] and the float32 weights;
  * accuracies out[8..10]: c = rint(out * n) within the ambiguous arg-max rows of the reference's count, the value
    bit-equal to loss_ref.accuracy_f32(c, n);
  * IoU means 1e-4 against oracle/box_iou.py, NaN without IoU;
  * the table row's B, nfg, nkeep and pad exact; every other table row and a NaN guard after the partials keep
    their bits; the state words and fcn_val_finalize's first_no_fg exact.
The cross-check runs fcn_det_loss and fcn_det_loss_deterministic on the dense layout of the same logits: the same
counts, the losses and IoU means within the sum of the two kernels' bounds, and every kernel's total and accuracies
exact as above.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import loss_ref as lr
from test_gpu_det_loss import KEYS, WEIGHTS, Call, _loss_tol, check, check_values, corner_tie_case, near_gt_case

pytestmark = pytest.mark.gpu
SENTINEL = 12345.678
GUARD = 64                        # NaN floats after the partials


def _lib():
    from frustum_convnet_b200 import _lib
    return _lib


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32)


class ValCall:
    """Device buffers of one fcn_val_batch call.  The case's dense logits go to a (B, T2 + pitch_extra, ld) buffer,
    ld = 2 + 3 + 2*NH + 4*NS + ld_extra, whose pad rows and columns hold NaN, so a read of them shows up in a sum.
    The partials are followed by GUARD NaN floats; the table has `capacity` rows of SENTINEL and the row is appended
    at state[0] = `row`."""

    def __init__(self, case, NH, NS, weights=WEIGHTS, with_iou=1, iou_thresh=0.7, pitch_extra=0, ld_extra=0, row=2,
                 capacity=5):
        lib = _lib()
        self.case, self.NH, self.NS, self.weights = case, NH, NS, weights
        self.with_iou, self.iou_thresh, self.row, self.capacity = with_iou, iou_thresh, row, capacity
        B, _, T2 = case["center_ref2"].shape
        self.B, self.T2, self.N = B, T2, B * T2
        W = 3 + 2 * NH + 4 * NS
        ld = 2 + W + ld_extra
        dense = np.concatenate([case["cls"], case["reg"]], 1).reshape(B, T2, 2 + W)
        self.logits = torch.full((B, T2 + pitch_extra, ld), math.nan, device="cuda")
        self.logits[:, :T2, :2 + W] = torch.from_numpy(dense).cuda()
        self.t = {k: torch.from_numpy(np.ascontiguousarray(case[k])).cuda() for k in KEYS if k not in ("cls", "reg")}
        n_part = int(lib.load().fcn_val_partials_floats(B, T2))
        assert n_part == -(-self.N // 128) * 16
        self.partials = torch.full((n_part + GUARD,), math.nan, device="cuda")
        self.table = torch.full((capacity, lib.VAL_ROW), SENTINEL, device="cuda")
        self.state = torch.zeros(4, dtype=torch.int32, device="cuda")
        self.res = torch.zeros(C.sizeof(lib.ValResult), dtype=torch.uint8, device="cuda")
        a = lib.ValBatchArgs()
        a.B, a.T2, a.NH, a.NS, a.with_iou, a.capacity = B, T2, NH, NS, with_iou, capacity
        a.logit_pitch, a.ld_logit = T2 + pitch_extra, ld
        a.logits, a.center_ref2 = self.logits.data_ptr(), self.t["center_ref2"].data_ptr()
        for f in ("cls_label", "size_class", "box3d_center", "box3d_heading", "box3d_size", "mean_size"):
            setattr(a, f, self.t[f].data_ptr())
        a.w_box, a.w_head_reg, a.w_size_reg, a.w_corner = weights
        a.iou_thresh = iou_thresh
        a.partials, a.state, a.table = self.partials.data_ptr(), self.state.data_ptr(), self.table.data_ptr()
        self.args = a

    def run(self):
        """One fcn_val_batch and one fcn_val_finalize; -> (the appended table row, the state words, the result)."""
        lib = _lib()
        s = torch.cuda.current_stream()
        self.state[0] = self.row
        lib.call("fcn_val_batch", C.byref(self.args), s.cuda_stream)
        lib.call("fcn_val_finalize", self.table.data_ptr(), self.capacity, self.state.data_ptr(), self.res.data_ptr(),
                 s.cuda_stream)
        s.synchronize()
        res = lib.ValResult.from_buffer_copy(self.res.cpu().numpy().tobytes())
        return self.table[self.row].cpu().numpy(), self.state.cpu().numpy(), res

    def ref(self):
        return lr.det_loss_ref(*(torch.from_numpy(np.ascontiguousarray(self.case[k])) for k in KEYS), self.weights,
                               self.NH, self.NS, iou_thresh=self.iou_thresh, with_iou=bool(self.with_iou))


def check_val(call, ref=None):
    """Run `call`, check the row, the untouched memory and the state against the reference; -> (row, ref)."""
    from frustum_convnet_b200 import _lib as lib
    ref = ref if ref is not None else call.ref()
    got, state, res = call.run()
    n_amb = check_values(got[:14], ref, call.N, call.weights, call.with_iou, call.iou_thresh)
    assert got[14] == call.B and got[15] == ref.nfg and got[16] == ref.nkeep and got[17] == 0, got[14:]
    others = [r for r in range(call.capacity) if r != call.row]
    assert bool((call.table[others] == SENTINEL).all()), "a table row other than the appended one was written"
    assert torch.equal(_bits(call.partials[-GUARD:]), _bits(torch.full((GUARD,), math.nan))), "partials guard"
    no_fg = ref.nfg == 0
    assert list(state) == [call.row + 1, lib.VAL_NO_FG if no_fg else 0, call.row if no_fg else 0, 0], state
    assert res.added == call.row + 1 and res.rows == min(call.row + 1, call.capacity)
    assert res.status == (lib.VAL_NO_FG if no_fg else 0) and res.first_no_fg == (call.row if no_fg else -1)
    print("rows %d fg %d keep %d | ambiguous arg-max cls/head/size %s" % (call.N, ref.nfg, ref.nkeep, n_amb))
    return got, ref


def _mean_size(NS):
    """The mean sizes of the dataset with NS size classes, or None (make_case draws them)."""
    from frustum_convnet_b200 import config
    for info in config.DATASET_INFO.values():
        if len(info.MEAN_SIZE_ARRAY) == NS:
            return np.asarray(info.MEAN_SIZE_ARRAY, np.float32)
    return None


# ============================================================================ head shapes, headings
@pytest.mark.parametrize("NH,NS", [(12, 1), (12, 3), (12, 8), (12, 10), (9, 8), (1, 1), (32, 32)])
def test_head_shapes(NH, NS):
    """NS = 3 and 10 with the KITTI and SUN-RGBD mean sizes; the others with random ones."""
    case = lr.make_case(6, 53, NH, NS, seed=NH * 100 + NS, mean_size=_mean_size(NS))
    got, ref = check_val(ValCall(case, NH, NS, pitch_extra=NS % 2, ld_extra=NH % 5))
    if NS == 1:
        assert got[5] == 0.0                          # one size cluster: the size cross-entropy is exactly 0
    assert int((~ref.use_g).sum()) > 0 and int(ref.use_g.sum()) > 0, "rows of both boxes"


@pytest.mark.parametrize("NH", [9, 11, 12, 13, 32])
def test_heading_kinds(NH):
    """Every GT heading kind of loss_ref.HEADING_KINDS on a frustum with foreground rows; exact heading arg-max ties
    and flipped-box rows among them."""
    B, T2 = 16, 40
    case = lr.make_case(B, T2, NH, 3, seed=20 + NH)
    _, ref = check_val(ValCall(case, NH, 3, pitch_extra=1))
    with_fg = np.unique(ref.fg_rows.numpy() // T2)
    kinds = lr.heading_kinds(case["box3d_heading"][with_fg], NH)
    assert kinds >= set(lr.HEADING_KINDS) - {"random", "near-pi"}, sorted(kinds)
    hs = case["reg"][ref.fg_rows.numpy(), 3:3 + NH]
    assert ((hs == hs.max(-1, keepdims=True)).sum(-1) > 1).any(), "an exact heading arg-max tie"
    assert (~ref.use_g).any() and ref.use_g.any()


@pytest.mark.parametrize("NH", [9, 11, 12, 13, 32])
def test_heading_bin_boundaries(NH):
    """GT headings on every bin boundary of NH bins and one ulp to each side, every row foreground."""
    B, T2 = 3 * NH, 4
    case = lr.make_case(B, T2, NH, 3, seed=NH)
    rng = np.random.default_rng(NH)
    case["box3d_heading"] = np.array([lr._heading_of_kind(kind, k, NH, rng) for k in range(NH)
                                      for kind in ("boundary", "boundary+ulp", "boundary-ulp")], np.float32)
    case["cls_label"][:] = 1
    _, ref = check_val(ValCall(case, NH, 3, pitch_extra=7))
    assert set(ref.hc.numpy()) == set(range(NH))


# ============================================================================ rows and logit layout
@pytest.mark.parametrize("B,T2", [(1, 1), (1, 127), (1, 128), (3, 43), (1, 257), (32, 280), (32, 700), (512, 511)])
def test_row_counts(B, T2):
    """1 row to 512 x 511 = 261 632 rows, whose 2 044 CTA slots the final sum adds one after the other;
    32 x 700 is the people workload's T2."""
    case = lr.make_case(B, T2, 12, 3, seed=B * 1000 + T2)
    if B * T2 == 1:
        case["cls_label"][:] = 1
    check_val(ValCall(case, 12, 3, pitch_extra=(0, 1, 7)[T2 % 3]))


@pytest.mark.parametrize("pitch_extra", [0, 1, 7])
@pytest.mark.parametrize("ld_extra", [0, 3])
def test_logit_layout(pitch_extra, ld_extra):
    """logit_pitch = T2, T2 + 1, T2 + 7 and ld_logit exact or wider, pads NaN: the same bits in every layout."""
    case = lr.make_case(3, 43, 12, 8, seed=43)
    got, _ = check_val(ValCall(case, 12, 8, pitch_extra=pitch_extra, ld_extra=ld_extra))
    dense = ValCall(case, 12, 8).run()[0]
    assert np.array_equal(got.view(np.int32), dense.view(np.int32))


# ============================================================================ labels, weights, row edges
@pytest.mark.parametrize("labels", ["mixed", "one_fg", "no_fg", "all_ignored"])
def test_labels(labels):
    case = lr.make_case(4, 30, 12, 3, seed=9)
    lab = case["cls_label"]
    assert (lab == -1).any() and (lab == 1).any() and (lab == 0).any()
    if labels == "one_fg":
        lab[lab == 1] = 0
        lab[2, 17] = 1
    elif labels == "no_fg":
        lab[lab == 1] = 0
    elif labels == "all_ignored":
        lab[:] = -1
    call = ValCall(case, 12, 3, pitch_extra=1, row=3)
    got, ref = check_val(call)
    if labels == "one_fg":
        assert ref.nfg == 1
    if labels in ("no_fg", "all_ignored"):
        assert np.isfinite(got[:14]).all() and (got[2:8] == 0).all() and (got[9:14] == 0).all()
        # a second batch without foreground leaves the first one's index in place
        call.row = 4
        again, state, res = call.run()
        assert np.array_equal(again.view(np.int32), got.view(np.int32))
        assert state[2] == 3 and res.first_no_fg == 3 and res.added == 5


@pytest.mark.parametrize("zero", [None, 0, 1, 2, 3])
def test_loss_weights(zero):
    w = list(WEIGHTS)
    if zero is not None:
        w[zero] = 0.0
    check_val(ValCall(lr.make_case(4, 61, 12, 3, seed=77), 12, 3, weights=tuple(w), ld_extra=1))


@pytest.mark.parametrize("gap", [0.0, 30.0, -30.0, 100.0, -100.0])
def test_focal_saturation(gap):
    """pt -> 0 and pt -> 1 on every row with a label (gap 0: pt = 1/2)."""
    case = lr.make_case(2, 64, 12, 3, seed=int(abs(gap)) + 3)
    case["cls"][:, 1] = case["cls"][:, 0] + np.float32(gap)
    _, ref = check_val(ValCall(case, 12, 3, pitch_extra=7))
    keep = case["cls_label"].reshape(-1) != -1
    pt = ref.pt.numpy()[keep]
    if gap == 0.0:
        assert (pt == 0.5).all()
    else:
        assert (pt < 1e-12).any() and (pt > 1 - 1e-12).any()


def test_corner_tie():
    """dg == df exactly: the corner loss of the GT box."""
    case, NH, NS = corner_tie_case()
    _, ref = check_val(ValCall(case, NH, NS, pitch_extra=1, ld_extra=3))
    assert float(ref.dg[0]) == float(ref.df[0]) and bool(ref.use_g[0])


# ============================================================================ IoU
def test_without_iou_gives_nan():
    check_val(ValCall(lr.make_case(3, 33, 12, 3, seed=4), 12, 3, with_iou=0, pitch_extra=1))


def test_iou_near_gt():
    case, NH, NS = near_gt_case()
    got, ref = check_val(ValCall(case, NH, NS, iou_thresh=0.5, pitch_extra=7, ld_extra=3))
    assert 0.2 < float(got[12]) < 0.95 and 0.0 < float(got[13]) < 1.0
    assert (ref.h_arg != ref.hc).any()


# ============================================================================ against the training loss
@pytest.mark.parametrize("B,T2,NH,NS", [(1, 1, 12, 3), (1, 128, 12, 8), (2, 61, 1, 1), (3, 43, 9, 8),
                                        (6, 53, 32, 32), (32, 280, 12, 10)])
def test_agrees_with_the_training_loss(B, T2, NH, NS):
    """fcn_val_batch, fcn_det_loss and fcn_det_loss_deterministic on the same logits (pitched and dense): the same
    counts, losses and IoU means within the sum of two kernels' bounds, each kernel's total and accuracies exact.
    How many of the 14 values are bit-identical within one CTA (N <= 128) is printed, not asserted."""
    from test_gpu_train_deterministic import DetCall
    case = lr.make_case(B, T2, NH, NS, seed=B + T2 + NH + NS)
    if B * T2 == 1:
        case["cls_label"][:] = 1
    val = ValCall(case, NH, NS, pitch_extra=1, ld_extra=2)
    ref = val.ref()
    v, _ = check_val(val, ref)
    N = B * T2
    tol = _loss_tol(ref, N, WEIGHTS)
    den = max(ref.nfg, 1)
    amb_iou = int(ref.amb_h.sum() + ref.amb_s.sum())
    near = int((np.abs(ref.iou[:, 1] - val.iou_thresh) <= 1e-4).sum()) + amb_iou
    for kind in (Call, DetCall):
        call = kind(case, NH, NS)
        out, dcls, dreg = call.run()
        check(call, out, dcls, dreg, ref)
        d = out.cpu().numpy()
        assert d[14] == v[15] and d[15] == v[16]
        diff = np.abs(d[:14].astype(np.float64) - v[:14])
        assert np.all(diff[1:8] <= 2 * tol[1:8]), (kind.__name__, d[:8], v[:8], tol)
        assert np.all(diff[11:13] <= 2 * (1e-4 + amb_iou / den)), (kind.__name__, d[11:14], v[11:14])
        assert diff[13] <= 2 * (near / den + 1e-6), (kind.__name__, d[13], v[13])
        if N <= 128:
            same = int((d[:14].view(np.int32) == v[:14].view(np.int32)).sum())
            print("%s vs fcn_val_batch at %d rows: %d of 14 values bit-identical" % (kind.__name__, N, same))
