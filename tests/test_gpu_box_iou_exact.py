"""GPU: the rotated-box IoU (csrc/box_iou.cuh, rbbox_iou_pair) in each of the five kernels that inline it, against
exact rational arithmetic (tests/iou_exact_ref.py) on boxes with collinear and shared edges.  Every kernel inlines
its own copy of the function and nvcc contracts each copy on its own, so each consumer is checked separately:

  * ``fcn_rbbox_iou_3d_pair``: every pair family of tests/test_box_iou_exact_cpu.py at every scale, both argument
    orders, per pair within that file's bound (K u D (perim_P + perim_Q) / union);
  * ``fcn_det_loss`` and ``fcn_val_batch``: foreground rows whose predicted box slides along its GT box with the
    bit-identical float32 heading and size (heading k * apc with a zero residual, size the class mean with a zero
    residual; the offset is in the centre logits).  The IoU means against the mean of the exact per-row IoU of the
    same float32 boxes: 1e-4, the bar of the existing tests; the kernels build corners with cosf / sinf, a few ulp
    from the float64-built ones, which moves a correct IoU by ~1e-6;
  * ``fcn_rotate_nms_3d`` and ``DetectionCollector``: lists of duplicate detections of one object slid along its
    heading or width, whose exact 3-D IoUs all lie at least 0.02 from the threshold, mixed with unrelated boxes.
    Keep lists equal oracle/nms.py / oracle/detect.py exactly (oracle/box_iou.py is within 1e-9 of exact on these
    families, tests/test_box_iou_exact_cpu.py).
"""
import numpy as np
import pytest
import torch

import iou_exact_ref as ex
import loss_ref as lr
from oracle import box_iou as ob

pytestmark = pytest.mark.gpu

N_PAIRS = 500
SEED = 7
MARGIN = 0.02
F32 = np.float32


# ================================================================================ fcn_rbbox_iou_3d_pair
def test_pair_kernel_within_bound_of_exact_on_every_family():
    from frustum_convnet_b200.box_iou import rbbox_iou_3d_pair
    bad, worst, rows = {}, 0.0, 0
    cs, qs, wants = [], [], []
    for scale in ex.SCALES:
        for name in ex.FAMILIES:
            A, B = ex.family_corners(name, scale, SEED, N_PAIRS)
            want = ex.exact_iou(A, B)
            for tag, (c, q) in (("", (A, B)), (" swapped", (B, A))):
                got = rbbox_iou_3d_pair(torch.from_numpy(c).cuda(), torch.from_numpy(q).cuda()).cpu().numpy()
                got = got.astype(np.float64)
                assert np.isfinite(got).all() and (got >= 0).all() and (got <= 1 + 1e-6).all(), (scale, name, tag)
                b = ex.iou_bound(c, q, want[:, 2])
                err = np.abs(got - want[:, :2])
                n_bad = int((err > b[:, None]).any(1).sum())
                if n_bad:
                    bad["%s/%s%s" % (scale, name, tag)] = (n_bad, float(err.max()))
                with np.errstate(divide="ignore", invalid="ignore"):
                    worst = max(worst, float(np.where(b[:, None] > 0, err / b[:, None], 0.0).max()))
                rows += len(c)
                cs.append(c), qs.append(q), wants.append(want[:, :2])
    print("\nfcn_rbbox_iou_3d_pair: %d pairs, worst fraction of the bound %.3g" % (rows, worst))
    assert not bad, "pairs out of bound (count, max error) per family: %s" % bad
    # the stats of one launch over all pairs follow from the per-pair values
    c, q, want = np.concatenate(cs), np.concatenate(qs), np.concatenate(wants)
    out, (m2, m3, frac) = rbbox_iou_3d_pair(torch.from_numpy(c).cuda(), torch.from_numpy(q).cuda(), iou_thresh=0.5)
    got = out.cpu().numpy().astype(np.float64)
    assert abs(float(m2) - got[:, 0].mean()) <= 1e-5 and abs(float(m3) - got[:, 1].mean()) <= 1e-5
    assert abs(float(m2) - want[:, 0].mean()) <= 1e-4 and abs(float(m3) - want[:, 1].mean()) <= 1e-4
    assert float(frac) == pytest.approx((got[:, 1] >= 0.5).mean(), abs=1e-6)


# ================================================================================ fcn_det_loss / fcn_val_batch
NH = 12
KS = (1, 2, 4, 5)            # bins whose start k * apc is below pi (no wrap) and off the axes


def _slide(rng, cgt, hgt, size):
    """Predicted centre (float64) slid along the heading or the width of the GT box by -1.1 .. 1.1 of that size."""
    L, W = ex._along(np.asarray([hgt], np.float64))
    fr = rng.uniform(-1.1, 1.1)
    return cgt + (L[0] * fr * size[0] if rng.random() < 0.6 else W[0] * fr * size[1])


def _exact_rows(cp, h, s, cgt, hgt, sgt):
    """Exact (BEV, 3-D) IoU of the float32 boxes the kernel decodes, per foreground row."""
    P = ob.box3d_corners(np.asarray(cp, np.float64), np.asarray(h, np.float64), np.asarray(s, np.float64))
    G = ob.box3d_corners(np.asarray(cgt, np.float64), np.asarray(hgt, np.float64), np.asarray(sgt, np.float64))
    return ex.exact_iou(P.astype(F32), G.astype(F32))[:, :2]


def test_det_loss_iou_metrics_on_boxes_slid_along_their_gt_box():
    from test_gpu_det_loss import Call
    NS, B, T2 = 3, 24, 48
    rng = np.random.default_rng(21)
    case = lr.make_case(B, T2, NH, NS, seed=21)
    apc = F32(2 * np.pi / NH)
    kb = rng.choice(KS, B)
    case["box3d_heading"] = (kb.astype(F32) * apc).astype(F32)
    ms, sc = case["mean_size"], case["size_class"]
    case["box3d_size"] = ms[sc].astype(F32)
    case["box3d_center"] = (case["box3d_center"] + F32(20) * rng.normal(0, 1, (B, 3)).astype(F32)).astype(F32)
    case["center_ref2"] = (case["box3d_center"][:, :, None] + rng.normal(0, 1.0, (B, 3, T2))).astype(F32)
    reg, lab = case["reg"], case["cls_label"].reshape(-1)
    fg = np.nonzero(lab == 1)[0]
    cps = []
    for r in fg:
        b, t = divmod(int(r), T2)
        cgt, hgt, sgt = case["box3d_center"][b], case["box3d_heading"][b], case["box3d_size"][b]
        ref = case["center_ref2"][b, :, t]
        ctr = (_slide(rng, cgt.astype(np.float64), float(hgt), sgt) - ref).astype(F32)
        reg[r, :3] = ctr
        reg[r, 3:3 + NH] = 0.0
        reg[r, 3 + kb[b]] = 5.0
        reg[r, 3 + NH:3 + 2 * NH] = 0.0
        reg[r, 3 + 2 * NH:3 + 2 * NH + NS] = 0.0
        reg[r, 3 + 2 * NH + sc[b]] = 5.0
        reg[r, 3 + 2 * NH + NS:] = 0.0
        cps.append(ref + ctr)                                   # float32 sum, as the kernel forms it
    bs = fg // T2
    want = _exact_rows(np.asarray(cps), case["box3d_heading"][bs], case["box3d_size"][bs],
                       case["box3d_center"][bs], case["box3d_heading"][bs], case["box3d_size"][bs])
    out, _, _ = Call(case, NH, NS, iou_thresh=0.5).run()
    out = out.double().cpu().numpy()                            # out[11], out[12]: IoU_2D, IoU_3D means
    assert len(fg) > 200 and 0.2 < want[:, 0].mean() < 0.8
    err = [abs(out[11] - want[:, 0].mean()), abs(out[12] - want[:, 1].mean())]
    print("\nfcn_det_loss: %d rows, |mean IoU error| BEV %.3g 3-D %.3g" % (len(fg), *err))
    assert max(err) <= 1e-4, (out[11:13], want.mean(0))
    near = int((np.abs(want[:, 1] - 0.5) <= 1e-4).sum())
    assert abs(out[13] - (want[:, 1] >= 0.5).mean()) <= near / len(fg) + 1e-6


def test_val_batch_iou_meters_on_boxes_slid_along_their_gt_box():
    from test_gpu_validate import _kitti, _Table
    from test_validate_cpu import make_batch
    _, ms = _kitti()
    NS = len(ms)
    rng = np.random.default_rng(22)
    apc = F32(2 * np.pi / NH)
    tb = _Table()
    expect = []
    for _ in range(3):
        B, T2 = 16, 40
        d = make_batch(rng, B, T2, NH, ms, 3 + 2 * NH + 4 * NS, near=False, neg_rows=True)
        kb = rng.choice(KS, B)
        sc = d["size_class"].reshape(-1)
        d["box3d_heading"] = (kb.astype(F32) * apc).astype(F32).reshape(B, 1)
        d["box3d_size"] = ms[sc].astype(F32)
        d["box3d_center"][:, [0, 2]] += rng.normal(0, 15, (B, 2)).astype(F32)
        d["center_ref2"] = (d["box3d_center"][:, :, None] + rng.normal(0, 1.0, (B, 3, T2))).astype(F32)
        lab = d["cls_label"]
        reg = d["reg"]
        rows = []
        for b in range(B):
            cgt, hgt, sgt = d["box3d_center"][b], d["box3d_heading"][b, 0], d["box3d_size"][b]
            for t in np.nonzero(lab[b] == 1)[0]:
                ref = d["center_ref2"][b, :, t]
                ctr = (_slide(rng, cgt.astype(np.float64), float(hgt), sgt) - ref).astype(F32)
                reg[b, :, t] = 0.0
                reg[b, 0:3, t] = ctr
                reg[b, 3 + kb[b], t] = 5.0
                reg[b, 3 + 2 * NH + sc[b], t] = 5.0
                rows.append((ref + ctr, hgt, sgt, cgt))
        cp, h, s, cg = (np.asarray(x) for x in zip(*rows))
        expect.append(_exact_rows(cp, h, s, cg, h, s).mean(0))
        tb.run(tb.args(d, ms))
    got = tb.rows()[:, 11:13].astype(np.float64)
    err = np.abs(got - np.asarray(expect))
    print("\nfcn_val_batch: |IoU meter error| per batch (BEV, 3-D) max %.3g" % err.max())
    assert err.max() <= 1e-4, (got, expect)


# ================================================================================ fcn_rotate_nms_3d / DetectionCollector
def _det_rows(box):
    ctr, head, size = box
    return np.concatenate([ctr, size, head[:, None]], 1)


def _duplicates(rng, scale, n_dup, n_other):
    """(n, 7) rows [cx, cy, cz, l, w, h, ry] (float32): n_dup copies of one object slid along its heading or its
    width, then n_other unrelated boxes at least 12 m away from it (and from each other)."""
    c, h, s = ex._base(scale, rng, 1)
    L, W = ex._along(h)
    fr = rng.uniform(-0.8, 0.8, n_dup)
    fr[0] = 0.0
    along = np.where((rng.random(n_dup) < 0.6)[:, None], L * s[0, 0], W * s[0, 1])
    dup = _det_rows((c + along * fr[:, None], np.repeat(h, n_dup), np.repeat(s, n_dup, 0)))
    oc, oh, os_ = ex._base(scale, rng, n_other)
    oc[:, 0] = c[0, 0] + 12.0 * (1 + np.arange(n_other))
    other = _det_rows((oc, oh, os_))
    return np.concatenate([dup, other]).astype(F32)


def _clear_of_threshold(rows, thresh):
    """Exact 3-D IoU of every pair whose bounding cubes overlap at least MARGIN from the threshold (float64 corners
    as oracle/nms.py builds them)."""
    from oracle import nms as onms
    c = onms.boxes3d2corners(rows)
    mn, mx = c.min(1), c.max(1)
    for i in range(len(rows)):
        for j in range(i + 1, len(rows)):
            ext = np.minimum(mx[i], mx[j]) - np.maximum(mn[i], mn[j])
            if (ext > 0).all() and abs(ex.exact_pair(c[i], c[j])[1] - thresh) < MARGIN:
                return False
            if abs(ext.min()) < 1e-3:                               # the cube test itself must be unambiguous
                return False
    return True


def _lists(seed, n_lists, thresh):
    rng = np.random.default_rng(seed)
    scales = list(ex.SCALES)
    out = []
    while len(out) < n_lists:
        rows = _duplicates(rng, scales[len(out) % len(scales)], int(rng.integers(4, 9)), int(rng.integers(0, 4)))
        if _clear_of_threshold(rows, thresh):
            out.append(rows)
    return out


@pytest.mark.parametrize("thresh", [0.25, 0.5, 0.7])
def test_nms_keep_lists_on_duplicates_slid_along_their_heading(thresh):
    from frustum_convnet_b200.nms import rotate_nms_3d_batched
    from oracle import nms as onms
    rng = np.random.default_rng(int(thresh * 100))
    lists = _lists(int(thresh * 1000), 150, thresh)
    segs = [np.concatenate([r, rng.permutation(len(r))[:, None].astype(F32) / len(r)], 1) for r in lists]
    off = np.concatenate([[0], np.cumsum([len(s) for s in segs])]).astype(np.int32)
    keep, cnt = rotate_nms_3d_batched(torch.from_numpy(np.concatenate(segs)).cuda(), torch.from_numpy(off), thresh)
    keep, cnt = keep.cpu().numpy(), cnt.cpu().numpy()
    wrong = []
    suppressed = 0
    for s, d in enumerate(segs):
        want = [off[s] + k for k in onms.rotate_nms_3d_cc(d, thresh)]
        suppressed += len(d) - len(want)
        if keep[s, :cnt[s]].tolist() != want:
            wrong.append(s)
    print("\nfcn_rotate_nms_3d thresh %.2f: %d lists, %d boxes suppressed, %d lists wrong" % (
        thresh, len(segs), suppressed, len(wrong)))
    assert suppressed > 100
    assert not wrong, "%d of %d keep lists differ from the oracle: %s" % (len(wrong), len(segs), wrong[:10])


def test_detection_collector_keep_lists_on_duplicates_slid_along_their_heading():
    """One frustum per image, every row foreground, rot_angle 0 and ref_center 0 (the decode then keeps the
    centre and heading bit-exact): the rows of a frustum are one list."""
    from oracle import detect as od
    from test_gpu_detect import _compare, _device, _flat
    thresh = 0.25
    rng = np.random.default_rng(23)
    T2, NS = 12, 8
    lists = _lists(2300, 96, thresh)
    F = len(lists)
    ctr = np.zeros((F, T2, 3), F32)
    head = np.zeros((F, T2), F32)
    size = np.zeros((F, T2, 3), F32)
    p1 = np.full((F, T2), 0.1, F32)                                       # background rows
    for f, rows in enumerate(lists):
        n = min(len(rows), T2)
        ctr[f, :n], size[f, :n], head[f, :n] = rows[:n, 0:3], rows[:n, 3:6], rows[:n, 6]
        ctr[f, :n, 1] -= size[f, :n, 2] / 2                               # KITTI label format adds h / 2 back
        p1[f, :n] = rng.permutation(np.linspace(0.55, 0.95, n)).astype(F32)
        ctr[f, n:] = ctr[f, 0] + F32(500.0)
        size[f, n:] = 1.0
    cls = np.stack([1 - p1, p1], -1).astype(F32)
    outs = [cls, ctr, head, size, np.zeros((F, T2, 12), F32), rng.dirichlet(np.ones(NS), (F, T2)).astype(F32)]
    rot = np.zeros(F, F32)
    ref = np.zeros((F, 3), F32)
    Bt = 8
    bt = [(s, tuple(o[s:s + Bt] for o in outs), rot[s:s + Bt], None, ref[s:s + Bt]) for s in range(0, F, Bt)]
    ids, types = list(range(F)), ["Car"] * F
    box2d = rng.uniform(0, 1000, (F, 4)).astype(F32)
    det = od.collect(bt, ids, types, list(box2d), "KITTI", "nms")
    pre = {(i, c): det[i][c] for i in det for c in det[i]}
    want, keeps = od.nms_results(det, thresh, "KITTI", "nms")
    assert sum(len(v) - len(keeps[k]) for k, v in pre.items()) > 100       # duplicates are suppressed
    _, got = _device(bt, ids, types, box2d, "KITTI", "nms", thresh)
    got, want = _flat(got), _flat(want)
    wrong = [k for k in want if k not in got or got[k].shape != want[k].shape
             or not np.array_equal(got[k][:, [0, 1, 2, 3, 7, 8, 9, 10, 11]], want[k][:, [0, 1, 2, 3, 7, 8, 9, 10, 11]])]
    print("\nDetectionCollector: %d lists, %d wrong" % (len(want), len(wrong)))
    assert not wrong, "%d of %d lists differ from the oracle: %s" % (len(wrong), len(want), wrong[:10])
    assert len(_compare(got, want, pre, "KITTI", thresh, "nms")) == len(want)
