"""GPU: batched rotated 3-D NMS (csrc/nms3d.cu, ``fcn_rotate_nms_3d``) against the oracle (oracle/nms.py).
The keep lists are index sets, so parity is EXACT wherever no pair sits within 1e-4 of the IoU threshold (fp32
kernel vs float64 oracle); inputs with such a pair are regenerated."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _dets(rng, n, spread):
    return np.concatenate([rng.normal([0, 1, 20], [spread, 0.2, spread], (n, 3)),
                           rng.uniform([3, 1.4, 1.3], [4.5, 1.9, 1.8], (n, 3)),
                           rng.uniform(-np.pi, np.pi, (n, 1)), rng.random((n, 1))], 1).astype(np.float32)


def test_single_list_matches_oracle_and_reference_contract():
    from frustum_convnet_b200.nms import cube_nms, rotate_nms_3d_cc
    from oracle import nms as onms
    rng = np.random.default_rng(1)
    done = 0
    while done < 12:
        n = int(rng.integers(2, 90))
        d = _dets(rng, n, spread=float(rng.uniform(1.0, 6.0)))
        thr = float(rng.choice([0.1, 0.25, 0.5, 0.7]))
        if onms.pair_margins(d, thr) < 1e-4:
            continue
        want = onms.rotate_nms_3d_cc(d, thr)
        got = rotate_nms_3d_cc(torch.from_numpy(d).cuda(), thr)
        assert got == want, (n, thr)
        done += 1
    assert cube_nms(torch.zeros((0, 8), device="cuda"), 0.5) == []
    one = torch.from_numpy(_dets(rng, 1, 1.0)).cuda()
    assert cube_nms(one, 0.5) == [0]
    with pytest.raises(RuntimeError):
        cube_nms(one.cpu(), 0.5)


def test_batched_segments_top_k_and_ties():
    from frustum_convnet_b200.nms import rotate_nms_3d_batched
    from oracle import nms as onms
    rng = np.random.default_rng(2)
    segs, lens = [], [0, 1, 37, 120, 300, 5]
    for n in lens:
        while True:
            d = _dets(rng, n, spread=3.0)
            if n < 2 or onms.pair_margins(d, 0.3) >= 1e-4:
                break
        segs.append(d)
    segs[5][:, 7] = 0.5                                   # all-equal scores: larger index first
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    dets = torch.from_numpy(np.concatenate(segs)).cuda()
    keep, cnt = rotate_nms_3d_batched(dets, torch.from_numpy(off), 0.3, top_k=40)
    keep, cnt = keep.cpu().numpy(), cnt.cpu().numpy()
    for s, d in enumerate(segs):
        want = [off[s] + k for k in onms.rotate_nms_3d_cc(d, 0.3, top_k=40)]
        assert cnt[s] == len(want) and keep[s, :cnt[s]].tolist() == want, s
        assert (keep[s, cnt[s]:] == -1).all()


def _overlap_margin(d, thr):
    """pair_margins restricted to the pairs whose bounding cubes overlap (every other pair has IoU 0, so its margin
    is thr): the same filter, affordable for lists of hundreds of boxes."""
    from oracle import box_iou as ob
    from oracle import nms as onms
    c = onms.boxes3d2corners(d)
    mn, mx = c.min(1), c.max(1)
    ext = np.minimum(mx[:, None], mx[None]) - np.maximum(mn[:, None], mn[None])
    i, j = np.nonzero(np.triu((ext > 0).all(2), 1))
    m = thr
    for a, b in zip(i, j):
        m = min(m, abs(ob.rbbox_iou_3d_pair(c[a:a + 1], c[b:b + 1])[0, 1] - thr))
    return m, len(i)


def test_list_capacity_refused_not_truncated():
    """One list holds at most fcn_rotate_nms_3d_max_dets() rows: a full list matches the oracle, one row more raises
    instead of silently keeping only its first rows."""
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200.nms import cube_nms, rotate_nms_3d_batched
    from oracle import nms as onms
    cap = int(_lib.load().fcn_rotate_nms_3d_max_dets())
    assert cap == 512
    rng = np.random.default_rng(3)
    while True:
        d = _dets(rng, cap, spread=25.0)
        d[:, 7] = rng.permutation(cap).astype(np.float32) / cap          # distinct scores
        margin, n_pairs = _overlap_margin(d, 0.25)
        if margin >= 1e-4:
            break
    assert n_pairs >= 50, n_pairs                                        # the list does suppress
    want = onms.rotate_nms_3d_cc(d, 0.25, top_k=cap)
    assert cube_nms(torch.from_numpy(d).cuda(), 0.25, top_k=cap) == want
    assert len(want) < cap
    extra = np.concatenate([d, _dets(rng, 1, 1.0)])
    extra[-1, 7] = 2.0                                                   # the best box is the one past the capacity
    with pytest.raises(RuntimeError, match="exceeds"):
        cube_nms(torch.from_numpy(extra).cuda(), 0.25)
    off = torch.tensor([0, 3, 3 + cap + 1], dtype=torch.int32)
    with pytest.raises(RuntimeError, match="exceeds"):
        rotate_nms_3d_batched(torch.from_numpy(np.concatenate([d[:3], extra])).cuda(), off.cuda(), 0.25)


def test_nan_and_signed_zero_scores_follow_the_oracle_order():
    """NaN scores rank above every number (numpy's argsort puts NaN last, the reversed order first), -0.0 ties
    with +0.0, and ties go to the larger index: the ranks stay a permutation and the keep lists equal the oracle's."""
    from frustum_convnet_b200.nms import rotate_nms_3d_batched
    from oracle import nms as onms
    rng = np.random.default_rng(4)
    segs = []
    for n, thr_spread in ((40, 2.0), (64, 3.0), (7, 1.0), (130, 4.0)):
        while True:
            d = _dets(rng, n, spread=thr_spread)
            s = rng.random(n).astype(np.float32)
            k = rng.permutation(n)
            s[k[:max(2, n // 8)]] = np.nan
            s[k[n // 8 + 2:n // 8 + 5]] = 0.0
            s[k[n // 8 + 5:n // 8 + 8]] = -0.0
            d[:, 7] = s
            if onms.pair_margins(d, 0.3) >= 1e-4:
                break
        segs.append(d)
    segs[2][:, 7] = np.nan                                              # a list of NaN scores only
    lens = [len(d) for d in segs]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    keep, cnt = rotate_nms_3d_batched(torch.from_numpy(np.concatenate(segs)).cuda(), torch.from_numpy(off), 0.3,
                                      top_k=200)
    keep, cnt = keep.cpu().numpy(), cnt.cpu().numpy()
    for s, d in enumerate(segs):
        want = [off[s] + k for k in onms.rotate_nms_3d_cc(d, 0.3, top_k=200)]
        assert cnt[s] == len(want) and keep[s, :cnt[s]].tolist() == want, s
        assert len(set(keep[s, :cnt[s]].tolist())) == cnt[s]
