"""GPU: the TF32 PointNet section max at every number of sections a warp's 16 rows can hold, compared BIT-EXACTLY
with the float64 reference of tests/exact_ref.py.

After each layer-3 chunk a warp takes one masked reduce-scatter pass per section that starts in its 16 rows (row 0
counts as a start), so the cases give the warp windows every section count 1..16, with the first section either
starting at row 0 or running in from the previous window (across warp, warpgroup and tile edges), and cut tiles
whose row count is not a multiple of 8, so that the rows past it (section -1) begin in the middle of a warp.  Every
third section is all-negative, so no atomic of its pass fires and its cells stay 0.  A last case raises b3 so that
the zero record the kernel stages past a tile's row count beats every real row in half the channels: those rows'
accumulators change the result unless the select leaves them out of every pass."""
import ctypes as C
import dataclasses

import pytest
import torch

import exact_ref as X

pytestmark = pytest.mark.gpu

MODES = [((64, 64, 128), 1), ((128, 128, 256), 1), ((128, 128, 256), 2), ((256, 256, 512), 1),
         ((256, 256, 512), 2)]
CUT = (128, 117, 128, 99, 128, 61, 36, 128, 13)     # row counts 117, 99, 61, 13: suffix from mid-warp


def window_frustums(n_frustums=4, n_windows=64, seed=3):
    """Frustums of 16-row windows: window i of frustum f holds k = 1 + (i + i // 8 + f) % 16 sections, so at
    128-row tiles every count 1..16 meets every warp of both warpgroups; in frustums 1 and 3 the window's first row
    continues the previous window's last section."""
    g = torch.Generator().manual_seed(seed)
    frustums = []
    for f in range(n_frustums):
        starts = []
        for i in range(n_windows):
            k = 1 + (i + i // 8 + f) % 16
            inner = (torch.randperm(15, generator=g)[:k - 1] + 1).tolist()
            cross = f % 2 == 1 and i > 0
            starts += sorted(16 * i + r for r in inner + ([] if cross else [0]))
        bounds = starts + [16 * n_windows]
        lengths = [b - a for a, b in zip(bounds, bounds[1:])]
        frustums.append([(n, "neg" if t % 3 == 2 else "pos") for t, n in enumerate(lengths)])
    return frustums


def window_counts(case):
    """{(warp of the tile, sections in its rows below nrows)}, and the row counts of the case's tiles."""
    rows_i = case.rows.view(torch.int32)
    seen, nrows = set(), []
    for b, row0, n, _ in case.tiles[:case.ntiles].tolist():
        sect = rows_i[b, row0:row0 + n, 3].tolist()
        nrows.append(n)
        for w in range(0, n, 16):
            seen.add((w // 16, len(set(sect[w:w + 16]))))
    return seen, nrows


def check(case, precision, what):
    from frustum_convnet_b200 import _lib
    dev = torch.device("cuda:0")
    d = X.pointnet_device_weights(case.W, dev)
    d["rows"] = case.rows.to(dev)
    d["tiles"] = case.tiles.to(dev)
    d["ntiles"] = torch.tensor([case.ntiles], dtype=torch.int32, device=dev)
    d["out"] = case.feat_init.to(dev)
    a = X.pointnet_args(case, d, precision)
    _lib.call("fcn_pointnet_tiles", C.byref(a), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    got, exp = d["out"].cpu(), X.pointnet_pooled_ref(case)
    assert X.bits_equal(got, exp), "%s:\n%s" % (what, X.describe_mismatch(got, exp))


def mode_id(m):
    return "%d-%d-%d-p%d" % (m[0] + (m[1],))


@pytest.mark.parametrize("cuts", [(128,), CUT], ids=["whole-tiles", "cut-tiles"])
@pytest.mark.parametrize("regime", ["R1", "R2"])
@pytest.mark.parametrize("dims,precision", MODES, ids=[mode_id(m) for m in MODES])
def test_pointnet_every_section_count_exact(dims, precision, regime, cuts):
    W = X.make_pointnet_weights(*dims, regime, seed=17 + sum(dims) + len(regime))
    case = X.make_pointnet_case(W, window_frustums(), 128, cuts, seed=9, ensure_argmax=False)
    seen, nrows = window_counts(case)
    if cuts == (128,):
        assert seen == {(w, k) for w in range(8) for k in range(1, 17)}, sorted(seen)
    else:
        assert {k for _, k in seen} == set(range(1, 17)), sorted(seen)
        assert any(n % 8 for n in nrows) and any(n % 16 == 4 for n in nrows), nrows
    check(case, precision, "section counts per window, cuts %s" % (cuts,))


def zero_record_wins(W):
    """W with b3 raised in every even channel so that the zero record (what the kernel stages for the rows past a
    tile's row count) has a larger value there than any record of the coordinate universe."""
    U = X.record_universe(W.coords.tolist())
    vals = X.pointnet_row_values(U, W)
    zero = X.pointnet_row_values(torch.zeros(1, 3, dtype=torch.float64), W)[0]
    shift = torch.clamp(vals.amax(0) - zero + 1, min=0)
    shift[1::2] = 0
    W2 = dataclasses.replace(W, b3=W.b3 + shift)
    X.check_pointnet_bounds(W2)
    return W2


@pytest.mark.parametrize("regime", ["R1", "R2"])
@pytest.mark.parametrize("dims,precision", MODES, ids=[mode_id(m) for m in MODES])
def test_pointnet_rows_past_nrows_excluded_exact(dims, precision, regime):
    W = zero_record_wins(X.make_pointnet_weights(*dims, regime, seed=23 + sum(dims) + len(regime)))
    case = X.make_pointnet_case(W, window_frustums(2, 24), 128, CUT, seed=13, ensure_argmax=False)
    # the same tiles with the zero records past nrows counted into the last section below nrows
    zero = X.pointnet_row_values(torch.zeros(1, 3, dtype=torch.float64), W)[0]
    rows_i = case.rows.view(torch.int32)
    leaky = X.pointnet_pooled_ref(case).clone()
    C3, partial = W.dims[2], 0
    for b, row0, n, _ in case.tiles[:case.ntiles].tolist():
        if n % 16:
            partial += 1
            t = int(rows_i[b, row0 + n - 1, 3])
            leaky[b, t, :C3] = torch.maximum(leaky[b, t, :C3].double(), zero).float()
    assert partial >= 4
    assert not X.bits_equal(leaky, X.pointnet_pooled_ref(case)), "the zero records would not change the result"
    check(case, precision, "zero records past nrows")
