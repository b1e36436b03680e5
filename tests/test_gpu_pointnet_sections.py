"""GPU: the section max of the TF32 PointNet kernel, by the shape of each warp's 16 rows, compared BIT-EXACTLY with
the float64 reference of tests/exact_ref.py.

A warp whose rows hold one or two sections reduces each section with a butterfly over its lanes; three or more take
the segmented suffix max.  The cases put every warp on each path: two sections with the boundary at every row
1..15 of the window in every warp of both warpgroups, one long section crossing warp, warpgroup and tile edges,
many short sections, and two-section windows cut by the tile's row count (the record slots past it hold NaN, which
the kernel never loads: it stages zero records there and leaves those rows out of every section).  Every third
section is all-negative (it never reaches the map), so a window often pairs it with a positive one."""
import ctypes as C

import pytest
import torch

import exact_ref as X

pytestmark = pytest.mark.gpu

MODES = [((64, 64, 128), 1), ((128, 128, 256), 1), ((128, 128, 256), 2), ((256, 256, 512), 1),
         ((256, 256, 512), 2)]


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


def _kind(i):
    return "neg" if i % 3 == 2 else "pos"


def two_section_windows(n_windows=120):
    """Section lengths such that 16-row window i has exactly two sections, split at row 1 + (i // 8) % 15: with
    128-row tiles window i is warp i % 8, so every boundary 1..15 falls in every warp of both warpgroups."""
    beta = [1 + (i // 8) % 15 for i in range(n_windows)]
    lengths = [beta[0]] + [16 + beta[i + 1] - beta[i] for i in range(n_windows - 1)] + [16 - beta[-1]]
    assert sum(lengths) == 16 * n_windows
    return [(n, _kind(i)) for i, n in enumerate(lengths)]


def one_section_windows():
    lengths = [16, 32, 48, 64, 37, 91, 128, 129, 200, 300, 64, 16]
    return [(n, "neg" if i == 5 else "pos") for i, n in enumerate(lengths)]


def short_sections(n=200):
    return [(1 + (7 * i) % 5, _kind(i)) for i in range(n)]


def window_shapes(case):
    """Number of sections (0, 1, 2, 3+) of every 16-row warp window of the case's tiles."""
    rows_i = case.rows.view(torch.int32)
    counts = [0, 0, 0, 0]
    for b, row0, n, _ in case.tiles[:case.ntiles].tolist():
        sect = rows_i[b, row0:row0 + n, 3].tolist()
        for w in range(0, case.tile_rows, 16):
            s = sect[w:min(w + 16, n)]
            counts[min(3, len(set(s)))] += 1
    return counts


PATTERNS = {
    # name: (frustums, tile cuts)
    "two-sections": ([two_section_windows()], (128,)),
    "one-section": ([one_section_windows(), one_section_windows()[::-1]], (128, 96, 128, 64)),
    "many-sections": ([short_sections()], (128, 128, 77)),
    "two-sections-cut": ([two_section_windows(64), two_section_windows(40)], (128, 125, 128, 119, 106, 73, 9)),
}


@pytest.mark.parametrize("pattern", sorted(PATTERNS))
@pytest.mark.parametrize("regime", ["R1", "R2"])
@pytest.mark.parametrize("dims,precision", MODES, ids=["%d-%d-%d-p%d" % (m[0] + (m[1],)) for m in MODES])
def test_pointnet_section_shapes_exact(dims, precision, regime, pattern):
    frustums, cuts = PATTERNS[pattern]
    W = X.make_pointnet_weights(*dims, regime, seed=31 + sum(dims) + len(regime))
    # sections are up to 30 rows long: too many to make every row of a 13..16-row one a strict arg-max at 128
    # channels; the bit-exact compare still covers every (section, channel) cell
    case = X.make_pointnet_case(W, frustums, 128, cuts, seed=5, ensure_argmax=False)
    shapes = window_shapes(case)
    if pattern.startswith("two-sections"):
        assert shapes[2] >= 0.5 * sum(shapes), shapes
    elif pattern == "one-section":
        assert shapes[1] >= 0.5 * sum(shapes), shapes
    else:
        assert shapes[3] >= 0.5 * sum(shapes), shapes
    check(case, precision, "%s windows (0/1/2/3+ sections: %s)" % (pattern, shapes))
