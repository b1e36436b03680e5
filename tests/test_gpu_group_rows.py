"""GPU: fcn_group_rows called directly through _lib.GroupArgs and compared BIT-EXACTLY with tests/group_ref.py.

Every case runs on both implementations (force_scan 0: the single-launch bit-matrix kernel where the shared-memory
rule allows it; 1: the count + emit pair) and in both row modes.  Records, counts and the feature map must match
bit for bit, the tile table as a multiset with each frustum's tiles in consecutive slots, and every buffer element
the call must not touch (record slots past a frustum's rows, feature pad rows, tile slots past the count, ntiles
entries of absent scales) keeps its sentinel.  The cases choose the edges: N at the 32-bit bit-matrix words and the
128-point ballot step, hits below / at / above K with the limit reached inside a ballot step, T at the 32-section
chunks and the 512 / 1024-thread scan rounds, eight scales, sorted centres with duplicates and unsorted ones (one
swapped pair, descending, one NaN), +-inf centres and depths, depths exactly at zc +- dis_z and pairs whose exact
distance is below dis_z but whose fp32 difference rounds onto it.

The engine-level tests tie the callers (eval plan, PointNetModule un-pooled path, TrainEngine) to the same
restatement at the shipped shapes, and the chained tests feed the kernel's own rows and tile table to
fcn_pointnet_tiles and check the result against tests/exact_ref.py."""
import ctypes as C
import functools
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import pytest
import torch

import exact_ref as X
import group_ref as G
from conftest import GOLDEN_CASES, load_golden

pytestmark = pytest.mark.gpu

F32 = np.float32
ROW_SENT = 0x7FA5A5A5             # NaN payloads the kernels never produce
FEAT_SENT = 0x7FB0B0B0
TILE_SENT = -0x21524111           # 0xDEADBEEF
CNT_SENT = -7
NTILES_GARBAGE = 0x5A5A5A5A


def dev():
    return torch.device("cuda:0")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return t.data_ptr() if t is not None else None


# ============================================================================ verification
def verify_scale(ref: G.ScaleRef, rows, cnt, tiles, ntile, tile_cap, tile_rows, what, pad_sentinel=True):
    """rows (B, row_cap, 4) float32, cnt (B, T) int32, tiles (slots, 4) int32 as the call left them."""
    assert np.array_equal(cnt, ref.cnt), "%s: cnt differs at %s" % (what, np.argwhere(cnt != ref.cnt)[:5].tolist())
    for b in range(cnt.shape[0]):
        n = ref.total(b)
        assert n <= rows.shape[1], what
        ok = G.record_bits_equal(rows[b, :n], ref.rows[b])
        if not ok.all():
            i = int(np.argmin(ok))
            raise AssertionError("%s: frustum %d, %d of %d records differ; first at row %d: got %r (tag %#x) expected "
                                 "%r (tag %#x)" % (what, b, int((~ok).sum()), n, i, rows[b, i, :3].tolist(),
                                                   rows[b, i].view(np.int32)[3] & 0xFFFFFFFF, ref.rows[b][i, :3].tolist(),
                                                   ref.rows[b][i].view(np.int32)[3] & 0xFFFFFFFF))
        if pad_sentinel:
            assert (rows[b, n:].view(np.int32) == ROW_SENT).all(), "%s: frustum %d record slots past row %d written" % (
                what, b, n)
    nt = len(ref.tiles)
    assert ntile == nt, "%s: ntiles %d, expected %d" % (what, ntile, nt)
    stored = min(nt, tile_cap)
    tb = tiles[:stored]
    assert (tb[:, 3] == 0).all(), what
    got = [tuple(r) for r in tb[:, :3].tolist()]
    if stored == nt:
        assert sorted(got) == sorted(ref.tiles), "%s: tile table differs" % what
        for b in np.unique(tb[:, 0]):      # one atomicAdd per (b, s): consecutive slots, row0 ascending
            pos = np.nonzero(tb[:, 0] == b)[0]
            assert pos[-1] - pos[0] + 1 == pos.size, "%s: tiles of frustum %d not contiguous" % (what, b)
            assert np.array_equal(tb[pos, 1], np.arange(pos.size) * tile_rows), what
    else:
        assert len(set(got)) == stored and set(got) <= set(ref.tiles), "%s: truncated tile table" % what
    if pad_sentinel:
        assert (tiles[stored:] == TILE_SENT).all(), "%s: tile slots past %d written" % (what, stored)


def verify_feat(got, init, T, c3, one_hot, num_vec, what):
    exp = G.feat_ref(init, T, c3, one_hot, num_vec)
    bad = got.view(np.int32) != exp.view(np.int32)
    assert not bad.any(), "%s: feature map differs at %s" % (what, np.argwhere(bad)[:5].tolist())


# ============================================================================ direct calls
@dataclass
class Scale:
    cen: np.ndarray           # (B, 3, T) float32
    K: int
    dis_z: float
    feat: bool = False
    c3: int = 0
    ld_feat: int = 0
    feat_pitch: int = 0       # 0 means T

    @property
    def T(self):
        return self.cen.shape[2]


@dataclass
class Case:
    pc: np.ndarray            # (B, 3, N) float32
    scales: List[Scale]
    tile_rows: int
    one_hot: Optional[np.ndarray] = None
    num_vec: int = 0
    row_extra: int = 3        # record slots past T*K per frustum (must keep their sentinel)
    tile_cap: Optional[int] = None   # capacity passed to the call (None: every tile fits)
    tile_extra: int = 4       # table slots past the capacity

    @property
    def B(self):
        return self.pc.shape[0]

    @property
    def N(self):
        return self.pc.shape[2]

    def Ts(self):
        return [s.T for s in self.scales]

    def Ks(self):
        return [s.K for s in self.scales]


class Run:
    """Device buffers of one case, sentinel-filled, and the GroupArgs that point at them."""

    def __init__(self, c: Case):
        B = c.B
        i32 = torch.int32
        self.pc = torch.from_numpy(c.pc).to(dev())
        self.one_hot = torch.from_numpy(c.one_hot).to(dev()) if c.one_hot is not None else None
        self.cen, self.rows, self.cnt, self.tiles, self.idx, self.feat, self.caps = [], [], [], [], [], [], []
        for sc in c.scales:
            TK = sc.T * sc.K
            self.cen.append(torch.from_numpy(np.ascontiguousarray(sc.cen)).to(dev()))
            self.rows.append(torch.full((B, TK + c.row_extra, 4), ROW_SENT, dtype=i32, device=dev()))
            self.cnt.append(torch.full((B, sc.T), CNT_SENT, dtype=i32, device=dev()))
            cap = c.tile_cap if c.tile_cap is not None else B * -(-TK // c.tile_rows)
            self.caps.append(cap)
            self.tiles.append(torch.full((cap + c.tile_extra, 4), TILE_SENT, dtype=i32, device=dev()))
            self.idx.append(torch.full((B, sc.T, sc.K), -3, dtype=i32, device=dev()))
            f = None
            if sc.feat:
                f = torch.full((B, sc.feat_pitch or sc.T, sc.ld_feat), FEAT_SENT, dtype=i32, device=dev())
            self.feat.append(f)
        self.ntiles = torch.full((8,), NTILES_GARBAGE, dtype=i32, device=dev())

    def args(self, c: Case, unique_rows: int, force_scan: int):
        from frustum_convnet_b200 import _lib
        g = _lib.GroupArgs()
        g.num_scales, g.B, g.N, g.num_vec = len(c.scales), c.B, c.N, c.num_vec
        g.tile_rows, g.unique_rows, g.force_scan = c.tile_rows, unique_rows, force_scan
        g.pc, g.one_hot = _ptr(self.pc), _ptr(self.one_hot)
        for s, sc in enumerate(c.scales):
            g.centers[s], g.T[s], g.K[s], g.dis_z[s] = _ptr(self.cen[s]), sc.T, sc.K, sc.dis_z
            g.c3[s], g.ld_feat[s] = (sc.c3, sc.ld_feat) if sc.feat else (0, 0)
            g.row_cap[s], g.tile_cap[s] = self.rows[s].shape[1], self.caps[s]
            g.rows[s], g.cnt[s], g.feat[s] = _ptr(self.rows[s]), _ptr(self.cnt[s]), _ptr(self.feat[s])
            g.tiles[s], g.idx_scratch[s], g.feat_pitch[s] = _ptr(self.tiles[s]), _ptr(self.idx[s]), sc.feat_pitch
        g.ntiles = _ptr(self.ntiles)
        return g

    def launch(self, c: Case, unique_rows: int, force_scan: int):
        from frustum_convnet_b200 import _lib
        g = self.args(c, unique_rows, force_scan)
        _lib.call("fcn_group_rows", C.byref(g), _stream())
        torch.cuda.synchronize()

    def snapshot(self):
        return dict(rows=[r.cpu().numpy().view(F32) for r in self.rows], cnt=[t.cpu().numpy() for t in self.cnt],
                    tiles=[t.cpu().numpy() for t in self.tiles], ntiles=self.ntiles.cpu().numpy(),
                    feat=[f.cpu().numpy().view(F32) if f is not None else None for f in self.feat])


def check_case(c: Case, refs: List[G.ScaleRef], snap, what):
    for s, (sc, ref) in enumerate(zip(c.scales, refs)):
        w = "%s scale %d (T=%d K=%d)" % (what, s, sc.T, sc.K)
        verify_scale(ref, snap["rows"][s], snap["cnt"][s], snap["tiles"][s], int(snap["ntiles"][s]),
                     c.tile_cap if c.tile_cap is not None else 1 << 30, c.tile_rows, w)
        if sc.feat:
            verify_feat(snap["feat"][s], _feat_init(c, s), sc.T, sc.c3, c.one_hot, c.num_vec, w)
    assert (snap["ntiles"][len(c.scales):] == 0).all(), "%s: ntiles of absent scales not reset" % what


def _feat_init(c: Case, s: int):
    sc = c.scales[s]
    return np.full((c.B, sc.feat_pitch or sc.T, sc.ld_feat), FEAT_SENT, dtype=np.int32).view(F32)


# ---------------------------------------------------------------------------- case builders
ZLO, ZHI = 0.0, 20.0
GRID = 1.0 / 64


def _points(rng, B, N, gap=None, specials=True, far=()):
    """Depths in [ZLO, ZHI): half of them on a 1/64 grid (duplicates, and exact zc +- dis_z against grid centres),
    NaN / +inf / -inf depths at random indices (point 0 of frustum 1 is NaN: empty sections gather it), frustums in
    `far` out of every section's reach."""
    pc = rng.uniform(-8, 8, (B, 3, N))
    z = rng.uniform(ZLO, ZHI, (B, N))
    if gap is not None:
        lo, hi = gap
        inside = (z > lo) & (z < hi)
        z[inside] = ZHI - (z[inside] - lo)
    z = np.where(rng.random((B, N)) < 0.5, np.round(z / GRID) * GRID, z)
    pc[:, 2] = z
    pc = pc.astype(F32)
    if specials and N >= 8:
        for b in range(B):
            k = rng.choice(np.arange(1, N), 3, replace=False)
            pc[b, 2, k] = [np.nan, np.inf, -np.inf]
        if B > 1:
            pc[1, 2, 0] = np.nan
    for b in far:
        pc[b, 2] = F32(1e6)
    return pc


def _centres(rng, B, T, kind="asc", D=0.5, inner=False, ends=False):
    """Section centres over [ZLO - 2D, ZHI + 2D] (sections past the points at both ends are empty), on the grid,
    ascending with one duplicate; kind: asc | swap (one adjacent pair swapped) | desc | nan | inf (-inf first,
    +inf last)."""
    lo, hi = (ZLO, ZHI) if inner else (ZLO - 2 * D, ZHI + 2 * D)
    z = np.sort(np.round(rng.uniform(lo, hi, (B, T)) / GRID) * GRID, axis=1)
    if T >= 4:
        z[:, T // 2] = z[:, T // 2 - 1]
    if ends:      # the first and the last section out of every point's reach
        z[:, 0], z[:, -1] = ZLO - 2 * D - 1, ZHI + 2 * D + 1
    if kind == "swap":
        for b in range(B):
            i = int(np.nonzero(np.diff(z[b]) > 0)[0][0])
            z[b, i], z[b, i + 1] = z[b, i + 1], z[b, i]
    elif kind == "desc":
        z = z[:, ::-1]
    elif kind == "nan":
        z[:, T // 3] = np.nan
    elif kind == "inf":
        z[:, 0], z[:, -1] = -np.inf, np.inf
    cen = rng.uniform(-8, 8, (B, 3, T))
    cen[:, 2] = z
    return cen.astype(F32)


def _generic(seed, B, N, scales, tile_rows, kind="asc", feat=False, one_hot=False, gap=None, far=(), inner=False,
             ends=False, pitch_extra=2, **kw):
    rng = np.random.default_rng(seed)
    pc = _points(rng, B, N, gap=gap, far=far)
    V = 3 if one_hot else 0
    sc = []
    for j, (T, K, D) in enumerate(scales):
        f = feat if not isinstance(feat, (list, tuple)) else feat[j]
        c3 = 8 * (j + 1)
        sc.append(Scale(_centres(rng, B, T, kind, D, inner, ends), K, D, bool(f), c3, (c3 + V + 2 + 3) // 4 * 4 + 4,
                        (T + pitch_extra) if (f and pitch_extra) else 0))
    oh = rng.integers(0, 2, (B, V)).astype(F32) + F32(0.5) if one_hot else None
    return Case(pc, sc, tile_rows, oh, V, **kw)


def _cluster(seed, K, B=2):
    """Isolated point clusters of exactly 0, 1, K-1, K, K+1 and 3K points (hits below, at and above K), scattered
    over the point indices so that the limit is reached inside a 128-point ballot step; frustum 1 takes its
    centres in descending order (unsorted path)."""
    rng = np.random.default_rng(seed)
    sizes = [0, 1, max(K - 1, 0), K, K + 1, 3 * K]
    N = 1024 if sum(sizes) < 900 else 2053
    D = 0.5
    pc = rng.uniform(-8, 8, (B, 3, N)).astype(F32)
    depths = 10.0 * (np.arange(len(sizes)) + 1)
    for b in range(B):
        perm = rng.permutation(N)
        z = np.empty(N)
        z[:] = depths[-1] + 5.0 + rng.uniform(0, 3, N)            # filler: out of every section's reach
        o = 0
        for d, n in zip(depths, sizes):
            z[perm[o:o + n]] = d + np.round(rng.uniform(-0.4, 0.4, n) / GRID) * GRID
            o += n
        pc[b, 2] = z.astype(F32)
        big = np.sort(perm[o - 3 * K:o])
        if K >= 32:   # the K-th and (K+1)-th hits share a 128-point step: the count stops inside the step
            assert big[K - 1] // 128 == big[K] // 128, "cluster seed does not reach K inside a ballot step"
    zc = np.concatenate([[0.0], depths, [depths[-1] + 3.0]])
    cen = rng.uniform(-8, 8, (B, 3, zc.size))
    cen[:, 2] = zc
    cen[1, 2] = zc[::-1]
    return Case(pc, [Scale(cen.astype(F32), K, D)], 64 if K < 128 else 128)


def _rounding(seed):
    """Centres with fine-ulp depths in (0.05, 0.45) and coarser ones in (1.05, 1.45), dis_z = 1: the points at
    zc +- 1 include depths whose exact distance is below 1 but whose fp32 difference is 1.0 (not hits), their
    neighbours one ulp inside, and depths at exactly zc +- 1.  Frustum 1 holds the centres shuffled (unsorted)."""
    rng = np.random.default_rng(seed)
    D = F32(1.0)
    T, N, B = 40, 256, 2
    zc = np.sort(np.concatenate([rng.uniform(0.05, 0.45, T // 2), rng.uniform(1.05, 1.45, T // 2)]).astype(F32))
    special = []
    for c in zc:
        for e in G.rounding_edges(c, D)[:2]:
            special += [e, np.nextafter(e, c)]
        for z in (F32(c - D), F32(c + D)):       # at exactly zc -+ 1 (when representable): not a hit
            if abs(float(c) - float(z)) == 1.0:
                special.append(z)
    special = np.array(special, dtype=F32)
    n_edges = sum(len(G.rounding_edges(c, D)) > 0 for c in zc)
    assert n_edges >= T // 2, "too few rounding edges (%d)" % n_edges
    pc = rng.uniform(-8, 8, (B, 3, N)).astype(F32)
    for b in range(B):
        z = rng.uniform(-1.0, 3.0, N).astype(F32)
        m = min(special.size, N - 8)
        z[rng.choice(N, m, replace=False)] = rng.permutation(special)[:m]
        pc[b, 2] = z
    cen = rng.uniform(-8, 8, (B, 3, T)).astype(F32)
    cen[0, 2] = zc
    cen[1, 2] = rng.permutation(zc)
    return Case(pc, [Scale(cen, 256, float(D))], 64)


CASES = {
    "n1": lambda: _generic(1, 3, 1, [(5, 1, 0.5), (3, 3, 2.0)], 7),
    "n31": lambda: _generic(2, 3, 31, [(33, 3, 0.5), (17, 1, 1.0)], 1),
    "n32": lambda: _generic(3, 1, 32, [(32, 32, 4.0)], 64, feat=True),
    "n33_b17": lambda: _generic(4, 17, 33, [(31, 32, 1.0), (16, 3, 0.5), (8, 1, 2.0)], 7, feat=True, one_hot=True),
    "n127": lambda: _generic(5, 3, 127, [(64, 128, 2.0)], 128, feat=True),
    "n128": lambda: _generic(6, 3, 128, [(129, 32, 0.5)], 64),
    "n129": lambda: _generic(7, 3, 129, [(127, 256, 1.0), (64, 3, 0.25)], 1),
    "t511": lambda: _generic(8, 3, 1024, [(511, 32, 0.25), (256, 64, 0.5)], 128, feat=True, one_hot=True),
    "t512": lambda: _generic(9, 2, 1024, [(512, 32, 0.25)], 64),
    "t513": lambda: _generic(10, 2, 1024, [(513, 32, 0.25)], 64, feat=True, pitch_extra=0),
    "t1023_1024_1025": lambda: _generic(11, 2, 127, [(1023, 8, 0.1), (1024, 3, 0.1), (1025, 1, 0.1)], 64,
                                        feat=(True, False, True), one_hot=True),
    "t2000": lambda: _generic(12, 3, 64, [(2000, 8, 0.1)], 64),
    "n2053": lambda: _generic(13, 2, 2053, [(200, 128, 0.5), (100, 256, 1.0)], 128, feat=True, one_hot=True),
    "scales8": lambda: _generic(14, 3, 300, [(40, 1, 0.5), (33, 3, 0.25), (32, 8, 1.0), (31, 32, 2.0), (20, 64, 0.5),
                                             (9, 128, 3.0), (2, 256, 8.0), (1, 5, 1.0)], 64,
                                feat=(True, False) * 4, one_hot=True),
    "swap": lambda: _generic(15, 2, 200, [(64, 16, 0.5), (33, 4, 1.0)], 64, kind="swap"),
    "desc": lambda: _generic(16, 2, 200, [(64, 16, 0.5), (33, 4, 1.0)], 64, kind="desc", feat=True),
    "nan_centre": lambda: _generic(17, 2, 200, [(64, 16, 0.5), (33, 4, 1.0)], 64, kind="nan"),
    "inf_centre": lambda: _generic(18, 2, 200, [(64, 16, 0.5), (33, 4, 1.0)], 64, kind="inf"),
    "switch517": lambda: _generic(19, 2, 1024, [(517, 64, 0.25)], 128),
    "switch518": lambda: _generic(20, 2, 1024, [(518, 64, 0.25)], 128),
    "empty": lambda: _generic(21, 3, 500, [(100, 16, 0.3)], 64, gap=(8.0, 12.0), far=(1,), ends=True),
    "tile_multiple": lambda: _generic(22, 2, 1000, [(64, 3, 2.0)], 64, inner=True),
    "tile_cap": lambda: _generic(23, 3, 256, [(64, 8, 0.5)], 7, tile_cap=10),
    "rounding": lambda: _rounding(24),
}
for _K in (1, 3, 32, 128, 256):
    CASES["hits_k%d" % _K] = functools.partial(_cluster, 30 + _K, _K)


@functools.lru_cache(maxsize=None)
def case(name) -> Case:
    return CASES[name]()


@functools.lru_cache(maxsize=None)
def reference(name, unique_rows):
    c = case(name)
    return [G.group_scale(c.pc, sc.cen, sc.dis_z, sc.K, unique_rows, c.tile_rows) for sc in c.scales]


@pytest.mark.parametrize("force_scan", [0, 1])
@pytest.mark.parametrize("unique_rows", [1, 0])
@pytest.mark.parametrize("name", list(CASES))
def test_group_rows_matches_restatement(name, unique_rows, force_scan):
    c = case(name)
    refs = reference(name, unique_rows)
    run = Run(c)
    first = None
    for call in range(2):     # the second call starts from the first call's ntiles and outputs
        run.launch(c, unique_rows, force_scan)
        snap = run.snapshot()
        check_case(c, refs, snap, "%s unique_rows=%d force_scan=%d call %d" % (name, unique_rows, force_scan, call))
        if first is None:
            first = snap
        else:
            for key in ("rows", "cnt", "feat"):
                for a, b in zip(first[key], snap[key]):
                    assert a is None or np.array_equal(a.view(np.int32), b.view(np.int32)), "%s differs on repeat" % key


def test_cases_reach_their_edges():
    """The case list really contains the edges it is meant to: which kernel each case takes under the shared-memory
    rule (recomputed here), empty sections, saturated sections, totals that are multiples of tile_rows, a
    truncated tile table and rounded-predicate pairs that are not hits."""
    assert G.bitmask_bytes(1024, [517], [64]) == 204732 and G.uses_bitmask(1024, [517], [64])
    assert G.bitmask_bytes(1024, [518], [64]) == 205128 and not G.uses_bitmask(1024, [518], [64])
    assert G.bitmask_bytes(64, [2000], [8]) == 104000
    for name in ("t2000", "t1023_1024_1025", "n2053", "switch517", "scales8", "rounding"):
        assert G.uses_bitmask(case(name).N, case(name).Ts(), case(name).Ks()), name
    assert not G.uses_bitmask(case("switch518").N, case("switch518").Ts(), case("switch518").Ks())
    # hits below, at and above K in every cluster case
    for K in (1, 3, 32, 128, 256):
        c = case("hits_k%d" % K)
        hits = G.group_scale(c.pc, c.scales[0].cen, c.scales[0].dis_z, 10 ** 6, 1, 64).cnt
        assert {0, 1, K, K + 1, 3 * K} <= set(hits.ravel().tolist()), K
    # empty sections at the start, the middle and the end; a frustum without any hit; saturated sections
    cnt = reference("empty", 1)[0].cnt
    assert cnt[0, 0] == 0 and cnt[0, -1] == 0 and (cnt[0, 1:-1] == 0).any() and (cnt[1] == 0).all()
    assert len([t for t in reference("empty", 1)[0].tiles if t[0] == 1]) == 0
    assert any((r.cnt == c.K).any() for r, c in zip(reference("t511", 1), case("t511").scales))
    tm = reference("tile_multiple", 1)[0]
    assert any(tm.total(b) > 0 and tm.total(b) % 64 == 0 for b in range(2))
    for u in (0, 1):
        assert len(reference("tile_cap", u)[0].tiles) > case("tile_cap").tile_cap
    # rounding pairs: some point at exact distance < dis_z is rejected by the rounded predicate
    c = case("rounding")
    z, zc = c.pc[0, 2].astype(np.float64), c.scales[0].cen[0, 2].astype(np.float64)
    exact = np.abs(zc[:, None] - z[None, :]) < 1.0
    rounded = np.abs((c.scales[0].cen[0, 2][:, None] - c.pc[0, 2][None, :]).astype(F32)) < F32(1.0)
    assert (exact & ~rounded).sum() >= 10


# ============================================================================ engine level: the shipped shapes
SHIPPED = [("car", 32), ("people", 8), ("sunrgbd", 8), ("refine_car", 32)] + [("golden", n) for n in GOLDEN_CASES]


def _workload_data(wl, B):
    from frustum_convnet_b200 import config, synth
    if wl == "golden":
        g, data, sd, w, cfg = load_golden(B)
        return data, w, cfg, sd
    cfg, w = config.load_workload(wl)
    data = synth.make_frustums(wl, B, seed=500 + B)
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=17)
    return data, w, cfg, sd


def _eval_model(w, sd, precision):
    modname = "det_base_sunrgbd" if w["arch"].num_scales == 5 else "det_base"
    mod = __import__("frustum_convnet_b200." + modname, fromlist=["PointNetDet"])
    m = mod.PointNetDet(3, num_vec=w["num_vec"])
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    m.precision = precision
    m.use_cuda_graph = False
    return m.to(dev()).eval()


def _inputs(data, S):
    pc = np.ascontiguousarray(data["point_cloud"][:, :3, :], dtype=F32)
    cen = [np.ascontiguousarray(data["center_ref%d" % (i + 1)], dtype=F32) for i in range(S)]
    return pc, cen


@pytest.mark.parametrize("wl,B", SHIPPED)
def test_eval_plan_grouping(wl, B):
    """The eval Plan's grouping call, launched alone (the feature map is read before PointNet writes into it)."""
    from frustum_convnet_b200 import _lib
    data, w, cfg, sd = _workload_data(wl, B)
    S = w["arch"].num_scales
    m = _eval_model(w, sd, precision=1)
    eng = m.engine()
    pc, cen = _inputs(data, S)
    B_ = pc.shape[0]
    plan = eng.plan(B_, pc.shape[2], [c.shape[2] for c in cen])
    plan.in_pc.copy_(torch.from_numpy(pc))
    for dst, c in zip(plan.in_centers, cen):
        dst.copy_(torch.from_numpy(c))
    V = eng.num_vec
    if V > 0:
        plan.in_onehot.copy_(torch.from_numpy(np.asarray(data["one_hot"], dtype=F32)))
    feat_init = []
    for s in range(S):
        plan.rows[s].view(torch.int32).fill_(ROW_SENT)
        plan.tiles[s].fill_(TILE_SENT)
        f = plan.buf["feat%d" % (s + 1)]
        f.view(torch.int32).fill_(FEAT_SENT)
        feat_init.append(f.cpu().numpy())
    plan.ntiles.fill_(NTILES_GARBAGE)
    g = plan.group_args
    g.pc, g.one_hot = _ptr(plan.in_pc), (_ptr(plan.in_onehot) if V > 0 else None)
    for s in range(S):
        g.centers[s] = _ptr(plan.in_centers[s])
    _lib.call("fcn_group_rows", C.byref(g), _stream())
    torch.cuda.synchronize()
    ntiles = plan.ntiles.cpu().numpy()
    one_hot = np.asarray(data["one_hot"], dtype=F32) if V > 0 else None
    for s in range(S):
        K = w["arch"].nsample[s]
        assert g.row_cap[s] == cen[s].shape[2] * K
        ref = G.group_scale(pc, cen[s], cfg.DATA.HEIGHT_HALF[s], K, 1, eng.tile_rows)
        what = "%s B=%d plan scale %d" % (wl, B_, s)
        verify_scale(ref, plan.rows[s].cpu().numpy(), plan.cnt[s].cpu().numpy(), plan.tiles[s].cpu().numpy(),
                     int(ntiles[s]), g.tile_cap[s], eng.tile_rows, what)
        verify_feat(plan.buf["feat%d" % (s + 1)].cpu().numpy(), feat_init[s], cen[s].shape[2], eng.c3[s], one_hot, V,
                    what)
    assert (ntiles[S:] == 0).all()


class _DevView:
    """A device buffer the caller only knows by address (torch.as_tensor reads __cuda_array_interface__)."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, data=(int(ptr), False),
                                             version=2, strides=None)


def _read(ptr, shape, typestr):
    return torch.as_tensor(_DevView(ptr, shape, typestr), device=dev()).cpu().numpy()


@pytest.mark.parametrize("wl,B", SHIPPED)
def test_pointnet_module_unpooled_grouping(wl, B, monkeypatch):
    """PointNetModule.forward (the un-pooled path) groups into buffers of its own: read them when its
    fcn_group_rows call returns."""
    from frustum_convnet_b200 import _lib
    data, w, cfg, sd = _workload_data(wl, B)
    S = w["arch"].num_scales
    m = _eval_model(w, sd, precision=0)
    pc, cen = _inputs(data, S)
    seen = []
    real = _lib.call

    def spy(name, *args):
        r = real(name, *args)
        if name == "fcn_group_rows":
            torch.cuda.synchronize()
            g = args[0]._obj
            Bg, T, K = g.B, g.T[0], g.K[0]
            seen.append(dict(g=g, dis_z=g.dis_z[0], unique=g.unique_rows, tile_rows=g.tile_rows, feat=g.feat[0],
                             rows=_read(g.rows[0], (Bg, g.row_cap[0], 4), "<f4"), cnt=_read(g.cnt[0], (Bg, T), "<i4"),
                             tiles=_read(g.tiles[0], (g.tile_cap[0], 4), "<i4"), tile_cap=g.tile_cap[0],
                             ntiles=_read(g.ntiles, (8,), "<i4")))
        return r

    monkeypatch.setattr(_lib, "call", spy)
    pct = torch.from_numpy(pc).to(dev())
    for s in range(S):
        mod = getattr(m.feat_net, "pointnet%d" % (s + 1))
        mod(pct, None, torch.from_numpy(cen[s]).to(dev()))
        torch.cuda.synchronize()
        got = seen.pop()
        K = w["arch"].nsample[s]
        assert got["unique"] == 0 and got["feat"] is None and got["dis_z"] == F32(cfg.DATA.HEIGHT_HALF[s])
        ref = G.group_scale(pc, cen[s], cfg.DATA.HEIGHT_HALF[s], K, 0, got["tile_rows"])
        verify_scale(ref, got["rows"], got["cnt"], got["tiles"], int(got["ntiles"][0]), got["tile_cap"],
                     got["tile_rows"], "%s B=%d module scale %d" % (wl, pc.shape[0], s), pad_sentinel=False)
        assert (got["ntiles"][1:] == 0).all()


@pytest.mark.parametrize("wl,B", SHIPPED)
def test_train_engine_rows(wl, B):
    """TrainEngine.rows / cnt after forward: every T*K row, back-fill duplicates included (unique_rows = 0)."""
    import train_ref as tr
    from frustum_convnet_b200.train_engine import TrainEngine
    data, w, cfg, sd = _workload_data(wl, B)
    S = w["arch"].num_scales
    model = tr.make_model(wl if wl != "golden" else GOLDEN_CASES[B][0], seed=5)
    pc, cen = _inputs(data, S)
    B_, N = pc.shape[0], pc.shape[2]
    eng = TrainEngine(model, B_, N, [c.shape[2] for c in cen])
    eng.use_graph = False
    for s in range(S):
        eng.rows[s].view(torch.int32).fill_(ROW_SENT)
        eng.tiles[s].fill_(TILE_SENT)
    eng.ntiles.fill_(NTILES_GARBAGE)
    one_hot = torch.from_numpy(np.asarray(data["one_hot"], dtype=F32)).to(dev()) if eng.V > 0 else None
    eng.forward(torch.from_numpy(pc).to(dev()), [torch.from_numpy(c).to(dev()) for c in cen], one_hot)
    torch.cuda.synchronize()
    ntiles = eng.ntiles.cpu().numpy()
    for s in range(S):
        T, K = cen[s].shape[2], eng.K[s]
        assert eng.group_args.row_cap[s] == T * K
        ref = G.group_scale(pc, cen[s], float(model.feat_net.dists[s]), K, 0, 64)
        assert F32(model.feat_net.dists[s]) == F32(cfg.DATA.HEIGHT_HALF[s])
        verify_scale(ref, eng.rows[s].view(B_, T * K, 4).cpu().numpy(), eng.cnt[s].cpu().numpy(),
                     eng.tiles[s].cpu().numpy(), int(ntiles[s]), eng.group_args.tile_cap[s], 64,
                     "%s B=%d train scale %d" % (wl, B_, s))
    assert (ntiles[S:] == 0).all()


# ============================================================================ chained: grouping -> PointNet
def _integer_case(seed, B=3, N=400, T=64, K=16):
    """Integer coordinates: every hit record lies in exact_ref's R1 coordinate universe ([-4, 4]^3), so the PointNet
    arithmetic on it is exact.  Centres past the points give empty sections; one frustum has no hit at all."""
    rng = np.random.default_rng(seed)
    pc = np.zeros((B, 3, N), dtype=F32)
    pc[:, :2] = rng.integers(0, 5, (B, 2, N))
    pc[:, 2] = rng.integers(0, 40, (B, N))
    pc[B - 1, 2] = 1000.0
    cen = np.zeros((B, 3, T), dtype=F32)
    cen[:, :2] = rng.integers(0, 5, (B, 2, T))
    cen[:, 2] = np.sort(rng.integers(-4, 46, (B, T)), axis=1)
    return pc, cen, K, 2.5


def _chain(unique_rows, precision, tile_rows, unpooled):
    from frustum_convnet_b200 import _lib
    W = X.make_pointnet_weights(64, 64, 128, "R1", seed=41)
    C3 = 128
    pc, cen, K, D = _integer_case(42)
    B, T = pc.shape[0], cen.shape[2]
    V = 3
    one_hot = np.eye(V, dtype=F32)[np.arange(B) % V]
    sc = Scale(cen, K, D, feat=not unpooled, c3=C3, ld_feat=C3 + 8, feat_pitch=0 if unpooled else T + 2)
    c = Case(pc, [sc], tile_rows, one_hot if not unpooled else None, V if not unpooled else 0, row_extra=0)
    run = Run(c)
    if not unpooled:
        run.feat[0].view(torch.float32).fill_(X.SENTINEL)
    run.launch(c, unique_rows, 0)
    ref = G.group_scale(pc, cen, D, K, unique_rows, tile_rows)
    snap = run.snapshot()
    verify_scale(ref, snap["rows"][0], snap["cnt"][0], snap["tiles"][0], int(snap["ntiles"][0]), run.caps[0],
                 tile_rows, "chain grouping")
    ntile = int(snap["ntiles"][0])
    assert ntile > 0 and (ref.cnt[B - 1] == 0).all() and (ref.cnt[0] == 0).any()
    feat0 = torch.from_numpy(snap["feat"][0].copy()) if not unpooled else None
    pcase = X.PointnetCase(W, torch.from_numpy(snap["rows"][0].copy()), torch.from_numpy(snap["tiles"][0][:ntile].copy()),
                           ntile, T, (T + 2) if not unpooled else T, C3 + 8, tile_rows,
                           feat0 if feat0 is not None else torch.zeros(1))
    d = X.pointnet_device_weights(W, dev())
    d["rows"], d["tiles"], d["ntiles"] = run.rows[0], run.tiles[0], run.ntiles
    if unpooled:
        out_init = torch.full((B, C3, T, K), float("nan"))
        d["out"] = out_init.to(dev())
    else:
        d["out"] = run.feat[0].view(torch.float32)
    a = X.pointnet_args(pcase, d, precision, K)
    a.max_tiles = run.tiles[0].shape[0]
    if unpooled:
        a.unpooled, a.ld_feat, a.feat_pitch = 1, 0, 0
    _lib.call("fcn_pointnet_tiles", C.byref(a), _stream())
    torch.cuda.synchronize()
    got = d["out"].cpu()
    exp = X.pointnet_unpooled_ref(pcase, K, out_init) if unpooled else X.pointnet_pooled_ref(pcase)
    assert X.bits_equal(got, exp), "chain unique_rows=%d precision=%d:\n%s" % (
        unique_rows, precision, X.describe_mismatch(got, exp))
    return got


@pytest.mark.parametrize("precision,tile_rows", [(0, 64), (1, 128)])
def test_chain_pooled_from_unique_rows(precision, tile_rows):
    """unique_rows = 1 rows and the kernel-built tile table -> pooled fcn_pointnet_tiles, bit-exact (R1)."""
    _chain(1, precision, tile_rows, unpooled=False)


def test_chain_unpooled_from_all_rows():
    """unique_rows = 0 rows (back-fill duplicates, masked empty sections) -> un-pooled fcn_pointnet_tiles."""
    got = _chain(0, 0, 64, unpooled=True)
    assert not torch.isnan(got).any()
