"""CPU: the restatement of fcn_group_rows in tests/group_ref.py against the golden fixtures and the literal query
loop, and the argument checks of fcn_group_rows (all of them run before any CUDA call, so they are testable
without a GPU)."""
import ctypes as C

import numpy as np
import pytest

import group_ref as G
from conftest import GOLDEN_CASES, load_golden

F32 = np.float32


# ============================================================================ the restatement
def _rows_loop(pc, cen, idx, cnt, unique_rows):
    """Row records written as a plain loop over (b, t, l) from a query's idx / cnt."""
    B, T, K = idx.shape
    out = []
    for b in range(B):
        recs = []
        for t in range(T):
            c = int(cnt[b, t])
            for l in range(c if unique_rows else K):
                k = int(idx[b, t, l])
                r = np.empty(4, dtype=F32)
                for j in range(3):
                    with np.errstate(invalid="ignore", over="ignore"):
                        r[j] = F32(pc[b, j, k]) - F32(cen[b, j, t])
                r.view(np.int32)[3] = t if c > 0 else (t | -0x80000000)
                recs.append(r)
        out.append(np.array(recs, dtype=F32).reshape(-1, 4))
    return out


@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_restatement_matches_golden_query(name):
    """idx / cnt of the restatement equal the golden fixtures (the reference model's own grouping), and its records
    are the gather and centre subtraction of that idx: fp32 subtraction, equal to float64-then-round."""
    g, data, sd, w, cfg = load_golden(name)
    pc = data["point_cloud"][:, :3, :]
    for i in range(w["arch"].num_scales):
        cen = data["center_ref%d" % (i + 1)]
        K = w["arch"].nsample[i]
        for unique in (0, 1):
            ref = G.group_scale(pc, cen, cfg.DATA.HEIGHT_HALF[i], K, unique, 64)
            assert np.array_equal(ref.idx, g["idx%d" % (i + 1)].astype(np.int64))
            assert np.array_equal(ref.cnt, g["cnt%d" % (i + 1)].astype(np.int32))
            for b in range(pc.shape[0]):
                assert ref.total(b) == (int(ref.cnt[b].sum()) if unique else cen.shape[2] * K)
                r = ref.rows[b]
                t = r.view(np.int32)[:, 3] & 0x7FFFFFFF
                k = ref.idx[b, t, np.arange(r.shape[0]) - np.searchsorted(t, t)] if unique else ref.idx[b].reshape(-1)
                assert G.same_bits(r[:, :3], G.records_f64(pc, cen, b, k, t)).all()
                n = ref.total(b)
                assert ref.tiles.count((b, 0, min(64, n))) == (1 if n else 0)


def _edge_inputs(seed, B, N, M, dz):
    rng = np.random.default_rng(seed)
    a = (rng.random((B, 3, N)) * 4 - 2).astype(F32)
    c = (rng.random((B, 3, M)) * 4 - 2).astype(F32)
    a[:, 2, ::5] = a[:, 2, 0:1]                      # duplicate depths
    if N > 6:
        a[0, 2, 3] = np.nan
        a[0, 2, 4], a[0, 2, 5] = np.inf, -np.inf
        c[0, 2, 0] = a[0, 2, 1] + F32(dz)              # at exactly zc - dis_z
    if M > 2:
        c[-1, 2, 1] = np.nan
        c[-1, 2, 2] = -np.inf
    return a, c


@pytest.mark.parametrize("B,N,M,K,dz", [(2, 50, 10, 4, 0.2), (1, 33, 5, 64, 0.5), (2, 31, 9, 3, 0.3),
                                        (3, 129, 17, 8, 0.4), (1, 1, 1, 1, 1.0), (2, 64, 8, 8, 1e-9)])
def test_restatement_matches_the_literal_loop(B, N, M, K, dz):
    """qdp_c (the restatement's query) equals oracle.qdp.qdp_loops, and the records, tiles and counts equal a plain
    loop over (b, t, l) in both row modes."""
    from oracle import qdp
    a, c = _edge_inputs(B * 100 + N, B, N, M, dz)
    for unique in (0, 1):
        ref = G.group_scale(a, c, dz, K, unique, 7)
        loop = G.group_scale(a, c, dz, K, unique, 7, qdp=qdp.qdp_loops)
        assert np.array_equal(ref.idx, loop.idx) and np.array_equal(ref.cnt, loop.cnt)
        assert ref.tiles == loop.tiles
        for b, exp in enumerate(_rows_loop(a, c, loop.idx, loop.cnt, unique)):
            assert exp.shape == ref.rows[b].shape
            assert G.record_bits_equal(ref.rows[b], exp).all()
            n = exp.shape[0]
            assert [t for t in ref.tiles if t[0] == b] == [(b, r0, min(7, n - r0)) for r0 in range(0, n, 7)]


def test_rounding_edges_are_rejected_by_the_rounded_predicate():
    """zc in [1, 2) has them below zc - 1 (z has the finer ulp); zc in [0.25, 0.5) only for some low bits of zc,
    above zc + 1."""
    fine = [F32(x) for x in np.linspace(0.26, 0.49, 64)]
    with_edges = [zc for zc in fine if G.rounding_edges(zc, 1.0)]
    assert 0 < len(with_edges) < len(fine)
    for zc in [F32(1.3), F32(1.05), F32(1.45)] + with_edges[:4]:
        edges = G.rounding_edges(zc, 1.0)
        assert edges, zc
        for z in edges:
            assert abs(float(zc) - float(z)) < 1.0 and abs(F32(zc - z)) == F32(1.0)
            idx, cnt = _query_one(z, zc, 1.0)
            assert cnt == 0


def _query_one(z, zc, dz):
    from oracle import qdp
    a = np.zeros((1, 3, 1), dtype=F32)
    a[0, 2, 0] = z
    c = np.zeros((1, 3, 1), dtype=F32)
    c[0, 2, 0] = zc
    idx, cnt = qdp.qdp_c(a, c, dz, 1)
    return idx, int(cnt[0, 0])


def test_feature_map_restatement():
    init = np.full((2, 7, 12), -3.5, dtype=F32)
    oh = np.array([[1, 0, 0], [0, 0.5, 2]], dtype=F32)
    f = G.feat_ref(init, 5, 8, oh, 3)
    assert (f[:, 5:] == -3.5).all() and (f[:, :5, :8] == 0).all() and (f[:, :5, 11] == 0).all()
    assert np.array_equal(f[:, :5, 8:11], np.broadcast_to(oh[:, None, :], (2, 5, 3)))
    assert (G.feat_ref(init, 5, 8, None, 3)[:, :5] == 0).all()


def test_shared_memory_rule():
    """The byte count that selects the bit-matrix kernel (T x ceil(N/32) words + 3T + T*K, largest scale)."""
    assert G.bitmask_bytes(1024, [517], [64]) == 204732 and G.uses_bitmask(1024, [517], [64])
    assert G.bitmask_bytes(1024, [518], [64]) == 205128 and not G.uses_bitmask(1024, [518], [64])
    assert G.bitmask_bytes(64, [2000], [8]) == 104000 and G.uses_bitmask(64, [2000], [8])
    assert not G.uses_bitmask(64, [2000], [8], force_scan=1)
    assert G.bitmask_bytes(1024, [517, 1], [64, 1]) == 204732


# ============================================================================ argument checks (no launch)
def _lib():
    from frustum_convnet_b200 import _lib as L
    return L


FAKE = 0x10000      # never dereferenced: every check below fails before the first CUDA call


def _valid_args(S=2, B=2, N=1024, T=(64, 32), K=(32, 16), force_scan=0):
    L = _lib()
    g = L.GroupArgs()
    g.num_scales, g.B, g.N, g.num_vec, g.tile_rows, g.unique_rows = S, B, N, 3, 64, 1
    g.pc, g.one_hot, g.ntiles, g.force_scan = FAKE, FAKE, FAKE, force_scan
    for s in range(S):
        g.centers[s], g.T[s], g.K[s], g.dis_z[s] = FAKE, T[s], K[s], 0.5
        g.c3[s], g.ld_feat[s], g.row_cap[s], g.tile_cap[s] = 8, 12, T[s] * K[s], 100
        g.rows[s], g.cnt[s], g.feat[s], g.tiles[s], g.idx_scratch[s] = FAKE, FAKE, FAKE, FAKE, FAKE
        g.feat_pitch[s] = T[s] + 1
    return g


def _expect_invalid(g, msg):
    L = _lib()
    lib = L.load()
    assert lib.fcn_group_rows(C.byref(g) if g is not None else None, None) == -1
    err = lib.fcn_last_error()
    assert msg.encode() in err, err


def _set(g, **kw):
    for k, v in kw.items():
        if isinstance(v, tuple):
            getattr(g, k)[v[0]] = v[1]
        else:
            setattr(g, k, v)
    return g


@pytest.mark.parametrize("change,msg", [
    (dict(num_scales=0), "num_scales out of range"),
    (dict(num_scales=9), "num_scales out of range"),
    (dict(B=-1), "bad B/N"),
    (dict(N=0), "bad B/N"),
    (dict(tile_rows=0), "tile_rows must be positive"),
    (dict(pc=None), "NULL pointer"),
    (dict(ntiles=None), "NULL pointer"),
    (dict(T=(1, 0)), "bad T/K"),
    (dict(K=(0, 0)), "bad T/K"),
    (dict(centers=(1, None)), "NULL per-scale pointer"),
    (dict(rows=(0, None)), "NULL per-scale pointer"),
    (dict(cnt=(1, None)), "NULL per-scale pointer"),
    (dict(tiles=(0, None)), "NULL per-scale pointer"),
    (dict(idx_scratch=(1, None)), "NULL idx_scratch"),
    (dict(row_cap=(1, 32 * 16 - 1)), "row_cap too small"),
    (dict(ld_feat=(0, 14)), "ld_feat must be a multiple of 4"),
    (dict(ld_feat=(1, 8)), "ld_feat too small"),
    (dict(B=65536), "grid too large"),
])
def test_each_check_fails_with_its_message(change, msg):
    _expect_invalid(_set(_valid_args(), **change), msg)


def test_null_args_and_staging_limit():
    _expect_invalid(None, "args is NULL")
    # T beyond the count + emit staging (5 ints per section in shared memory), on both selections of the path
    for fs in (0, 1):
        _expect_invalid(_valid_args(S=1, N=64, T=(10241,), K=(1,), force_scan=fs),
                        "T too large for the shared-memory staging")


@pytest.mark.parametrize("force_scan", [0, 1])
def test_null_idx_scratch_is_rejected_on_both_paths(force_scan):
    """idx_scratch is required whichever kernel the shape selects, so a caller that works at small shapes does not
    start failing when a larger shape switches to the count + emit pair."""
    assert G.uses_bitmask(1024, [64, 32], [32, 16])
    g = _valid_args(force_scan=force_scan)
    g.idx_scratch[0] = None
    _expect_invalid(g, "NULL idx_scratch")


def test_empty_batch_is_a_no_op():
    """B = 0 returns before any per-scale check or launch."""
    L = _lib()
    g = L.GroupArgs()
    g.num_scales, g.B, g.N, g.tile_rows, g.pc, g.ntiles = 3, 0, 16, 64, FAKE, FAKE
    assert L.load().fcn_group_rows(C.byref(g), None) == 0
