"""CPU: the exact-arithmetic references of tests/exact_ref.py restate the kernel contracts correctly.

The GPU tests compare kernels bit-exactly with these references, so the references themselves are pinned here
against independent formulations: float64 torch.nn.functional convolutions composed as ConvFeatNet does, a plain
per-section amax, and an integer implementation of the TF32 rounding."""
import pytest
import torch
import torch.nn.functional as F

import exact_ref as X


# ------------------------------------------------------------------ TF32 rounding
def test_tf32_rna_matches_integer_round_half_away():
    from frustum_convnet_b200.engine import tf32_rna
    g = torch.Generator().manual_seed(3)
    ints = torch.arange(-20000, 20001, dtype=torch.float32)                  # every tie of [2^11, 2^14)
    rnd = torch.randn(50000, generator=g) * torch.exp2(torch.randint(-30, 30, (50000,), generator=g).float())
    # exact ties and their neighbours at many exponents, both signs
    base = (torch.randint(1 << 23, 1 << 24, (5000,), generator=g) & ~0x1FFF).to(torch.int32)
    ties = torch.cat([base | 0x1000, base | 0x0FFF, base | 0x1001, base | 0x1FFF])
    ties = ties.to(torch.int32) | (torch.randint(1, 250, ties.shape, generator=g).to(torch.int32) << 23)
    ties = ties.view(torch.float32)
    x = torch.cat([ints, rnd, ties, -ties, torch.tensor([0.0, -0.0, 1.0, -1.0, 2047.0, 2049.0, -2049.0])])
    x = x[torch.isfinite(x)]
    got = tf32_rna(x).double()
    exp = torch.tensor([X.tf32_int_reference(float(v)) for v in x], dtype=torch.float64)
    assert torch.equal(got, exp)
    assert int(X.is_tie(x).sum()) >= 10000
    assert X.tf32_int_reference(2049.0) == 2050.0 and X.tf32_int_reference(-2049.0) == -2050.0     # away from 0
    assert X.tf32_int_reference(2051.0) == 2052.0 and X.tf32_int_reference(-4098.0) == -4100.0


# ------------------------------------------------------------------ generators honour their bounds
@pytest.mark.parametrize("regime", ["R1", "R2"])
@pytest.mark.parametrize("dims", [(64, 64, 128), (128, 128, 256), (256, 256, 512)])
def test_pointnet_generator_bounds(dims, regime):
    W = X.make_pointnet_weights(*dims, regime, seed=sum(dims))
    U = X.record_universe(W.coords.tolist())
    h1_pre = torch.relu(U @ W.w1t + W.b1)
    h1 = X.tf32(h1_pre)
    h2_pre = torch.relu(h1 @ W.w2t + W.b2)
    h2 = X.tf32(h2_pre)
    pre3 = h2 @ W.w3t
    lim = X.TF32_EXACT if regime == "R1" else X.EXACT_LIMIT
    # every partial sum: |partial| <= sum |a||w| + |b| over the whole record universe
    for a, w, b in ((U, W.w1t, W.b1), (h1, W.w2t, W.b2), (h2, W.w3t, W.b3)):
        assert float((a.abs() @ w.abs() + b.abs()).max()) < lim
    assert float((pre3 + W.b3).abs().max()) < lim
    for t in (h1_pre, h2_pre, pre3 + W.b3):
        assert torch.equal(t, torch.round(t)) and torch.equal(t.float().double(), t)
    if regime == "R1":
        assert torch.equal(h1, h1_pre) and torch.equal(h2, h2_pre)
    else:
        # the rounding points really round, and some inputs of the rounding are exact ties
        assert not torch.equal(h1, h1_pre) and not torch.equal(h2, h2_pre)
        assert X.is_tie(h1_pre).any() and X.is_tie(h2_pre).any() and X.is_tie(pre3 + W.b3).any()
    # the (0,0,0) record of the all-negative sections: every pre-activation <= 0
    zero = X.pointnet_row_values(torch.zeros(1, 3, dtype=torch.float64), W)
    assert (zero <= 0).all()


def test_generator_bound_assertion_fires():
    g = torch.Generator().manual_seed(0)
    w = X.sparse_ints(g, 64, 8, 64, 4)
    with pytest.raises(AssertionError):
        X.check_bound(torch.full((64,), 70000.0), w, None, X.EXACT_LIMIT, "too large")


# ------------------------------------------------------------------ PointNet reference
def _small_case(regime, tile_rows=128, cuts=(128, 7, 65, 1, 9, 64, 8, 63, 127)):
    W = X.make_pointnet_weights(64, 64, 128, regime, seed=5)
    lens = [(n, "pos") for n in list(range(1, 21)) + [31, 32, 33, 0, 63, 64, 65]] + [(12, "neg"), (3, "pos")]
    return X.make_pointnet_case(W, [lens, lens[::-1], lens[5:]], tile_rows, cuts, seed=9)


@pytest.mark.parametrize("regime", ["R1", "R2"])
def test_pointnet_reference_equals_per_section_amax(regime):
    case = _small_case(regime)
    fast = X.pointnet_pooled_ref(case)
    loop = X.pointnet_pooled_loop_ref(case)
    assert X.bits_equal(fast, loop)
    # plain float64 torch per-section amax straight from the row records of the tiles
    C3 = case.W.dims[2]
    exp = case.feat_init.clone()
    rows_i = case.rows.view(torch.int32)
    recs = {}
    for b, row0, n, _ in case.tiles[:case.ntiles].tolist():
        for r in range(row0, row0 + n):
            recs.setdefault((b, int(rows_i[b, r, 3])), []).append(case.rows[b, r, :3].double())
    for (b, t), xs in recs.items():
        xyz = torch.stack(xs)
        h1 = X.tf32(torch.relu(xyz @ case.W.w1t + case.W.b1))
        h2 = X.tf32(torch.relu(h1 @ case.W.w2t + case.W.b2))
        v = X.tf32(h2 @ case.W.w3t + case.W.b3).amax(0).clamp(min=0)
        exp[b, t, :C3] = v.float()
    assert X.bits_equal(fast, exp)


def test_pointnet_case_layout():
    case = _small_case("R1")
    C3 = case.W.dims[2]
    t = case.tiles
    assert case.ntiles < t.shape[0]                                      # decoys past ntiles
    assert set(t[:case.ntiles, 2].tolist()) >= {1, 7, 8, 9, 63, 64, 65, 127, 128}
    assert (t[:case.ntiles, 1] % case.tile_rows == 0).all()
    # slots past a tile's nrows hold NaN; records inside are finite
    for b, row0, n, _ in t[:case.ntiles].tolist():
        assert torch.isfinite(case.rows[b, row0:row0 + n]).all()
        assert torch.isnan(case.rows[b, row0 + n:row0 + case.tile_rows, :3]).all()
    # the decoys would change the result if they were processed
    full = X.PointnetCase(**{**case.__dict__, "ntiles": t.shape[0]})
    assert not X.bits_equal(X.pointnet_pooled_ref(full), X.pointnet_pooled_ref(case))
    # sentinel everywhere outside [valid rows x C3], sections without rows and all-negative sections stay 0
    ref = X.pointnet_pooled_ref(case)
    assert (ref[:, case.T:] == X.SENTINEL).all() and (ref[:, :, C3:] == X.SENTINEL).all()
    for b, secs in enumerate(case.sections):
        for ti, (n, kind) in enumerate(secs):
            if n == 0 or kind == "neg":
                assert (ref[b, ti, :C3] == 0).all()
            else:
                assert (ref[b, ti, :C3] > 0).any()
    # every section of <= 16 rows: each row position is the strict arg-max of some channel
    for per in case.sect_rows:
        for ti, xyz in per:
            if xyz.shape[0] <= 16 and xyz.abs().sum() > 0:
                assert X.argmax_covers(X.pointnet_row_values(xyz, case.W))


# ------------------------------------------------------------------ conv reference vs torch.nn.functional
def _fcn_like(B, T, seed):
    """A ConvFeatNet-shaped chain in float64: conv k3 s1 -> conv k3 s2 -> merge (cat + 1x1) -> deconv + crop."""
    g = torch.Generator().manual_seed(seed)
    C0, C1, C2, Cf, Cd, up = 37, 64, 32, 45, 32, 4
    x = X._ints(g, -3, 3, (B, C0, T))
    f2 = X._ints(g, -3, 3, (B, Cf, (T + 1) // 2))
    w1 = X._ints(g, -1, 1, (C1, C0, 3)); b1 = X._ints(g, -5, 5, (C1,))
    w2 = X._ints(g, -1, 1, (C2, C1, 3)); b2 = X._ints(g, -5, 5, (C2,))
    wm = X._ints(g, -1, 1, (C2, C2 + Cf, 1)); bm = X._ints(g, -5, 5, (C2,))
    wd = X._ints(g, -1, 1, (C2, Cd, up)); bd = X._ints(g, -5, 5, (Cd,))
    return x, f2, (w1, b1), (w2, b2), (wm, bm), (wd, bd), up


def _to_pm(x_bct, pitch, ld, garbage=0.0):
    """(B, C, T) channel-first -> (B, pitch, ld) position-major, zero pad rows, channel pad = garbage."""
    B, Cc, T = x_bct.shape
    out = torch.zeros(B, pitch, ld, dtype=torch.float64)
    out[:, :T, :Cc] = x_bct.permute(0, 2, 1)
    out[:, :T, Cc:] = garbage
    return out


def _pad32(c):
    return (c + 31) // 32 * 32


def test_conv_reference_matches_torch_conv_composition():
    B, T = 3, 23
    x, f2, (w1, b1), (w2, b2), (wm, bm), (wd, bd), up = _fcn_like(B, T, seed=1)
    # torch (float64), as ConvFeatNet composes it
    y1 = torch.relu(F.conv1d(x, w1, b1, stride=1, padding=1))
    y2 = torch.relu(F.conv1d(y1, w2, b2, stride=2, padding=1))
    ym = torch.relu(F.conv1d(torch.cat([y2, f2], 1), wm, bm))
    yd = torch.relu(F.conv_transpose1d(ym, wd, bd, stride=up))
    T2 = (T + 1) // 2
    T_store = T2 * up - 3                                                # crop
    # the same chain through conv_ref on position-major maps with pads and channel garbage
    P1 = 2 * (T2 + 1)
    xm = _to_pm(x, P1, 40, garbage=1e30)

    def k3(w):
        ci = w.shape[1]
        wt = torch.zeros(3 * _pad32(ci), 64, dtype=torch.float64)
        for j in range(3):
            wt[j * _pad32(ci): j * _pad32(ci) + ci, :w.shape[0]] = w[:, :, j].t()
        return wt

    def bias(b, n):
        out = torch.zeros(n, dtype=torch.float64)
        out[:b.shape[0]] = b
        return out

    spec1 = X.ConvSpec(B, T, P1, [X.ConvSeg(xm, 37, T, j - 1, 1) for j in range(3)], k3(w1), bias(b1, 64),
                       64, 1, 1, 0, torch.zeros(B, P1, 64, dtype=torch.float64), T, 0)
    for s in spec1.segs:
        s.src = xm
    a1 = X.conv_ref(spec1).double()
    assert torch.equal(a1[:, :T].permute(0, 2, 1), y1)
    spec2 = X.ConvSpec(B, T2, P1 // 2, [X.ConvSeg(a1, 64, T, j - 1, 2) for j in range(3)], k3(w2), bias(b2, 64),
                       32, 1, 1, 0, torch.zeros(B, P1 // 2, 32, dtype=torch.float64), T2, 0)
    a2 = X.conv_ref(spec2).double()
    assert torch.equal(a2[:, :T2].permute(0, 2, 1), y2)
    fm = _to_pm(f2, P1 // 2, 48, garbage=1e30)
    wt = torch.zeros(32 + 64, 64, dtype=torch.float64)
    wt[:32, :32] = wm[:, :32, 0].t()
    wt[32:32 + 45, :32] = wm[:, 32:, 0].t()
    spec3 = X.ConvSpec(B, T2, P1 // 2, [X.ConvSeg(a2, 32, T2, 0, 1), X.ConvSeg(fm, 45, T2, 0, 1)], wt,
                       bias(bm, 64), 32, 1, 1, 0, torch.zeros(B, P1 // 2, 32, dtype=torch.float64), T2, 0)
    a3 = X.conv_ref(spec3).double()
    assert torch.equal(a3[:, :T2].permute(0, 2, 1), ym)
    wt = torch.zeros(32, 128, dtype=torch.float64)
    bb = torch.zeros(128, dtype=torch.float64)
    for j in range(up):
        wt[:, j * 32:(j + 1) * 32] = wd[:, :, j]
        bb[j * 32:(j + 1) * 32] = bd
    c_off, ld_out = 8, 48
    init = torch.full((B, up * (P1 // 2), ld_out), float("nan"), dtype=torch.float64)
    spec4 = X.ConvSpec(B, T2, P1 // 2, [X.ConvSeg(a3, 32, T2, 0, 1)], wt, bb, 32, up, 1, 0, init, T_store, c_off)
    a4 = X.conv_ref(spec4)
    assert torch.equal(a4[:, :T_store, c_off:c_off + 32].double().permute(0, 2, 1), yd[:, :, :T_store])
    # the store mask: everything else keeps the sentinel
    keep = torch.ones_like(a4, dtype=torch.bool)
    keep[:, :T_store, c_off:c_off + 32] = False
    assert torch.isnan(a4[keep]).all()
    # relu = 0, round_out on an R2-sized result
    spec4.relu, spec4.round_out = 0, 1
    spec4.wt = spec4.wt * 700
    a5 = X.conv_ref(spec4)
    raw = F.conv_transpose1d(ym, wd * 700, bd, stride=up)[:, :, :T_store]
    assert torch.equal(a5[:, :T_store, c_off:c_off + 32].double().permute(0, 2, 1), X.tf32(raw))
    assert not torch.equal(X.tf32(raw), raw)
