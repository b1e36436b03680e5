"""GPU: fcn_conv_gemm called directly, compared BIT-EXACTLY with the float64 reference of tests/exact_ref.py.

The same fcn_conv_args run through every variant: precision 0 (fp32 SIMT), 1 / 2 (wgmma, cp.async gather, N tile
128 / 64) and 3 / 4 (wgmma, TMA-fed, N tile 128 / 64).  Integer operands keep every partial sum exact (R1: outputs
< 2^11, TF32 rounding is the identity, all five variants; R2: outputs really round, TF32 variants).  The cases
cover k=3 convs with stride 1 and 2 over odd and even lengths, concat segments whose K stages straddle a segment
boundary, a trailing all-zero K block, transposed convs with up = 2/4/8, an output channel offset and a crop, a
heads-like layer (no ReLU, no rounding, 32 skipped columns), GEMM row counts around the 128-row tile and a batch
whose second warpgroup has no valid row.  The source channel pad holds 1e30 (read against zero weights) and the
output buffer starts as NaN: every element outside the stored slice must keep it."""
import pytest
import torch

import exact_ref as X

pytestmark = pytest.mark.gpu

GARBAGE = 1e30


def dev():
    return torch.device("cuda:0")


def _pad32(c):
    return (c + 31) // 32 * 32


def _source(g, B, T_src, pitch, C, ld, amax):
    """(B, pitch, ld): integers in [-amax, amax] on the valid rows and channels, GARBAGE in the channel pad,
    zero pad rows (the engine keeps them zero)."""
    s = torch.zeros(B, pitch, ld, dtype=torch.float64)
    s[:, :T_src, :C] = X._ints(g, -amax, amax, (B, T_src, C))
    s[:, :T_src, C:] = GARBAGE
    return s


# name: (B, [(C, ld, tap, stride)...] sharing one source when `shared`, T_src, pitch, Cout, up, relu, round_out,
#        n_cols, T_store or None, c_off, ld_out)
CASES = {
    # k=3 stride 1, odd length, channel pad, B*P_m = 120
    "k3_s1_odd": dict(B=3, segs=[(61, 64, t, 1) for t in (-1, 0, 1)], shared=True, T_src=37, pitch=40, Cout=128),
    # k=3 stride 1, even length, B*P_m = 130
    "k3_s1_even": dict(B=2, segs=[(128, 128, t, 1) for t in (-1, 0, 1)], shared=True, T_src=64, pitch=65, Cout=128),
    # k=3 stride 2, odd length: T_out = 43 = P_m, B*P_m = 129
    "k3_s2_odd": dict(B=3, segs=[(64, 64, t, 2) for t in (-1, 0, 1)], shared=True, T_src=85, pitch=86, Cout=128),
    # k=3 stride 2, even length: B*P_m = 128
    "k3_s2_even": dict(B=4, segs=[(96, 100, t, 2) for t in (-1, 0, 1)], shared=True, T_src=62, pitch=64, Cout=256),
    # merge 128 + 131 (ld 128, 132): K 128 + 160, a trailing all-zero K block; B*P_m = 305
    "merge_128_131": dict(B=5, segs=[(128, 128, 0, 1), (131, 132, 0, 1)], shared=False, T_src=60, pitch=61,
                          Cout=128, K_extra=32),
    # merge 96 + 131: the second 64-wide stage straddles the two segments; B = 1, T_out = 5: the second
    # warpgroup has no valid row
    "merge_96_131": dict(B=1, segs=[(96, 100, 0, 1), (131, 132, 0, 1)], shared=False, T_src=5, pitch=6, Cout=128),
    # transposed convs: pixel shuffle, output channel offset, crop, P_store = up * P_m
    "deconv_up2": dict(B=1, segs=[(128, 128, 0, 1)], shared=True, T_src=126, pitch=127, Cout=128, up=2,
                       T_store=2 * 126 - 1, c_off=64, ld_out=64 + 128 + 32),
    "deconv_up4": dict(B=2, segs=[(64, 64, 0, 1)], shared=True, T_src=30, pitch=32, Cout=64, up=4,
                       T_store=4 * 30 - 3, c_off=32, ld_out=128),
    "deconv_up8": dict(B=3, segs=[(45, 48, 0, 1)], shared=True, T_src=42, pitch=43, Cout=32, up=8,
                       T_store=8 * 42 - 7, c_off=128, ld_out=192),
    # heads-like: no ReLU, no rounding, Cout = 96 of n_cols = 128 (columns 96..127 skipped); B*P_m = 315
    "heads": dict(B=7, segs=[(200, 204, 0, 1)], shared=True, T_src=44, pitch=45, Cout=96, n_cols=128, relu=0,
                  round_out=0),
}

# amax of the sources, |w|, |b| per regime (R1: every output < 2^11; R2: outputs well above 2^11, exact sums)
REGIMES = {"R1": (3, 1, 8), "R2": (1500, 3, 1000)}


def make_spec(name, regime, seed=0):
    c = dict(CASES[name])
    amax, wmax, bmax = REGIMES[regime]
    g = torch.Generator().manual_seed(seed + 1000 * list(CASES).index(name) + len(regime))
    B, T_src, pitch = c["B"], c["T_src"], c["pitch"]
    up, Cout = c.get("up", 1), c["Cout"]
    stride = c["segs"][0][3]
    P_m = pitch // stride
    T_out = T_src if stride == 1 else (T_src + 1) // 2
    srcs, segs = [], []
    for j, (Cc, ld, tap, st) in enumerate(c["segs"]):
        if c["shared"] and srcs:
            src = srcs[0]
        else:
            src = _source(g, B, T_src, pitch, Cc, ld, amax)
            srcs.append(src)
        segs.append(X.ConvSeg(src, Cc, T_src, tap, st))
    K = sum(_pad32(s.C) for s in segs)
    K_pad = (K + 63) // 64 * 64
    assert K_pad - K == c.get("K_extra", K_pad - K)
    n_cols = c.get("n_cols", (up * Cout + 63) // 64 * 64)
    wt = torch.zeros(K_pad, n_cols, dtype=torch.float64)
    k = 0
    for s in segs:
        wt[k:k + s.C] = X._ints(g, -wmax, wmax, (s.C, n_cols))
        k += _pad32(s.C)
    bias = X._ints(g, -bmax, bmax, (n_cols,))
    relu, round_out = c.get("relu", 1), c.get("round_out", 1 if regime == "R2" else 0)
    T_store = c.get("T_store") or T_out
    ld_out, c_off = c.get("ld_out", Cout), c.get("c_off", 0)
    out = torch.full((B, up * P_m, ld_out), float("nan"), dtype=torch.float64)
    spec = X.ConvSpec(B, T_out, P_m, segs, wt, bias, Cout, up, relu, round_out, out, T_store, c_off)
    X.conv_operand_bound(spec, X.TF32_EXACT if regime == "R1" else X.EXACT_LIMIT)
    return spec


PARAMS = [pytest.param(n, p, r, id="%s-p%d-%s" % (n, p, r))
          for n in CASES for r in ("R1", "R2") for p in ((0, 1, 2, 3, 4) if r == "R1" else (1, 2, 3, 4))]


@pytest.mark.parametrize("name,precision,regime", PARAMS)
def test_conv_gemm_exact(name, precision, regime):
    spec = make_spec(name, regime)
    exp = X.conv_ref(spec)
    if regime == "R2" and spec.round_out:
        _, pre, _ = X.conv_ref(spec, with_abs=True)
        assert (pre.abs() >= X.TF32_EXACT).any()            # the rounding is exercised
    got = X.ConvLaunch(spec, precision, dev()).run()
    assert X.bits_equal(got, exp), "%s p%d %s:\n%s" % (name, precision, regime, X.describe_mismatch(got, exp))
