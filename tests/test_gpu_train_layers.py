"""GPU: the training kernels of csrc/train.cu through their C ABI (fcn_train_forward / _backward / _pool /
_finalize, fcn_adam_step), layer by layer, against the float64 reference of tests/train_ref.py computed from the
kernel call's own inputs.

Exact regime (small integers, every partial sum < 2^22: fp32 accumulation is exact in any order): Y, dW, dX,
dbias and the dsums of layers without BN are compared BIT-EXACTLY.  Gradient buffers start non-zero (the kernels
accumulate) and every element a call must not touch starts as NaN and must keep its bits.

BN regime (random floats) bounds, from the kernels' arithmetic:
  * statistics, from the kernel's own Y: every fp32 partial chain has at most 128 terms before the fp64 atomics,
    so |dSum y| <= 2^-17 * Sum|y| and |dSum y^2| <= 2^-17 * Sum y^2;  the variance derived from them then has
    |dvar| <= 2^-16 * E[y^2], which contains the cancellation term E[y^2] - mean^2 (a channel with mean/std = 100
    is part of the cases);
  * contractions of length K (Y: K = sum of segment channels, dW: K = rows, dX: K = columns):
    |delta| <= (K + 8) * 2^-23 * sum_k |a_k| |b_k|, with |a| = |x||scale| + |beta| + |mean*scale| of the source
    operand and |b| = |scale| (|dz| + |m1| + (|y| + |mean|) invstd |m2|) of the BN backward (+8: the fp32
    evaluation of those operands and of the final accumulation into a non-zero buffer, whose |value| is added to
    the sum);
  * reductions (dsums): as the statistics, 2^-17 * sum of |terms|.
Generated BN data keeps every pre-activation at least 1e-4 * (|y*scale| + |shift|) away from 0 (resampled), so
ReLU masks are unambiguous; real model data (the TrainEngine cases) cannot, and the few elements whose ReLU decision
is within rounding of 0 add their whole contribution to the bound.

Adam (f), u = 2^-24, G = |g|*grad_scale + wd*|p| (the magnitude of the two terms of g' = g*grad_scale + wd*p,
which may cancel, so |dg'| <= 2u*G):
  * exp_avg  m' = b1*m + (1-b1)*g'  ((1-b1) is exact): |dm'| <= 3u*(b1|m| + G) + |dg'| <= 5u*(b1|m| + G),
    tested as 4 ulp(m') + 8u*(b1|m| + G);
  * exp_avg_sq  v' = b2*v + (1-b2)*g'^2: non-negative terms, relative error <= 4u, plus (1-b2)*2|g'||dg'|
    <= 4u*(1-b2)*G^2 from g': tested as 8 ulp(v') + 16u*(1-b2)*G^2;
  * the update lr/bc1 * m'/(sqrt(v')/sqrt(bc2) + eps): with sc = lr/bc1 * (b1|m| + (1-b1)G)/denom >= |update|,
    the error of m' contributes <= 5u*sc, the correlated error of sqrt(v') (g' in numerator and denominator)
    <= 4u*sc, and the seven remaining fp32 operations (sqrtf, divisions, products, the sum with eps) <= 7u*|update|:
    about 16u*sc, tested as 64u*sc = 2^-18*sc.  bc1 = 1 - powf(b1, step) and bc2 likewise: CUDA's powf is within
    4 ulp, so bc1 is off by up to 2^-21 * b1^step / bc1 relative (and sqrt(bc2) by half of that for b2); that
    relative error times |update| is added.  The rounding of p' = p - update itself and a floor: 4 ulp(p') +
    1e-6*lr.
"""
import ctypes as C
import math
import zlib

import pytest
import torch

import train_ref as tr
from exact_ref import bits_equal, describe_mismatch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _lib():
    from frustum_convnet_b200 import _lib
    return _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _forward(L, ws=None, wsn=0):
    _lib().call("fcn_train_forward", C.byref(L), ws.data_ptr() if ws is not None else None, wsn, _stream())
    torch.cuda.synchronize()


def _backward(L, mask):
    _lib().call("fcn_train_backward", C.byref(L), mask, _stream())
    torch.cuda.synchronize()


def _assert_bits(got, exp, what):
    assert bits_equal(got, exp), what + ": " + describe_mismatch(got.cpu(), exp.cpu())


def _assert_within(got, exp, tol, what):
    err = (got.double() - exp.double()).abs()
    bad = ~(err <= tol)
    if bad.any():
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError("%s: %d of %d elements out of bound; first at %d: got %r expected %r tol %r" % (
            what, int(bad.sum()), err.numel(), i, float(got.reshape(-1)[i]), float(exp.reshape(-1)[i]),
            float(tol.reshape(-1)[i])))


def _seg_K(L):
    return sum(L.seg[j].C for j in range(L.n_seg))


# ============================================================================ (a) exact regime, generic kernels
def _exact_cases():
    S = tr.SrcDesc
    c = {}
    c["k3s1_M1_N2_bias"] = tr.conv1d_layer(1, 1, [S(1, 19)], 19, 2, 3, bias=True)
    c["k3s1_M63_N39_bias"] = tr.conv1d_layer(3, 21, [S(21, 35)], 35, 39, 3, bias=True)
    c["k3s2_oddT_M64_N64"] = tr.conv1d_layer(2, 63, [S(63, 19)], 19, 64, 3, stride=2)
    c["k3s2_evenT_M65_N96"] = tr.conv1d_layer(5, 26, [S(26, 21)], 21, 96, 3, stride=2)
    c["k3s1_M129_N64_bn"] = tr.conv1d_layer(3, 43, [S(43, 50)], 50, 64, 3, has_bn=1, relu=1)
    c["concat2_M129_N39"] = tr.concat_layer(3, 43, [S(43, 19), S(43, 30)], [19, 30], 39, bias=True)
    c["concat4_M65_N96"] = tr.concat_layer(1, 65, [S(65, 7), S(65, 23), S(65, 11), S(65, 40)], [7, 23, 11, 40], 96)
    for up, T, cup in ((2, 20, 24), (4, 9, 16), (8, 5, 8)):
        # pixel-shuffled source with a crop (T_out < T*up) and a channel offset
        c["up%d_crop_c0" % up] = tr.concat_layer(2, T * up - 3, [S(T, 5 + up * cup + 3, up=up, cup=cup, c0=5)],
                                                 [cup], 39, bias=True)
    for up, co in ((2, 32), (4, 24), (8, 8)):
        c["deconv%d_layout" % up] = tr.deconv_layer(2, 33, [S(33, 20)], 20, co, up)
    return c


EXACT = _exact_cases()
# three segments, two of them at channel offsets (c0 != 0), one source without a gradient buffer
EXACT["concat3_c0_nograd"] = tr.LayerDesc(
    2, 32, 64, 64, [tr.SegDesc(0, 13, 0, 1, 1, 0), tr.SegDesc(1, 18, 0, 1, 1, 13), tr.SegDesc(2, 9, 0, 1, 1, 31)],
    [tr.SrcDesc(32, 37), tr.SrcDesc(32, 37, c0=15), tr.SrcDesc(32, 12, c0=3, grad=False)], s_co=40)


def _seed(name):
    return zlib.crc32(name.encode()) % 100003


def _workspaces(L):
    need = int(_lib().load().fcn_train_workspace_floats(C.byref(L)))
    M = L.B * L.T_out
    out = [("null", None, 0), ("too_small", torch.empty(M * L.N, device=DEV), M * L.N)]
    if need:
        out.append(("exact", torch.empty(need, device=DEV), need))
        out.append(("larger", torch.empty(2 * need + 7, device=DEV), 2 * need + 7))
    return need, out


@pytest.mark.parametrize("name", sorted(EXACT))
def test_exact_forward_is_bit_exact_with_every_workspace(name):
    case = tr.LayerCase(EXACT[name], DEV)
    L = tr.exact_fill(case, seed=_seed(name))
    exp = tr.forward_ref(L, case.mem)[0].float()
    need, wss = _workspaces(L)
    for wname, ws, n in wss:
        case.Y.fill_(float("nan"))
        _forward(L, ws, n)
        _assert_bits(case.Y, exp, "%s Y (workspace %s, %d floats)" % (name, wname, n))
    if need:
        ws = torch.empty(need, device=DEV)
        _forward(L, ws, need)
        first = case.Y.clone()
        _forward(L, ws, need)
        _assert_bits(case.Y, first, "two runs with the same workspace")


@pytest.mark.parametrize("mask", ["all", "skip_first", "none"])
@pytest.mark.parametrize("name", sorted(n for n in EXACT if not EXACT[n].has_bn))    # BN backward: BN regime
def test_exact_backward_accumulates_bit_exactly(name, mask):
    d = EXACT[name]
    case = tr.LayerCase(d, DEV)
    L = tr.exact_fill(case, seed=_seed(name) + 1)
    full = (1 << len(d.segs)) - 1
    m = {"all": full, "skip_first": full & ~1, "none": 0}[mask]
    _forward(L)
    tr.prefill_grads(case, full, seed=5)          # every segment's region non-zero, the rest NaN
    g0 = [b["grad"].clone() if b["grad"] is not None else None for b in case.src]
    dW0 = case.dW.clone()
    case.dsums.fill_(0)
    _backward(L, m)
    dy = tr.dy_ref(L, case.mem)
    ds, _, _ = tr.reduce_ref(L, case.mem, dy)
    _assert_bits(case.dsums[:L.N].float(), ds.float(), name + " dsums")
    exp_dW = dW0.double()
    for j in range(L.n_seg):
        widx, v, _, _ = tr.dw_ref(L, j, case.mem, dy)
        exp_dW.index_add_(0, widx.reshape(-1), v.reshape(-1))
    _assert_bits(case.dW, exp_dW.float(), name + " dW (+= onto the bucket, NaN outside the layout)")
    for i, b in enumerate(case.src):
        if b["grad"] is None:
            continue
        exp = g0[i].double().reshape(-1).clone()
        for j, sg in enumerate(d.segs):
            if sg.src == i and (m >> j) & 1:
                idx, v, _, _ = tr.dx_ref(L, j, case.mem, dy)
                exp.index_add_(0, idx.reshape(-1), v.reshape(-1))
        _assert_bits(b["grad"], exp.float().view_as(b["grad"]), "%s dX source %d (mask %s)" % (name, i, mask))


# ============================================================================ (b) BN regime, plain and generic
def _bn_cases():
    S = tr.SrcDesc

    def plain(B, T, Cc, N, stats=True, coff=0):
        return tr.concat_layer(B, T, [S(T, Cc, stats=stats, Cstat=Cc, coff=coff)], [Cc], N, has_bn=1, relu=1)

    c = {
        "plain_C64_N64_M128": plain(2, 64, 64, 64),
        "plain_C64_N512_M127": plain(1, 127, 64, 512),
        "plain_C512_N64_M129": plain(3, 43, 512, 64),
        "plain_C512_N512_M256": plain(4, 64, 512, 512),
        "plain_C128_N128_M1500": plain(3, 500, 128, 128),
        "plain_C64_N128_M4500": plain(9, 500, 64, 128),
        "plain_nostats_M257": plain(1, 257, 64, 64, stats=False),
        "plain_coff_wrap": plain(2, 100, 64, 64, coff=5),
        "fallback_C576_N64": plain(2, 100, 576, 64),
        "fallback_C64_N576": plain(2, 100, 64, 576),
        "k3s2_src_norelu": tr.conv1d_layer(2, 31, [S(31, 40, stats=True, Cstat=40, relu=0)], 40, 48, 3, stride=2,
                                           has_bn=1, relu=1),
        "k3s1_src_nostats": tr.conv1d_layer(3, 20, [S(20, 24)], 24, 40, 3, has_bn=1, relu=1),
        "coff_Cstat_wrap": tr.concat_layer(2, 30, [S(30, 40, stats=True, Cstat=24, coff=17)], [40], 64, has_bn=1,
                                           relu=1),
        "concat_bn_and_plain_src": tr.concat_layer(2, 45, [S(45, 70, stats=True, Cstat=70), S(45, 9)], [70, 9], 96,
                                                   has_bn=1, relu=1),
        "wide_mean_src": tr.concat_layer(2, 60, [S(60, 48, stats=True, Cstat=48)], [48], 64, has_bn=1, relu=1),
        "wide_mean_layer": tr.concat_layer(2, 200, [S(200, 40)], [40], 64, has_bn=1, relu=1),
    }
    for up, co in ((2, 32), (4, 24), (8, 16)):
        c["deconv%d_bn" % up] = tr.deconv_layer(2, 20, [S(20, 48, stats=True, Cstat=48)], 48, co, up, has_bn=1, relu=1)
    return c


BN = _bn_cases()


def _bn_fill(case, name, seed):
    d = case.d
    g = torch.Generator().manual_seed(seed)
    for i, s in enumerate(d.srcs):
        if s.stats:
            tr.bn_source_fill(case, i, seed + i, wide_channel=(3 if name == "wide_mean_src" else None))
        else:
            case.src[i]["raw"].copy_(torch.randn(case.src[i]["raw"].shape, generator=g))
    nw = case.W.numel()
    case.W.fill_(float("nan"))
    case.dW.fill_(float("nan"))
    for sg in d.segs:
        widx = tr.weight_index_d(d, sg).reshape(-1)
        case.W[widx.to(DEV)] = (torch.randn(widx.numel(), generator=g) / math.sqrt(sum(x.C for x in d.segs))).to(DEV)
        case.dW[widx.to(DEV)] = torch.randn(widx.numel(), generator=g).to(DEV)
    if name == "wide_mean_layer":
        # input channel 0 ~ 100 + N(0,1) feeds output channel 0 with weight 1: that channel has mean/std ~ 100
        case.src[0]["raw"][:, 0] += 100.0
        w0 = tr.weight_index_d(d, d.segs[0])
        case.W[w0[:, 0].to(DEV)] = (torch.randn(w0.shape[0], generator=g) * 0.01).to(DEV)
        case.W[int(w0[0, 0])] = 1.0
    sign = torch.where(torch.rand(d.Cout, generator=g) < 0.2, -1.0, 1.0)
    case.gamma.copy_((torch.rand(d.Cout, generator=g) + 0.5) * sign)
    case.beta.copy_(torch.rand(d.Cout, generator=g) - 0.5)
    case.dA.copy_(torch.randn(case.dA.shape, generator=g))
    assert nw


def _check_stats(L, case, what):
    got = case.sums
    exp, scale = tr.stats_ref(L, case.Y)
    _assert_within(got, exp, tr.sum_tol(scale), what + " Sum(y), Sum(y^2)")
    cnt = tr.bn_count(L)
    C_ = L.Cout
    mean_k, mean_r = got[:C_] / cnt, exp[:C_] / cnt
    var_k = got[C_:] / cnt - mean_k ** 2
    var_r = exp[C_:] / cnt - mean_r ** 2
    _assert_within(var_k, var_r, 2.0 ** -16 * exp[C_:] / cnt, what + " variance (cancellation bound)")


@pytest.mark.parametrize("name", sorted(BN))
def test_bn_layer_forward_backward_within_bounds(name):
    d = BN[name]
    case = tr.LayerCase(d, DEV)
    L = case.layer()
    _bn_fill(case, name, seed=_seed(name))
    ws_n = int(_lib().load().fcn_train_workspace_floats(C.byref(L)))
    ws = torch.empty(max(ws_n, 1), device=DEV)
    case.sums.zero_()
    _forward(L, ws, ws_n)
    Y, S = tr.forward_ref(L, case.mem)
    _assert_within(case.Y, Y, tr.contraction_tol(_seg_K(L), S), name + " Y")
    _check_stats(L, case, name)
    if name == "wide_mean_layer":
        m = case.Y[:, 0].double()
        assert float(m.mean() / m.std()) > 50, "the wide channel lost its mean/std ratio"
    # backward: Y is an input; keep its ReLU decisions unambiguous under the kernel's own statistics
    tr.keep_relu_margin(L, case.mem, seed=1)
    full = (1 << len(d.segs)) - 1
    tr.prefill_grads(case, full, seed=7, ints=False)
    g0 = [b["grad"].clone() if b["grad"] is not None else None for b in case.src]
    dW0 = case.dW.clone()
    case.dsums.zero_()
    _backward(L, full)
    dy = tr.dy_ref(L, case.mem)
    assert dy["namb"] == 0
    ds, dss, _ = tr.reduce_ref(L, case.mem, dy)
    _assert_within(case.dsums, ds, tr.sum_tol(dss), name + " dsums")
    exp_dW, S_dW = dW0.double(), dW0.double().abs()
    for j in range(L.n_seg):
        widx, v, a, _ = tr.dw_ref(L, j, case.mem, dy)
        exp_dW.index_add_(0, widx.reshape(-1), v.reshape(-1))
        S_dW.index_add_(0, widx.reshape(-1), a.reshape(-1))
    M = L.B * L.T_out
    nanw = torch.isnan(dW0)
    assert torch.isnan(case.dW[nanw]).all(), name + " dW outside the layout was written"
    _assert_within(case.dW[~nanw], exp_dW[~nanw], tr.contraction_tol(M, S_dW[~nanw]), name + " dW")
    for i, b in enumerate(case.src):
        if b["grad"] is None:
            continue
        exp, Sx = g0[i].double().reshape(-1).clone(), g0[i].double().reshape(-1).abs()
        for j, sg in enumerate(d.segs):
            if sg.src == i:
                idx, v, a, _ = tr.dx_ref(L, j, case.mem, dy)
                exp.index_add_(0, idx.reshape(-1), v.reshape(-1))
                Sx.index_add_(0, idx.reshape(-1), a.reshape(-1))
        got = b["grad"].reshape(-1)
        nan = torch.isnan(g0[i].reshape(-1))
        assert torch.isnan(got[nan]).all(), "%s dX wrote outside its region" % name
        _assert_within(got[~nan], exp[~nan], tr.contraction_tol(L.N, Sx[~nan]),
                       "%s dX of source %d accumulated onto a non-zero gradient" % (name, i))


# ============================================================================ (d) pooling
def _pool_case(B, T, K, Cc, V, seed):
    g = torch.Generator().manual_seed(seed)
    BT = B * T
    y = torch.randint(-512, 513, (BT, K, Cc), generator=g).float() / 64
    # bit-identical duplicate rows (the back-fill duplicates of the grouping): ties -> first index
    y[:, K - 1] = y[:, 1]
    y[::3, 2] = y[::3, 0]
    cnt = torch.randint(1, K + 1, (BT,), generator=g, dtype=torch.int32)
    cnt[1::4] = 0
    count = float(BT * K)
    var = torch.rand(Cc, generator=g, dtype=torch.float64) * 1.5 + 0.5
    sums = torch.cat([torch.zeros(Cc, dtype=torch.float64), var * count])     # mean 0: shift = beta exactly
    sign = torch.where(torch.rand(Cc, generator=g) < 0.3, -1.0, 1.0)
    gamma = (torch.randint(1, 9, (Cc,), generator=g).float() / 4) * sign
    beta = torch.randint(-8, 9, (Cc,), generator=g).float() / 16
    beta[5] = -1000.0                                                      # an all-negative column
    one_hot = torch.randn(B, max(V, 1), generator=g)
    return dict(Y=y.reshape(-1, Cc), cnt=cnt, sums=sums, gamma=gamma, beta=beta, one_hot=one_hot, count=count)


def _kernel_scale(sums, gamma, count, Cc):
    """The kernel's fp32 scale for mean 0: float(1/sqrt(var + 1e-5f)) in double, times gamma in fp32."""
    inv = 1.0 / count
    var = sums[Cc:].double() * inv
    invstd = (1.0 / torch.sqrt(var + tr.EPS)).float()
    return gamma.float() * invstd


@pytest.mark.parametrize("B,T,K,Cc,V", [(2, 3, 7, 64, 0), (1, 5, 16, 128, 3), (3, 2, 5, 125, 10), (2, 4, 32, 96, 3)])
def test_pool_forward_and_backward(B, T, K, Cc, V):
    _l = _lib()
    h = _pool_case(B, T, K, Cc, V, seed=B * 100 + Cc + V)
    BT = B * T
    ld = Cc + V + 3
    dev = {k: v.to(DEV).contiguous() for k, v in h.items() if torch.is_tensor(v)}
    feat = torch.full((BT, ld), float("nan"), device=DEV)
    argmax = torch.full((BT, Cc), -7, dtype=torch.int32, device=DEV)
    dfeat = torch.randn(BT, ld, device=DEV)
    dA = torch.zeros(BT * K, Cc, device=DEV)
    P = _l.TrainPool()
    P.B, P.T, P.K, P.C, P.V, P.ld_feat = B, T, K, Cc, V, ld
    P.Y, P.cnt, P.sums = dev["Y"].data_ptr(), dev["cnt"].data_ptr(), dev["sums"].data_ptr()
    P.gamma, P.beta = dev["gamma"].data_ptr(), dev["beta"].data_ptr()
    P.one_hot = dev["one_hot"].data_ptr() if V else None
    P.feat, P.argmax, P.dfeat, P.dA = feat.data_ptr(), argmax.data_ptr(), dfeat.data_ptr(), dA.data_ptr()
    _l.call("fcn_train_pool", C.byref(P), 0, _stream())
    torch.cuda.synchronize()
    scale = _kernel_scale(h["sums"], h["gamma"], h["count"], Cc)
    # fmaf(y, scale, beta): y has <= 10 significant bits, so y*scale + beta is exact in float64
    z = (h["Y"].double().view(BT, K, Cc) * scale.double() + h["beta"].double()).float().clamp_min(0.0)
    z = z * (h["cnt"] > 0).float()[:, None, None]
    exp_feat = torch.full((BT, ld), float("nan"))
    exp_feat[:, :Cc] = z.amax(1)
    if V:
        exp_feat[:, Cc:Cc + V] = h["one_hot"][torch.arange(BT) // T, :V]
    _assert_bits(feat.cpu(), exp_feat, "pooled features, one-hot columns, untouched tail")
    exp_arg = z.argmax(1).int()                      # first index of the maximum
    assert torch.equal(argmax.cpu(), exp_arg), "argmax (first index on exact ties)"
    assert (z[:, :, 5] == 0).all() and (argmax.cpu()[:, 5] == 0).all()
    _l.call("fcn_train_pool", C.byref(P), 1, _stream())
    torch.cuda.synchronize()
    exp_dA = torch.zeros(BT, K, Cc)
    src = torch.where((h["cnt"] > 0)[:, None], dfeat.cpu()[:, :Cc], torch.zeros(()))
    exp_dA.scatter_(1, exp_arg.long()[:, None, :], src[:, None, :])
    _assert_bits(dA.cpu(), exp_dA.view(BT * K, Cc), "pool backward scatter (everything else stays 0)")


# ============================================================================ (e) finalize
def _ulp(x):
    x = x.float().abs()
    return torch.nextafter(x, torch.full_like(x, float("inf"))) - x


@pytest.mark.parametrize("update_running", [1, 0])
def test_finalize_mixed_table(update_running):
    S = tr.SrcDesc
    descs = [tr.concat_layer(2, 50, [S(50, 16)], [16], 40, has_bn=1, relu=1),
             tr.concat_layer(1, 1, [S(1, 16)], [16], 24, has_bn=1, relu=1),            # count 1: biased branch
             tr.deconv_layer(2, 10, [S(10, 16)], 16, 20, 4, has_bn=1, relu=1),
             tr.concat_layer(3, 7, [S(7, 16)], [16], 39, bias=True),
             tr.concat_layer(3, 7, [S(7, 16)], [16], 2)]                               # no BN, no bias
    g = torch.Generator().manual_seed(9)
    cases = [tr.LayerCase(d, DEV) for d in descs]
    before = []
    for c in cases:
        L = c.layer()
        n = c.dsums.numel()
        c.dsums.copy_(torch.randn(n, generator=g, dtype=torch.float64) * 100)
        if c.d.has_bn:
            cnt = tr.bn_count(L)
            mean = torch.randn(c.d.Cout, generator=g, dtype=torch.float64) * 3
            var = torch.rand(c.d.Cout, generator=g, dtype=torch.float64) * 4 + (0.0 if cnt > 1 else 1.0)
            c.sums.copy_(torch.cat([mean * cnt, (var + mean * mean) * cnt]))
            for t in (c.dgamma, c.dbeta, c.run_mean):
                t.copy_(torch.randn(t.shape, generator=g))
            c.run_var.copy_(torch.rand(c.d.Cout, generator=g) + 0.5)
        elif c.dbias is not None:
            c.dbias.copy_(torch.randn(c.dbias.shape, generator=g))
        before.append({k: getattr(c, k).clone() for k in ("dgamma", "dbeta", "dbias", "run_mean", "run_var")
                       if getattr(c, k) is not None})
    arr = (_lib().TrainLayer * len(cases))(*[c.layer() for c in cases])
    table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(DEV)
    _lib().call("fcn_train_finalize", table.data_ptr(), len(cases), update_running, _stream())
    torch.cuda.synchronize()
    for c, b in zip(cases, before):
        d = c.d
        if d.has_bn:
            _assert_bits(c.dbeta, b["dbeta"] + c.dsums[:d.Cout].float(), "dbeta +=")
            _assert_bits(c.dgamma, b["dgamma"] + c.dsums[d.Cout:].float(), "dgamma +=")
            if update_running:
                rm, rv = tr.finalize_running_ref(c.sums, tr.bn_count(c.layer()), b["run_mean"], b["run_var"], d.Cout)
                _assert_within(c.run_mean, rm, _ulp(rm).double(), "running mean (1 ulp)")
                _assert_within(c.run_var, rv, _ulp(rv).double(), "running var (1 ulp)")
            else:
                _assert_bits(c.run_mean, b["run_mean"], "running mean untouched")
                _assert_bits(c.run_var, b["run_var"], "running var untouched")
        elif c.dbias is not None:
            _assert_bits(c.dbias, b["dbias"] + c.dsums[:d.N].float(), "dbias +=")


# ============================================================================ (f) Adam
@pytest.mark.parametrize("n,step,wd,gscale,zero", [(1, 1, 0.0, 1.0, False), (255, 2, 1e-4, 0.125, False),
                                                   (257, 1000, 1e-4, 1.0, False), (10 ** 6, 10 ** 6, 0.0, 0.125, False),
                                                   (10 ** 6, 1, 1e-4, 0.125, False), (300, 1, 0.0, 1.0, True),
                                                   (300, 1000, 0.0, 1.0, True)])
def test_adam_step_matches_float64_restatement(n, step, wd, gscale, zero):
    g = torch.Generator().manual_seed(n % 1000 + step % 1000)
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    p = torch.randn(n, generator=g)
    grad = torch.zeros(n) if zero else torch.randn(n, generator=g) * torch.rand(n, generator=g) * 8
    if step == 1 or zero:
        m, v = torch.zeros(n), torch.zeros(n)
    else:
        m = torch.randn(n, generator=g) * 0.1
        v = m * m + torch.rand(n, generator=g) * 0.01
    dp, dg, dm, dv = (t.to(DEV).contiguous() for t in (p, grad, m, v))
    _lib().call("fcn_adam_step", dp.data_ptr(), dg.data_ptr(), dm.data_ptr(), dv.data_ptr(), n, lr, b1, b2, eps, wd,
                step, gscale, _stream())
    torch.cuda.synchronize()
    ep, em, ev, sc = tr.adam_ref(p, grad, m, v, lr, b1, b2, eps, wd, step, gscale)
    # bounds derived in the module docstring, section (f)
    G = grad.abs().double() * gscale + wd * p.abs().double()
    f1, f2 = tr.f32(b1), tr.f32(b2)
    bc_rel = 2.0 ** -21 * f1 ** step / (1 - f1 ** step) + 2.0 ** -22 * f2 ** step / (1 - f2 ** step)
    upd = (p.double() - ep).abs()
    tol = 4 * _ulp(ep).double() + 1e-6 * lr + 2.0 ** -18 * sc + bc_rel * upd
    _assert_within(dp.cpu(), ep, tol, "param")
    _assert_within(dm.cpu(), em, 4 * _ulp(em).double() + 2.0 ** -21 * (f1 * m.abs().double() + G), "exp_avg")
    _assert_within(dv.cpu(), ev, 8 * _ulp(ev).double() + 2.0 ** -20 * (1 - f2) * G ** 2, "exp_avg_sq")
    if zero:
        _assert_bits(dp, p.to(DEV), "zero gradient, no decay: parameters unchanged")


# ============================================================================ (c) real shapes: every TrainEngine layer
def _engine_mem(eng, model):
    mem = tr.Mem(eng.flat.param, eng.flat.grad, *eng.rows, *eng.cnt, *eng._keep, eng.in_onehot)
    for a in eng.act.values():
        for k in ("Y", "dA", "sums", "dsums"):
            if a.get(k) is not None:
                mem.add(a[k])
    for b in model.buffers():
        mem.add(b)
    return mem


@pytest.mark.parametrize("wl,B", [("refine_car", 4), ("refine_car", 32), ("car", 2), ("people", 1), ("sunrgbd", 2)])
def test_every_engine_layer_against_the_reference(wl, B):
    from frustum_convnet_b200 import synth
    from frustum_convnet_b200.train_engine import TrainStep
    model = tr.make_model(wl, seed=B + 3)
    data = {k: torch.from_numpy(v).cuda() for k, v in synth.make_frustums(wl, B, seed=60 + B, with_labels=True).items()}
    run0 = {n: b.clone() for n, b in model.named_buffers()}
    ts = TrainStep(model)
    ts.forward_backward(data)
    torch.cuda.synchronize()
    eng = next(iter(ts.engines.values()))
    mem = _engine_mem(eng, model)
    layers, names = eng.layers, eng.names
    grad_exp, grad_S, dA_targets = {}, {}, {}
    ambiguous = {}
    for li, L in enumerate(layers):
        nm = names[li]
        M = L.B * L.T_out
        Y, S = tr.forward_ref(L, mem)
        got = mem.get(L.Y, M * L.N).view(M, L.N)
        _assert_within(got, Y, tr.contraction_tol(_seg_K(L), S), "%s %s Y" % (wl, nm))
        if L.has_bn:
            exp, sc = tr.stats_ref(L, got)
            _assert_within(mem.get(L.sums, 2 * L.Cout), exp, tr.sum_tol(sc), "%s %s sums" % (wl, nm))
        dy = tr.dy_ref(L, mem)
        ambiguous[nm] = dy["namb"]
        ds, dss, amb = tr.reduce_ref(L, mem, dy)
        _assert_within(mem.get(L.dsums, ds.numel()), ds, tr.sum_tol(dss) + amb, "%s %s dsums" % (wl, nm))
        # dW of all segments -> the layer's slice of the flat bucket (zeroed at the start of the step)
        dWv, dWs, dWi = [], [], []
        for j in range(L.n_seg):
            widx, v, a, am = tr.dw_ref(L, j, mem, dy)
            dWi.append(widx.reshape(-1))
            dWv.append(v.reshape(-1))
            dWs.append((tr.contraction_tol(M, a) + am).reshape(-1))
        widx = torch.cat(dWi)
        nW = int(widx.max()) + 1
        ev, es = tr.scatter(nW, widx, torch.cat(dWv), torch.cat(dWs))
        gflat = eng.flat.grad
        off = (L.dW - gflat.data_ptr()) // 4
        _assert_within(gflat[off:off + nW], ev, es, "%s %s dW" % (wl, nm))
        # dX: summed over every consumer of each source
        for j in range(L.n_seg):
            s = L.seg[j].src
            if not ((eng.dx_mask[li] >> j) & 1) or not s.grad:
                continue
            idx, v, a, am = tr.dx_ref(L, j, mem, dy)
            n_src = L.B * s.T * s.ld
            key = s.grad
            tv, ts_ = tr.scatter(n_src, idx, v, tr.contraction_tol(L.N, a) + am)
            if key in grad_exp:
                grad_exp[key] += tv
                grad_S[key] += ts_
            else:
                grad_exp[key], grad_S[key] = tv, ts_
            dA_targets[key] = n_src
        if L.has_bn:
            dsums = mem.get(L.dsums, 2 * L.Cout)
            _assert_bits(mem.get(L.dbeta, L.Cout), dsums[:L.Cout].float(), "%s %s dbeta" % (wl, nm))
            _assert_bits(mem.get(L.dgamma, L.Cout), dsums[L.Cout:].float(), "%s %s dgamma" % (wl, nm))
        elif L.dbias:
            _assert_bits(mem.get(L.dbias, L.N), mem.get(L.dsums, L.N).float(), "%s %s dbias" % (wl, nm))
    # pooling: features, argmax, and the backward into the last PointNet layer's dA
    for s, P in enumerate(eng.pools):
        BT = P.B * P.T
        feat, err, Yp, z = tr.pool_ref(P, mem)
        gotf = mem.get(P.feat, BT * P.ld_feat).view(BT, P.ld_feat)
        _assert_within(gotf[:, :P.C], feat, err, "%s pool %d features" % (wl, s))
        am = mem.get(P.argmax, BT * P.C).view(BT, P.C).long()
        zsel = z.gather(1, am[:, None, :])[:, 0]
        assert (zsel >= feat - 2 * err).all(), "%s pool %d: argmax is not a maximum" % (wl, s)
        # identical rows before the argmax (back-fill duplicates) would have been picked first
        ysel = Yp.gather(1, am[:, None, :])
        k = torch.arange(P.K, device=am.device)[None, :, None]
        dup_before = ((Yp == ysel) & (k < am[:, None, :])).any(1)
        valid = (mem.get(P.cnt, BT) > 0)[:, None] & (feat > 0)
        assert not (dup_before & valid).any(), "%s pool %d: a bit-identical earlier row was not chosen" % (wl, s)
        key = P.dA
        exp_dA = tr.pool_bwd_ref(P, mem, am.int()).reshape(-1)
        grad_exp[key] = grad_exp.get(key, 0) + exp_dA
        grad_S[key] = grad_S.get(key, 0) + torch.zeros_like(exp_dA)
        dA_targets[key] = exp_dA.numel()
    for key, n in dA_targets.items():
        got = mem.get(key, n)
        _assert_within(got, grad_exp[key], grad_S[key], "%s dA of the tensor at 0x%x (sum over consumers)" % (wl, key))
    # running statistics: one update from the kernel's statistics
    for li, L in enumerate(layers):
        if not L.has_bn:
            continue
        rm_t = mem.get(L.run_mean, L.Cout)
        name = [n for n, b in model.named_buffers() if b.data_ptr() == L.run_mean][0]
        base = name[:-len("running_mean")]
        rm, rv = tr.finalize_running_ref(mem.get(L.sums, 2 * L.Cout), tr.bn_count(L), run0[base + "running_mean"],
                                         run0[base + "running_var"], L.Cout)
        _assert_within(rm_t, rm, _ulp(rm).double(), "%s %s running mean" % (wl, names[li]))
        _assert_within(mem.get(L.run_var, L.Cout), rv, _ulp(rv).double(), "%s %s running var" % (wl, names[li]))
    print("%s B=%d: %d layers checked; ReLU decisions within rounding of 0: %d" % (wl, B, len(layers),
                                                                                   sum(ambiguous.values())))
