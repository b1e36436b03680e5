"""Float64 statement of the training-layer contract of include/frustum_b200.h (section 7, csrc/train.cu).

A layer is described once (``LayerDesc``: segments, sources, parameter layout); ``LayerCase`` allocates its
buffers and produces the ctypes records (``_lib.TrainLayer``).  The reference functions read the buffers a
kernel call read, through the pointers of the ctypes record (``Mem`` resolves a pointer to the tensor that holds
it), so the same code checks a synthetic case and every layer of a ``TrainEngine`` from the engine's own buffers.

Each stage is checked against ITS OWN inputs: BN scale / shift of a source come from that source's ``sums`` as
the kernel left them, the BN backward of a layer from the layer's ``sums`` and ``dsums`` as the kernel left them.

Every contraction reference returns the value and an absolute-value companion built from the operands:
    |a| = |x|*|scale| + |beta| + |mean*scale|   for a BN source (|x| without statistics), 0 where ReLU is off,
    |b| = |scale| * (|dz| + |m1| + (|y| + |mean|) * invstd * |m2|)   (|dA| for a layer without BN),
the magnitudes of the terms the kernel rounds when it forms the operand.  Bounds (``contraction_tol`` etc.) are
stated on these companions.  Elements whose ReLU decision is within rounding of 0 ("ambiguous") cannot be
resolved by a float64 reference; their full contribution is returned separately so a test can either assert there
are none (generated data keeps a margin) or add it to the bound (real model data).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import List, Optional

import torch

from exact_ref import EXACT_LIMIT

EPS = float(torch.tensor(1e-5, dtype=torch.float32))    # the kernels' BN epsilon is the fp32 constant 1e-5f
U = 2.0 ** -24                                         # unit round-off of fp32
AMBIG = 16 * U                                         # |pre| below this * (|y*scale| + |shift|): ReLU undecidable
F64 = torch.float64


# ============================================================================ pointer -> tensor
class Mem:
    """Resolves raw pointers of a ctypes record to the tensors that hold them."""

    def __init__(self, *tensors):
        self._t = []
        for t in tensors:
            self.add(t)

    def add(self, t):
        if t is not None:
            self._t.append(t)
        return t

    def get(self, ptr: int, n: int) -> torch.Tensor:
        """1-D view of the n elements starting at `ptr` (dtype of the tensor that holds it)."""
        assert ptr, "NULL pointer"
        for t in self._t:
            base, es = t.data_ptr(), t.element_size()
            if base <= ptr < base + t.numel() * es:
                off = ptr - base
                assert off % es == 0 and off // es + n <= t.numel(), "pointer range leaves its tensor"
                return t.reshape(-1)[off // es: off // es + n]
        raise KeyError("pointer 0x%x is not in any registered tensor" % ptr)


# ============================================================================ description -> buffers -> ctypes
@dataclass
class SrcDesc:
    T: int                      # positions per frustum before the pixel shuffle
    ld: int
    up: int = 1
    cup: int = 0
    c0: int = 0
    stats: bool = False         # a BN layer's raw output: scale/shift (+ ReLU) applied on load
    Cstat: int = 1
    coff: int = 0
    relu: int = 1
    grad: bool = True           # has a gradient buffer


@dataclass
class SegDesc:
    src: int                    # index into LayerDesc.srcs
    C: int
    tap: int = 0
    stride: int = 1
    s_ci: int = 1
    w_off: int = 0


@dataclass
class LayerDesc:
    B: int
    T_out: int
    N: int
    Cout: int
    segs: List[SegDesc]
    srcs: List[SrcDesc]
    s_co: int
    s_j: int = 0
    up: int = 1
    has_bn: int = 0
    relu: int = 0
    bias: bool = False

    @property
    def M(self):
        return self.B * self.T_out

    def w_numel(self):
        return max(int(weight_index_d(self, g).max()) for g in self.segs) + 1


def weight_index_d(d, g) -> torch.Tensor:
    """(C, N) flat indices of the weight elements of segment g: w_off + c*s_ci + (n%Cout)*s_co + (n/Cout)*s_j."""
    n = torch.arange(d.N)
    c = torch.arange(g.C)
    return g.w_off + c[:, None] * g.s_ci + (n % d.Cout)[None] * d.s_co + (n // d.Cout)[None] * d.s_j


# --- parameter layouts of the model's layers
def conv1d_layer(B, T_in, srcs, Ci, Co, k=1, stride=1, **kw) -> LayerDesc:
    """Conv1d(Ci, Co, k, stride, padding=k//2) over source 0, weight (Co, Ci, k); k=1 is also Conv2d (Co,Ci,1,1)."""
    pad = k // 2
    T_out = (T_in + 2 * pad - k) // stride + 1
    segs = [SegDesc(0, Ci, j - pad, stride, k, j) for j in range(k)]
    return LayerDesc(B, T_out, Co, Co, segs, srcs, s_co=Ci * k, **kw)


def concat_layer(B, T_out, srcs, Cs, Co, **kw) -> LayerDesc:
    """1x1 conv over the channel concat of the sources (weight (Co, sum Cs, 1)): one segment per source."""
    segs, off = [], 0
    for i, c in enumerate(Cs):
        segs.append(SegDesc(i, c, 0, 1, 1, off))
        off += c
    return LayerDesc(B, T_out, Co, Co, segs, srcs, s_co=off, **kw)


def deconv_layer(B, T_in, srcs, Ci, Co, k, **kw) -> LayerDesc:
    """ConvTranspose1d(Ci, Co, k, stride=k), weight (Ci, Co, k): N = k*Co columns, column n = tap n/Co."""
    return LayerDesc(B, T_in, k * Co, Co, [SegDesc(0, Ci, 0, 1, Co * k, 0)], srcs, s_co=k, s_j=1, up=k, **kw)


def _ptr(t):
    return t.data_ptr() if t is not None else None


class LayerCase:
    """Buffers of one layer call (one device, fp32 / fp64 / int like the kernels) and its ctypes record.
    Source i: raw (B*T, ld), grad (B*T, ld) or None, sums (2*Cstat) fp64, gamma / beta (Cstat)."""

    def __init__(self, d: LayerDesc, device, dtype=torch.float32):
        self.d, self.dev = d, device
        f, f64 = dict(dtype=dtype, device=device), dict(dtype=F64, device=device)
        self.mem = Mem()
        self.src = []
        for s in d.srcs:
            b = dict(raw=torch.zeros(d.B * s.T, s.ld, **f))
            b["grad"] = torch.zeros(d.B * s.T, s.ld, **f) if s.grad else None
            if s.stats:
                b.update(sums=torch.zeros(2 * s.Cstat, **f64), gamma=torch.ones(s.Cstat, **f),
                         beta=torch.zeros(s.Cstat, **f))
            for t in b.values():
                self.mem.add(t)
            self.src.append(b)
        nw = d.w_numel()
        Cs = d.Cout if d.has_bn else d.N
        self.W = torch.zeros(nw, **f)
        self.dW = torch.zeros(nw, **f)
        self.bias = torch.zeros(d.N, **f) if d.bias else None
        self.dbias = torch.zeros(d.N, **f) if d.bias else None
        self.Y = torch.zeros(d.M, d.N, **f)
        self.dA = torch.zeros(d.M, d.N, **f)
        self.sums = torch.zeros(2 * d.Cout, **f64) if d.has_bn else None
        self.dsums = torch.zeros(2 * Cs, **f64)
        bn = [torch.zeros(d.Cout, **f) for _ in range(6)] if d.has_bn else [None] * 6
        self.gamma, self.beta, self.dgamma, self.dbeta, self.run_mean, self.run_var = bn
        if d.has_bn:
            self.gamma.fill_(1.0)
            self.run_var.fill_(1.0)
        for t in (self.W, self.dW, self.bias, self.dbias, self.Y, self.dA, self.sums, self.dsums, *bn):
            self.mem.add(t)

    def layer(self) -> "C.Structure":
        from frustum_convnet_b200 import _lib
        d = self.d
        L = _lib.TrainLayer()
        L.B, L.T_out, L.n_seg, L.N, L.Cout, L.up = d.B, d.T_out, len(d.segs), d.N, d.Cout, d.up
        L.s_co, L.s_j, L.has_bn, L.relu = d.s_co, d.s_j, d.has_bn, d.relu
        for i, g in enumerate(d.segs):
            s, b = d.srcs[g.src], self.src[g.src]
            S = L.seg[i].src
            S.raw, S.grad = _ptr(b["raw"]), _ptr(b["grad"])
            if s.stats:
                S.sums, S.gamma, S.beta = _ptr(b["sums"]), _ptr(b["gamma"]), _ptr(b["beta"])
                S.count, S.Cstat, S.coff, S.relu = float(self.src_count(g.src)), s.Cstat, s.coff, s.relu
            else:
                S.count, S.Cstat, S.coff, S.relu = 1.0, 1, 0, 0
            S.ld, S.T, S.up, S.cup, S.c0 = s.ld, s.T, s.up, s.cup, s.c0
            G = L.seg[i]
            G.C, G.tap, G.stride, G.s_ci, G.w_off = g.C, g.tap, g.stride, g.s_ci, g.w_off
        L.W, L.dW, L.bias, L.dbias = _ptr(self.W), _ptr(self.dW), _ptr(self.bias), _ptr(self.dbias)
        L.Y, L.dA, L.sums, L.dsums = _ptr(self.Y), _ptr(self.dA), _ptr(self.sums), _ptr(self.dsums)
        L.gamma, L.beta, L.dgamma, L.dbeta = _ptr(self.gamma), _ptr(self.beta), _ptr(self.dgamma), _ptr(self.dbeta)
        L.run_mean, L.run_var = _ptr(self.run_mean), _ptr(self.run_var)
        return L

    def src_count(self, i):
        s = self.d.srcs[i]
        return self.d.B * s.T * s.up

    def written_mask(self, i, dx_mask) -> torch.Tensor:
        """(B*T, ld) bool: elements of source i's gradient that the segments in dx_mask address."""
        d, s = self.d, self.d.srcs[i]
        m = torch.zeros(d.B * s.T * s.ld, dtype=torch.bool, device=self.dev)
        for j, g in enumerate(d.segs):
            if g.src == i and (dx_mask >> j) & 1:
                idx, valid = src_index(d.B, d.T_out, g.tap, g.stride, g.C, s.T, s.up, s.ld, s.cup, s.c0, self.dev)
                m[idx[valid].reshape(-1)] = True
        return m.view(d.B * s.T, s.ld)


# ============================================================================ reference maths
def src_index(B, T_out, tap, stride, C, T, up, ld, cup, c0, device):
    """(M, C) flat indices into a source (raw[(b*T + p/up)*ld + c0 + (p%up)*cup + c], p = t*stride + tap) and the
    (M,) mask of rows whose position lies in [0, T*up)."""
    r = torch.arange(B * T_out, device=device)
    b, t = r // T_out, r % T_out
    p = t * stride + tap
    valid = (p >= 0) & (p < T * up)
    pc = p.clamp(0, T * up - 1)
    base = (b * T + pc // up) * ld + c0 + (pc % up) * cup
    return base[:, None] + torch.arange(C, device=device)[None], valid


def bn_coef(sums, gamma, beta, count, ch):
    """float64 mean, invstd, scale, shift of channels `ch` from Sum(y), Sum(y^2) (biased variance)."""
    Cs = gamma.numel()
    s = sums.double()
    mean = s[ch] / count
    var = (s[Cs + ch] / count - mean * mean).clamp_min(0.0)
    invstd = 1.0 / torch.sqrt(var + EPS)
    scale = gamma.double()[ch] * invstd
    return mean, invstd, scale, beta.double()[ch] - mean * scale


def operand(L, j, mem):
    """Segment j's A operand: (act (M, C), |a| (M, C), flat source index (M, C), valid rows (M,))."""
    g = L.seg[j]
    s = g.src
    raw = mem.get(s.raw, L.B * s.T * s.ld)
    idx, valid = src_index(L.B, L.T_out, g.tap, g.stride, g.C, s.T, s.up, s.ld, s.cup, s.c0, raw.device)
    x = raw.double()[idx]
    if s.sums:
        ch = (s.coff + torch.arange(g.C, device=raw.device)) % s.Cstat
        mean, _, scale, shift = bn_coef(mem.get(s.sums, 2 * s.Cstat), mem.get(s.gamma, s.Cstat),
                                        mem.get(s.beta, s.Cstat), s.count, ch)
        pre = x * scale + shift
        a_abs = x.abs() * scale.abs() + mem.get(s.beta, s.Cstat).double()[ch].abs() + (mean * scale).abs()
        if s.relu:
            x = pre.clamp_min(0.0)
            a_abs = a_abs * (pre > -AMBIG * a_abs)     # near-zero pre-activations: the kernel may keep a rounding
        else:
            x = pre
    else:
        a_abs = x.abs()
    v = valid[:, None].double()
    return x * v, a_abs * v, idx, valid


def weights(L, j, mem):
    """Segment j's weights (C, N) and their flat indices in the parameter layout."""
    g = L.seg[j]
    n = torch.arange(L.N)
    c = torch.arange(g.C)
    widx = g.w_off + c[:, None] * g.s_ci + (n % L.Cout)[None] * L.s_co + (n // L.Cout)[None] * L.s_j
    W = mem.get(L.W, int(widx.max()) + 1)
    widx = widx.to(W.device)
    return W.double()[widx], widx


def forward_ref(L, mem):
    """Y (M, N) = sum over segments act(X) @ W (+ bias) and its |a|@|w| (+|bias|) companion."""
    Y = S = None
    for j in range(L.n_seg):
        a, aa, _, _ = operand(L, j, mem)
        w, _ = weights(L, j, mem)
        Y = a @ w if Y is None else Y + a @ w
        S = aa @ w.abs() if S is None else S + aa @ w.abs()
    if L.bias:
        b = mem.get(L.bias, L.N).double()
        Y, S = Y + b, S + b.abs()
    return Y, S


def fold(L, t: torch.Tensor) -> torch.Tensor:
    """(M, N) -> per channel n % Cout: sum over rows and the `up` column groups."""
    return t.reshape(-1, L.N // L.Cout, L.Cout).sum((0, 1))


def stats_ref(L, Y):
    """Sum(y), Sum(y^2) per BN channel from the kernel's own Y and Sum|y|, Sum y^2 (their error scales)."""
    Y = Y.double()
    s1, s2 = fold(L, Y), fold(L, Y * Y)
    return torch.cat([s1, s2]), torch.cat([fold(L, Y.abs()), s2])


def bn_count(L):
    return float(L.B * L.T_out * L.up)


def dy_ref(L, mem):
    """dY (M, N) with the BN / ReLU backward applied; |b| companion; ambiguous part |scale*dA| where the ReLU
    decision is within rounding; plus dz and xh (and |xh|) for the reduction."""
    M, N = L.B * L.T_out, L.N
    dA = mem.get(L.dA, M * N).double().view(M, N)
    if not L.has_bn:
        z = torch.zeros_like(dA)
        return dict(dY=dA, abs=dA.abs(), amb=z, dz=dA, xh=None, xh_abs=None, namb=0)
    Y = mem.get(L.Y, M * N).double().view(M, N)
    co = torch.arange(N, device=dA.device) % L.Cout
    cnt = bn_count(L)
    mean, invstd, scale, shift = bn_coef(mem.get(L.sums, 2 * L.Cout), mem.get(L.gamma, L.Cout),
                                         mem.get(L.beta, L.Cout), cnt, co)
    ds = mem.get(L.dsums, 2 * L.Cout).double()
    m1, m2 = ds[co] / cnt, ds[L.Cout + co] / cnt
    pre = Y * scale + shift
    amb = torch.zeros_like(dA, dtype=torch.bool)
    dz = dA
    if L.relu:
        amb = pre.abs() <= AMBIG * ((Y * scale).abs() + shift.abs())
        dz = dA * (pre > 0)
    xh = (Y - mean) * invstd
    xh_abs = (Y.abs() + mean.abs()) * invstd
    dY = scale * (dz - m1 - xh * m2)
    b_abs = scale.abs() * (dz.abs() + m1.abs() + xh_abs * m2.abs())
    return dict(dY=dY, abs=b_abs, amb=(scale.abs() * dA.abs()) * amb, dz=dz, xh=xh, xh_abs=xh_abs,
                namb=int(amb.sum()), amb_mask=amb, dA=dA)


def reduce_ref(L, mem, dy=None):
    """Expected dsums: BN layer [Sum dz, Sum dz*xh] per channel; plain layer [Sum dA] per column.
    Returns (value, |terms| companion, ambiguous part)."""
    dy = dy or dy_ref(L, mem)
    if not L.has_bn:
        return dy["dY"].sum(0), dy["abs"].sum(0), torch.zeros(L.N, dtype=F64, device=dy["dY"].device)
    dz, xh = dy["dz"], dy["xh"]
    v = torch.cat([fold(L, dz), fold(L, dz * xh)])
    a = torch.cat([fold(L, dz.abs()), fold(L, dz.abs() * dy["xh_abs"])])
    am = dy["amb_mask"] * dy["dA"].abs()
    amb = torch.cat([fold(L, am), fold(L, am * dy["xh_abs"])])
    return v, a, amb


def dw_ref(L, j, mem, dy=None):
    """Segment j's dW contribution: (flat weight indices (C, N), value, |a|^T|b| companion, ambiguous part)."""
    dy = dy or dy_ref(L, mem)
    a, aa, _, _ = operand(L, j, mem)
    _, widx = weights(L, j, mem)
    return widx, a.t() @ dy["dY"], aa.t() @ dy["abs"], aa.t() @ dy["amb"]


def dx_ref(L, j, mem, dy=None):
    """Segment j's dX contribution scattered into the source layout: (flat source indices of the valid rows
    (R, C), value, |b||w| companion, ambiguous part), all (R, C)."""
    dy = dy or dy_ref(L, mem)
    w, _ = weights(L, j, mem)
    _, _, idx, valid = operand(L, j, mem)
    return idx[valid], (dy["dY"] @ w.t())[valid], (dy["abs"] @ w.abs().t())[valid], (dy["amb"] @ w.abs().t())[valid]


def scatter(n, idx, *vals):
    """Dense float64 vectors of length n holding sum over (idx -> val) for each of `vals`."""
    out = []
    for v in vals:
        o = torch.zeros(n, dtype=F64, device=v.device)
        o.index_add_(0, idx.reshape(-1), v.reshape(-1))
        out.append(o)
    return out


# --- bounds
def contraction_tol(K, S):
    """|delta| <= (K + 8) * 2^-23 * sum_k |a_k||b_k| for an fp32 FMA contraction of length K (+8: the fp32
    evaluation of the BN / ReLU operands and the final additions)."""
    return (K + 8) * 2.0 ** -23 * S


def sum_tol(S):
    """Statistics / reductions: every fp32 partial chain has at most 128 terms before the fp64 atomics."""
    return 2.0 ** -17 * S


# --- pooling (fcn_train_pool)
def pool_ref(P, mem):
    """-> (feat (B*T, C) float64 max_k relu(bn(y)) * (cnt > 0), per-element error scale (B*T, C), Y (B*T, K, C)
    float64, post-activation values (B*T, K, C))."""
    BT = P.B * P.T
    Y = mem.get(P.Y, BT * P.K * P.C).double().view(BT, P.K, P.C)
    cnt = mem.get(P.cnt, BT)
    ch = torch.arange(P.C, device=Y.device)
    mean, _, scale, shift = bn_coef(mem.get(P.sums, 2 * P.C), mem.get(P.gamma, P.C), mem.get(P.beta, P.C),
                                    float(P.B * P.T * P.K), ch)
    z = (Y * scale + shift).clamp_min(0.0) * (cnt > 0).double()[:, None, None]
    err = 8 * U * (Y.abs() * scale.abs() + mem.get(P.beta, P.C).double().abs() + (mean * scale).abs())
    return z.amax(1), err.amax(1), Y, z


def pool_bwd_ref(P, mem, argmax):
    """dA (B*T*K, C) that the backward scatter must produce in a zero-filled buffer."""
    BT = P.B * P.T
    dfeat = mem.get(P.dfeat, BT * P.ld_feat).double().view(BT, P.ld_feat)[:, :P.C]
    cnt = mem.get(P.cnt, BT)
    dA = torch.zeros(BT, P.K, P.C, dtype=F64, device=dfeat.device)
    dA.scatter_(1, argmax.long()[:, None, :], torch.where((cnt > 0)[:, None], dfeat, 0.0)[:, None, :])
    return dA.view(BT * P.K, P.C)


# --- finalize
def finalize_running_ref(sums, count, run_mean, run_var, C):
    """float64 running statistics after one update (momentum 0.1, unbiased variance; biased when count == 1)."""
    s = sums.double()
    mean = s[:C] / count
    var = (s[C:2 * C] / count - mean * mean).clamp_min(0.0)
    unb = var * count / (count - 1.0) if count > 1.0 else var
    return 0.9 * run_mean.double() + 0.1 * mean, 0.9 * run_var.double() + 0.1 * unb


# --- Adam (fcn_adam_step)
def f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def adam_ref(p, g, m, v, lr, b1, b2, eps, wd, step, gscale):
    """torch.optim.Adam (L2 weight decay added to the gradient) in float64 with the hyper-parameters rounded to
    fp32 as the kernel receives them; the gradient is multiplied by grad_scale first.
    -> (p, m, v, |update| scale of the cancellation-prone terms)."""
    lr, b1, b2, eps, wd, gscale = map(f32, (lr, b1, b2, eps, wd, gscale))
    p, g, m, v = (t.double() for t in (p, g, m, v))
    gi = g * gscale + wd * p
    m1 = b1 * m + (1 - b1) * gi
    v1 = b2 * v + (1 - b2) * gi * gi
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    denom = torch.sqrt(v1) / math.sqrt(bc2) + eps
    upd = lr / bc1 * m1 / denom
    scale = lr / bc1 * (b1 * m.abs() + (1 - b1) * (g.abs() * gscale + wd * p.abs())) / denom
    return p - upd, m1, v1, scale


# ============================================================================ models
def make_model(workload: str, seed: int):
    """PointNetDet of `workload` (KITTI or SUN-RGBD architecture) with the seeded synthetic state dict, on the
    device, in train() mode."""
    import numpy as np
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload(workload)
    if w["arch"].num_scales == 5:
        from frustum_convnet_b200.det_base_sunrgbd import PointNetDet
    else:
        from frustum_convnet_b200.det_base import PointNetDet
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=seed)
    m = PointNetDet(3, num_vec=w["num_vec"])
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    return m.cuda().train()


# ============================================================================ operand generators
def exact_fill(case: LayerCase, seed: int, amax=3, wmax=2, dmax=3, gmax=5):
    """Exact regime: small-integer sources (no statistics), weights, bias, dA, and pre-filled gradients.
    Every buffer element the kernels must not touch starts as NaN (weights' unaddressed slots, dW outside the
    layout, source gradients outside the region the layer's segments address)."""
    d = case.d
    g = torch.Generator().manual_seed(seed)

    def ints(lo, hi, shape):
        return torch.randint(lo, hi + 1, tuple(shape), generator=g).float().to(case.dev)

    for b in case.src:
        b["raw"].copy_(ints(-amax, amax, b["raw"].shape))
    nan = float("nan")
    case.W.fill_(nan)
    case.dW.fill_(nan)
    for sg in d.segs:
        widx = weight_index_d(d, sg).reshape(-1).to(case.dev)
        case.W[widx] = ints(-wmax, wmax, widx.shape)
        case.dW[widx] = ints(-gmax, gmax, widx.shape)
    if case.bias is not None:
        case.bias.copy_(ints(-4, 4, case.bias.shape))
        case.dbias.copy_(ints(-gmax, gmax, case.bias.shape))
    case.dA.copy_(ints(-dmax, dmax, case.dA.shape))
    case.Y.fill_(nan)
    # exactness: every forward partial sum below 2^22 (dW and dX sums are far smaller at these shapes)
    L = case.layer()
    _, S = forward_ref(L, case.mem)
    assert float(S.max()) < EXACT_LIMIT
    return L


def prefill_grads(case: LayerCase, dx_mask: int, seed: int, ints: bool = True):
    """Source gradients: NaN, then non-zero values where the segments in dx_mask write (accumulation check)."""
    g = torch.Generator().manual_seed(seed)
    for i, b in enumerate(case.src):
        if b["grad"] is None:
            continue
        w = case.written_mask(i, dx_mask)
        b["grad"].fill_(float("nan"))
        n = int(w.sum())
        if ints:
            sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
            v = torch.randint(1, 6, (n,), generator=g).float() * sign
        else:
            v = torch.randn(n, generator=g)
        b["grad"][w] = v.to(case.dev)


def bn_source_fill(case: LayerCase, i: int, seed: int, tau: float = 1e-4, wide_channel: Optional[int] = None):
    """BN regime source i: statistics of random per-channel mean / std, raw values drawn from them, gamma in
    +-[0.5, 1.5], beta in [-0.5, 0.5].  Every pre-activation keeps |pre| >= tau * (|x*scale| + |shift|)
    (resampled otherwise) so the ReLU mask is unambiguous.  `wide_channel`: that statistics channel gets
    mean/std = 100."""
    d, s, b = case.d, case.d.srcs[i], case.src[i]
    g = torch.Generator().manual_seed(seed)
    Cs = s.Cstat
    mean = torch.randn(Cs, generator=g, dtype=F64) * 0.5
    std = torch.rand(Cs, generator=g, dtype=F64) + 0.5
    if wide_channel is not None:
        mean[wide_channel] = 100.0 * std[wide_channel]
    cnt = case.src_count(i)
    b["sums"].copy_(torch.cat([mean * cnt, (std * std + mean * mean) * cnt]))
    sign = torch.where(torch.rand(Cs, generator=g) < 0.2, -1.0, 1.0)
    b["gamma"].copy_((torch.rand(Cs, generator=g) + 0.5) * sign)
    b["beta"].copy_(torch.rand(Cs, generator=g) - 0.5)
    # raw values are drawn per reading segment, from the statistics of the channel that segment applies
    raw = torch.randn(b["raw"].shape, generator=g, dtype=F64).to(case.dev)
    out = raw.clone()
    for sg in d.segs:
        if sg.src != i:
            continue
        idx, valid = src_index(d.B, d.T_out, sg.tap, sg.stride, sg.C, s.T, s.up, s.ld, s.cup, s.c0, case.dev)
        ch = ((s.coff + torch.arange(sg.C)) % Cs).to(case.dev)
        mu, sd = mean.to(case.dev)[ch], std.to(case.dev)[ch]
        out.view(-1)[idx[valid]] = (mu + sd * raw.view(-1)[idx[valid]])
    b["raw"].copy_(out.float())
    for _ in range(20):
        bad_any = False
        for sg in d.segs:
            if sg.src != i:
                continue
            idx, valid = src_index(d.B, d.T_out, sg.tap, sg.stride, sg.C, s.T, s.up, s.ld, s.cup, s.c0, case.dev)
            xr = b["raw"].view(-1)[idx].double()
            ch = ((s.coff + torch.arange(sg.C)) % Cs).to(case.dev)
            _, _, scale, shift = bn_coef(b["sums"], b["gamma"], b["beta"], float(cnt), ch)
            pre = xr * scale + shift
            bad = (pre.abs() < tau * ((xr * scale).abs() + shift.abs())) & valid[:, None]
            if bad.any():
                bad_any = True
                fix = idx[bad]
                b["raw"].view(-1)[fix] = b["raw"].view(-1)[fix] + (0.01 * sd_of(std, ch, bad)).float().to(case.dev)
        if not bad_any:
            return
    raise AssertionError("could not keep the pre-activations away from 0")


def sd_of(std, ch, bad):
    return std.to(ch.device)[ch].expand_as(bad)[bad]


def keep_relu_margin(L, mem, tau: float = 1e-4, seed: int = 0):
    """For the BN backward of layer L: resample (from the same column) the Y values whose pre-activation under
    the layer's own statistics lies within tau * (|y*scale| + |shift|) of 0.  Y is an INPUT of the backward."""
    if not (L.has_bn and L.relu):
        return 0
    M, N = L.B * L.T_out, L.N
    Y = mem.get(L.Y, M * N).view(M, N)
    co = torch.arange(N, device=Y.device) % L.Cout
    _, _, scale, shift = bn_coef(mem.get(L.sums, 2 * L.Cout), mem.get(L.gamma, L.Cout), mem.get(L.beta, L.Cout),
                                 bn_count(L), co)
    y = Y.double()
    bad = (y * scale + shift).abs() < tau * ((y * scale).abs() + shift.abs())
    nb = int(bad.sum())
    if nb:
        g = torch.Generator(device="cpu").manual_seed(seed)
        good = ~bad
        for n in bad.any(0).nonzero().view(-1).tolist():
            rows = bad[:, n].nonzero().view(-1)
            pool = good[:, n].nonzero().view(-1)
            pick = pool[torch.randint(0, pool.numel(), (rows.numel(),), generator=g).to(pool.device)]
            Y[rows, n] = Y[pick, n]
    return nb
