"""Exact-arithmetic operands and float64 references for kernel-level bit-exact tests.

Inputs, weights and biases are small integers, chosen so that every product and every partial sum of a
contraction is an integer of magnitude < 2^22: fp32 accumulation is then exact in any order (and under the
tensor core's operand alignment), so a kernel result can be compared with ``torch.equal`` / bit equality.

Two regimes:
  R1 ("tf32-transparent"): every value that a kernel rounds to TF32 is an integer < 2^11, so the rounding is the
      identity and the fp32 SIMT path and all TF32 paths must give the same bits;
  R2 ("rounding"): layer outputs exceed 2^11, so the TF32 rounding (``engine.tf32_rna``) really rounds, ties
      included; the references apply it at the same points as the kernels.  TF32 paths only.

Every generator checks its own bound (sum |a|*|w| + |b| per output, over every input the case can contain).

References restate two C-ABI contracts of include/frustum_b200.h:
  ``pointnet_pooled_ref``  fcn_pointnet_tiles, pooled output;
  ``pointnet_unpooled_ref`` fcn_pointnet_tiles, un-pooled output of the fp32 path;
  ``conv_ref``             fcn_conv_gemm (segments, taps, strides, pitches, channel pad, pixel shuffle, crop,
                           output slice, relu, round_out).
``pointnet_args`` and ``ConvLaunch`` turn the same descriptions into kernel arguments (ctypes structs, tensor maps).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import torch

EXACT_LIMIT = 1 << 22          # every partial sum below this: fp32 accumulation is exact in any order
TF32_EXACT = 1 << 11           # integers below this are TF32 values: rounding to TF32 is the identity


def tf32(x: torch.Tensor) -> torch.Tensor:
    """engine.tf32_rna on float64 data holding fp32 values (round to nearest, ties away from zero)."""
    from frustum_convnet_b200.engine import tf32_rna
    f = x.float()
    assert torch.equal(f.double(), x.double()), "value is not an fp32 number"
    return tf32_rna(f).double()


def tf32_int_reference(x: float) -> float:
    """Round one finite fp32 value to TF32 with integer arithmetic only: keep 11 significant bits of the 24-bit
    significand, half away from zero.  An independent statement of the rounding the kernels use."""
    if x == 0.0 or not math.isfinite(x):
        return x
    m, e = math.frexp(abs(x))              # |x| = m * 2^e, m in [0.5, 1)
    M = int(m * (1 << 24))                 # exact: fp32 has a 24-bit significand
    assert M * 2.0 ** (e - 24) == abs(x)
    R = (M + (1 << 12)) >> 13 << 13        # drop 13 bits, halves round up in magnitude
    return math.copysign(R * 2.0 ** (e - 24), x)


def is_tie(x: torch.Tensor) -> torch.Tensor:
    """fp32 values whose 13 dropped bits are exactly 0x1000 (half-way between two TF32 values)."""
    return (x.float().view(torch.int32) & 0x1FFF) == 0x1000


def _ints(g: torch.Generator, lo: int, hi: int, shape) -> torch.Tensor:
    return torch.randint(lo, hi + 1, tuple(shape), generator=g).double()


def sparse_ints(g: torch.Generator, rows: int, cols: int, nnz: int, wmax: int) -> torch.Tensor:
    """(rows, cols) integer matrix with `nnz` non-zeros in every column, values in [-wmax, wmax] \\ {0}."""
    w = torch.zeros(rows, cols, dtype=torch.float64)
    mag = _ints(g, 1, wmax, (nnz, cols))
    sign = torch.where(torch.rand(nnz, cols, generator=g) < 0.5, -1.0, 1.0).double()
    for c in range(cols):
        idx = torch.randperm(rows, generator=g)[:nnz]
        w[idx, c] = mag[:, c] * sign[:, c]
    return w


def check_bound(amax: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], limit: int, what: str) -> float:
    """Assert sum_k amax_k*|w_kc| + |b_c| < limit for every output c (amax_k = largest |input k|).
    Returns the largest bound."""
    bound = amax.double().abs() @ w.double().abs()
    if b is not None:
        bound = bound + b.double().abs()
    worst = float(bound.max()) if bound.numel() else 0.0
    assert worst < limit, "%s: operand bound %.0f >= %d, the arithmetic is no longer exact" % (what, worst, limit)
    return worst


# ============================================================================ PointNet (fcn_pointnet_tiles)
@dataclass
class PointnetWeights:
    w1t: torch.Tensor   # (3, C1)
    b1: torch.Tensor
    w2t: torch.Tensor   # (C1, C2)
    b2: torch.Tensor
    w3t: torch.Tensor   # (C2, C3)
    b3: torch.Tensor
    coords: torch.Tensor  # the values a record coordinate may take (1-D)
    regime: str

    @property
    def dims(self):
        return self.w1t.shape[1], self.w2t.shape[1], self.w3t.shape[1]


# (coordinate values, |w1|, b1 range, nnz2, |w2|, |b2|, nnz3, |w3|)
_PN_REGIMES = {
    "R1": (list(range(-4, 5)), 3, (-6, 0), 8, 2, 12, 4, 1),
    "R2": ([-60, -53, -41, -37, -29, -17, -11, -3, 0, 5, 13, 23, 31, 43, 51, 61], 16, (-200, 0), 8, 3, 300, 8, 3),
}


def record_universe(coords) -> torch.Tensor:
    """Every (dx, dy, dz) record a case may contain, float64 (U, 3)."""
    c = torch.tensor(coords, dtype=torch.float64)
    return torch.cartesian_prod(c, c, c)


def pointnet_layers(xyz: torch.Tensor, W: PointnetWeights, round_tf32: bool):
    """Per-row chain in float64 -> (h1, h2, layer-3 pre-activation without bias)."""
    h1 = torch.relu(xyz @ W.w1t + W.b1)
    if round_tf32:
        h1 = tf32(h1)
    h2 = torch.relu(h1 @ W.w2t + W.b2)
    if round_tf32:
        h2 = tf32(h2)
    return h1, h2, h2 @ W.w3t


def make_pointnet_weights(C1: int, C2: int, C3: int, regime: str, seed: int) -> PointnetWeights:
    """Integer weights for one PointNet scale.  b1 <= 0, so the record (0,0,0) gives h1 = 0; b3 is chosen so
    that such rows have a layer-3 pre-activation <= 0 in every channel (the all-negative sections)."""
    coords, w1m, (b1lo, b1hi), nnz2, w2m, b2m, nnz3, w3m = _PN_REGIMES[regime]
    g = torch.Generator().manual_seed(seed)
    w1t = _ints(g, -w1m, w1m, (3, C1))
    b1 = _ints(g, b1lo, b1hi, (C1,))
    w2t = sparse_ints(g, C1, C2, nnz2, w2m)
    b2 = _ints(g, -b2m, b2m, (C2,))
    w3t = sparse_ints(g, C2, C3, nnz3, w3m)
    neg = torch.relu(b2) @ w3t                                # layer 3 of the (0,0,0) record
    b3 = torch.clamp(-neg, max=0.0) - _ints(g, 0, 3, (C3,))
    W = PointnetWeights(w1t, b1, w2t, b2, w3t, b3, torch.tensor(coords, dtype=torch.float64), regime)
    check_pointnet_bounds(W)
    return W


def check_pointnet_bounds(W: PointnetWeights):
    """Exactness over every record the coordinate set allows; R1 also keeps every rounded value < 2^11."""
    U = record_universe(W.coords.tolist())
    h1, h2, pre3 = pointnet_layers(U, W, round_tf32=True)
    lim = TF32_EXACT if W.regime == "R1" else EXACT_LIMIT
    check_bound(U.abs().amax(0), W.w1t, W.b1, lim, "layer 1")
    check_bound(h1.abs().amax(0), W.w2t, W.b2, lim, "layer 2")
    check_bound(h2.abs().amax(0), W.w3t, W.b3, lim, "layer 3")
    if W.regime == "R1":
        h1r, h2r, pre3r = pointnet_layers(U, W, round_tf32=False)
        assert torch.equal(h1r, h1) and torch.equal(h2r, h2) and torch.equal(pre3r, pre3)
    else:
        assert (h1.abs() >= TF32_EXACT).any() and (h2.abs() >= TF32_EXACT).any(), "R2 must round"


def pointnet_row_values(xyz: torch.Tensor, W: PointnetWeights, round_tf32: bool = True) -> torch.Tensor:
    """Value each row contributes to the pooled max: tf32(layer3 + b3) (TF32 paths) or layer3 + b3 (fp32)."""
    v = pointnet_layers(xyz, W, round_tf32)[2] + W.b3
    return tf32(v) if round_tf32 else v


@dataclass
class PointnetCase:
    """Inputs of one fcn_pointnet_tiles call (CPU tensors) + what the reference needs."""
    W: PointnetWeights
    rows: torch.Tensor          # (B, row_cap, 4) float32 records {dx, dy, dz, bits(section)}
    tiles: torch.Tensor         # (max_tiles, 4) int32 {b, row0, nrows, 0}; entries >= ntiles are decoys
    ntiles: int
    T: int
    feat_pitch: int
    ld_feat: int
    tile_rows: int
    feat_init: torch.Tensor     # (B, feat_pitch, ld_feat) float32
    sections: list = field(default_factory=list)   # per frustum: list of (length, kind)
    sect_rows: list = field(default_factory=list)  # per frustum: list of (T_index, xyz rows (n, 3))

    @property
    def B(self):
        return self.rows.shape[0]

    @property
    def row_cap(self):
        return self.rows.shape[1]


SENTINEL = -3.5     # negative: an integer atomicMax of any positive feature would replace it


def _draw_section(g, U_vals, n, kind, universe, ensure_argmax):
    if kind == "neg":
        return torch.zeros(n, 3, dtype=torch.float64)
    for _ in range(200):
        pick = torch.randint(0, universe.shape[0], (n,), generator=g)
        if not ensure_argmax or n > 16 or argmax_covers(U_vals[pick]):
            return universe[pick]
    raise AssertionError("could not draw a section of %d rows whose every row is a strict arg-max" % n)


def argmax_covers(vals: torch.Tensor) -> bool:
    """True when every row of the section (rows x channels values) is the unique, positive maximum of at least
    one channel: dropping or misplacing any row then changes the pooled feature."""
    n = vals.shape[0]
    if n == 1:
        return bool((vals > 0).any())
    top2 = vals.topk(2, dim=0).values
    uniq = (top2[0] > top2[1]) & (top2[0] > 0)
    winners = vals.argmax(0)[uniq]
    return len(set(winners.tolist())) == n


def make_pointnet_case(W: PointnetWeights, frustums: Sequence[Sequence], tile_rows: int, cuts: Sequence[int],
                       seed: int, pad_rows: int = 2, ld_extra: int = 8, n_decoys: int = 3,
                       shuffle_tiles: bool = True, round_tf32: bool = True,
                       ensure_argmax: bool = True) -> PointnetCase:
    """frustums[b] = list of (length, kind) sections (kind "pos" or "neg"; length 0 = empty section), laid end to
    end.  Each frustum's row stream is cut into tiles of the sizes in `cuts` (cycled, each <= tile_rows); every
    tile starts at a multiple of tile_rows, the slots past its nrows hold NaN records.  A decoy slot per frustum
    holds records that WOULD change the result; the decoy tiles sit in the table past `ntiles`.
    ensure_argmax: redraw every section of <= 16 rows until each row is the strict arg-max of some channel."""
    g = torch.Generator().manual_seed(seed)
    universe = record_universe(W.coords.tolist())
    U_vals = pointnet_row_values(universe, W, round_tf32)
    T = max(len(s) for s in frustums)
    B = len(frustums)
    streams, sect_rows = [], []
    for secs in frustums:
        recs, per = [], []
        for t, (n, kind) in enumerate(secs):
            if n == 0:
                continue
            xyz = _draw_section(g, U_vals, n, kind, universe, ensure_argmax)
            per.append((t, xyz))
            recs.append(torch.cat([xyz, torch.full((n, 1), float(t), dtype=torch.float64)], 1))
        streams.append(torch.cat(recs, 0) if recs else torch.zeros(0, 4, dtype=torch.float64))
        sect_rows.append(per)
    # cut into tiles
    tiles_b, slots = [], []
    ci = 0
    for b, st in enumerate(streams):
        pos, slot = 0, 0
        while pos < st.shape[0]:
            n = min(cuts[ci % len(cuts)], st.shape[0] - pos)
            ci += 1
            tiles_b.append((b, slot * tile_rows, n, pos))
            pos += n
            slot += 1
        slots.append(slot)
    row_cap = (max(slots) + 1) * tile_rows           # + the decoy slot
    assert row_cap >= T
    rows = torch.full((B, row_cap, 4), float("nan"), dtype=torch.float32)
    rows_i = rows.view(torch.int32)
    for b, row0, n, pos in tiles_b:
        chunk = streams[b][pos:pos + n]
        rows[b, row0:row0 + n, :3] = chunk[:, :3].float()
        rows_i[b, row0:row0 + n, 3] = chunk[:, 3].to(torch.int32)
    order = list(range(len(tiles_b)))
    if shuffle_tiles:
        order = torch.randperm(len(tiles_b), generator=g).tolist()
    table = [tiles_b[i][:3] for i in order]
    # decoys: records with the largest row value of the universe, filed under section 0
    big = universe[U_vals.amax(1).argmax()]
    for d in range(n_decoys):
        b = d % B
        row0 = (row_cap // tile_rows - 1) * tile_rows
        rows[b, row0:row0 + tile_rows, :3] = big.float()
        rows_i[b, row0:row0 + tile_rows, 3] = 0
        table.append((b, row0, tile_rows))
    tiles = torch.tensor([[b, r0, n, 0] for b, r0, n in table], dtype=torch.int32).view(-1, 4)
    C3 = W.dims[2]
    ld_feat = C3 + ld_extra
    pitch = T + pad_rows
    feat = torch.full((B, pitch, ld_feat), SENTINEL, dtype=torch.float32)
    feat[:, :T, :C3] = 0.0
    return PointnetCase(W, rows, tiles, len(tiles_b), T, pitch, ld_feat, tile_rows, feat,
                        [list(s) for s in frustums], sect_rows)


def pointnet_pooled_ref(case: PointnetCase, round_tf32: bool = True) -> torch.Tensor:
    """Expected feature map of fcn_pointnet_tiles (pooled): for the first `ntiles` tiles, every record row
    r < nrows with section t adds  tf32(layer3 + b3)  to the max of feat[b, t, :C3]; channels >= C3, pad rows
    and sections without rows keep what the map held; values <= 0 change nothing (the map starts at 0)."""
    C3 = case.W.dims[2]
    rows_i = case.rows.view(torch.int32)
    idx_b, idx_r = [], []
    for b, row0, n, _ in case.tiles[:case.ntiles].tolist():
        idx_b.append(torch.full((n,), b, dtype=torch.long))
        idx_r.append(torch.arange(row0, row0 + n))
    ib, ir = torch.cat(idx_b), torch.cat(idx_r)
    xyz = case.rows[ib, ir, :3].double()
    sect = rows_i[ib, ir, 3].long()
    assert (sect >= 0).all() and (sect < case.T).all()
    uniq, inv = torch.unique(xyz, dim=0, return_inverse=True)
    vals = pointnet_row_values(uniq, case.W, round_tf32)[inv]
    key = ib * case.feat_pitch + sect
    pooled = torch.full((case.B * case.feat_pitch, C3), float("-inf"), dtype=torch.float64)
    pooled.scatter_reduce_(0, key[:, None].expand(-1, C3), vals, "amax", include_self=True)
    out = case.feat_init.clone().view(-1, case.ld_feat)
    cur = out[:, :C3].double()
    out[:, :C3] = torch.where(pooled > cur, pooled, cur).float()
    return out.view_as(case.feat_init)


def pointnet_unpooled_ref(case: PointnetCase, K: int, out_init: torch.Tensor) -> torch.Tensor:
    """Expected output of fcn_pointnet_tiles, un-pooled (fp32 path): out (B, C3, T*K) channel-first.  Every record
    row r < nrows of the first `ntiles` tiles, at flat position p = row0 + r of frustum b, writes
    relu(layer3 + b3) to out[b, :, p], or 0 when its tag has the sign bit set (a masked section, whose coordinates
    are never evaluated); positions no tile covers keep out_init."""
    C3 = case.W.dims[2]
    rows_i = case.rows.view(torch.int32)
    out = out_init.clone().view(case.B, C3, case.T * K)
    for b, row0, n, _ in case.tiles[:case.ntiles].tolist():
        p = torch.arange(row0, row0 + n)
        tag = rows_i[b, p, 3]
        live = tag >= 0
        assert (tag[live] < case.T).all() and (p < case.T * K).all()
        vals = torch.zeros(n, C3, dtype=torch.float64)
        if live.any():
            vals[live] = torch.relu(pointnet_row_values(case.rows[b, p[live], :3].double(), case.W, round_tf32=False))
        out[b][:, p] = vals.t().float()
    return out.view_as(out_init)


def pointnet_pooled_loop_ref(case: PointnetCase, round_tf32: bool = True) -> torch.Tensor:
    """The same contract written as a plain per-section loop (amax over the section's rows), for cross-checks."""
    C3 = case.W.dims[2]
    out = case.feat_init.clone()
    for b, per in enumerate(case.sect_rows):
        for t, xyz in per:
            v = pointnet_row_values(xyz, case.W, round_tf32).amax(0)
            out[b, t, :C3] = torch.maximum(out[b, t, :C3].double(), v).float()
    return out


# ============================================================================ conv GEMM (fcn_conv_gemm)
@dataclass
class ConvSeg:
    src: torch.Tensor    # (B, pitch, ld) position-major; rows [T_src, pitch) zero
    C: int
    T_src: int
    tap: int
    stride: int


@dataclass
class ConvSpec:
    B: int
    T_out: int
    P_m: int
    segs: List[ConvSeg]
    wt: torch.Tensor      # (K_pad, n_cols) float64, segment s at rows [k0_s, k0_s + C_s)
    bias: torch.Tensor    # (n_cols,)
    Cout: int
    up: int
    relu: int
    round_out: int
    out: torch.Tensor     # (B, P_store, ld_out) initial output buffer (sentinel-filled)
    T_store: int
    c_off: int

    @property
    def K_pad(self):
        return self.wt.shape[0]

    @property
    def n_cols(self):
        return self.wt.shape[1]

    def k_offsets(self):
        offs, k = [], 0
        for s in self.segs:
            offs.append(k)
            k += (s.C + 31) // 32 * 32
        return offs


def conv_gather(spec: ConvSpec, s: int) -> torch.Tensor:
    """(B, T_out, C) float64 A-operand block of segment s: src[b, t*stride + tap, :C], zero outside [0, T_src)."""
    sg = spec.segs[s]
    t = torch.arange(spec.T_out, device=sg.src.device)
    ts = t * sg.stride + sg.tap
    ok = (ts >= 0) & (ts < sg.T_src)
    a = sg.src[:, ts.clamp(0, sg.src.shape[1] - 1), :sg.C].double()
    return a * ok[None, :, None]


def conv_ref(spec: ConvSpec, with_abs: bool = False):
    """Expected `out` of fcn_conv_gemm: out[b, t*up + j, c_off + co] = act(sum_seg A_seg @ W_seg + bias)[j*Cout + co]
    for t < T_out, t*up + j < T_store; everything else keeps its initial value.  act = ReLU (relu) then TF32
    rounding (round_out).  Weights are used as given (a TF32 path consumes tf32(wt); integer weights are TF32).
    with_abs: also return the pre-activation and sum |a|*|w| + |b| per stored output (float64, (B, n_t, Cout)).
    Runs on the device of the sources."""
    N = spec.up * spec.Cout
    Y = torch.zeros(spec.B, spec.T_out, N, dtype=torch.float64, device=spec.segs[0].src.device)
    S = torch.zeros_like(Y)
    for s, k0 in enumerate(spec.k_offsets()):
        a = conv_gather(spec, s)
        w = spec.wt[k0:k0 + spec.segs[s].C, :N].double().to(a.device)
        Y += a @ w
        if with_abs:
            S += a.abs() @ w.abs()
    Y += spec.bias[:N].double().to(Y.device)
    S += spec.bias[:N].double().abs().to(Y.device)
    pre = Y
    if spec.relu:
        Y = torch.relu(Y)
    if spec.round_out:
        Y = tf32(Y)
    out = spec.out.clone()
    Y = Y.to(out.device)
    n_t = min(spec.T_store, spec.T_out * spec.up)
    shuf = Y.reshape(spec.B, spec.T_out * spec.up, spec.Cout)[:, :n_t]
    out[:, :n_t, spec.c_off:spec.c_off + spec.Cout] = shuf.float()
    if not with_abs:
        return out
    return out, pre.reshape(spec.B, spec.T_out * spec.up, spec.Cout)[:, :n_t], \
        S.reshape(spec.B, spec.T_out * spec.up, spec.Cout)[:, :n_t]


def conv_operand_bound(spec: ConvSpec, limit: int):
    """Assert sum |a|*|w| + |b| < limit for every output of the spec (exactness of the accumulation)."""
    _, _, S = conv_ref(spec, with_abs=True)
    worst = float(S.max()) if S.numel() else 0.0
    assert worst < limit, "conv operand bound %.0f >= %d" % (worst, limit)
    return worst


# ============================================================================ ctypes builders
def _ptr(t):
    return t.data_ptr() if t is not None else None


def pointnet_args(case: PointnetCase, dev_bufs: dict, precision: int, K: int = 1):
    """PointnetArgs for `case` with its tensors on the device (dev_bufs: rows, tiles, ntiles, out, w1t, b1, w2t, b2,
    w3t, b3, w2_tc, w3_tc)."""
    from frustum_convnet_b200 import _lib
    C1, C2, C3 = case.W.dims
    a = _lib.PointnetArgs()
    a.C1, a.C2, a.C3, a.T, a.K = C1, C2, C3, case.T, K
    a.ld_feat, a.row_cap, a.tile_rows = case.ld_feat, case.row_cap, case.tile_rows
    a.unpooled, a.precision, a.B = 0, precision, case.B
    a.rows, a.tiles, a.ntiles = _ptr(dev_bufs["rows"]), _ptr(dev_bufs["tiles"]), _ptr(dev_bufs["ntiles"])
    a.max_tiles = case.tiles.shape[0]
    for n in ("w1t", "b1", "w2t", "b2", "w3t", "b3", "w2_tc", "w3_tc"):
        setattr(a, n, _ptr(dev_bufs.get(n)))
    a.out = _ptr(dev_bufs["out"])
    a.feat_pitch = case.feat_pitch
    return a


def pointnet_device_weights(W: PointnetWeights, device) -> dict:
    from frustum_convnet_b200.engine import pack_sw128
    C1, C2, C3 = W.dims
    d = {n: getattr(W, n).float().contiguous().to(device) for n in ("w1t", "b1", "w2t", "b2", "w3t", "b3")}
    d["w2_tc"] = pack_sw128(W.w2t.t().float().contiguous(), min(C2, 128)).to(device)
    d["w3_tc"] = pack_sw128(W.w3t.t().float().contiguous(), 128).to(device)
    return d


class ConvLaunch:
    """fcn_conv_gemm arguments for a ConvSpec at one precision; keeps the device tensors and tensor maps alive."""

    def __init__(self, spec: ConvSpec, precision: int, device):
        from frustum_convnet_b200 import _lib
        from frustum_convnet_b200.engine import pack_sw128
        self.srcs = [s.src.float().contiguous().to(device) for s in spec.segs]
        self.wt = spec.wt.float().contiguous().to(device)
        self.bias = spec.bias.float().contiguous().to(device)
        self.out = spec.out.float().contiguous().to(device)
        a = _lib.ConvArgs()
        a.B, a.T_out, a.n_seg = spec.B, spec.T_out, len(spec.segs)
        for j, (s, t) in enumerate(zip(spec.segs, self.srcs)):
            a.seg[j].src, a.seg[j].ld, a.seg[j].C = _ptr(t), t.shape[2], s.C
            a.seg[j].T_src, a.seg[j].tap, a.seg[j].stride, a.seg[j].pitch = s.T_src, s.tap, s.stride, t.shape[1]
        a.K_pad, a.n_cols, a.Cout, a.up = spec.K_pad, spec.n_cols, spec.Cout, spec.up
        a.relu, a.precision, a.round_out = spec.relu, precision, spec.round_out
        a.wt, a.bias = _ptr(self.wt), _ptr(self.bias)
        self.w_tc = None
        if precision >= 1:
            nt = 128 if precision in (1, 3) else 64
            self.w_tc = pack_sw128(spec.wt.t().float().contiguous(), nt).to(device)
            a.w_tc = _ptr(self.w_tc)
        self.maps = None
        if precision in (3, 4):
            self.maps = (C.c_ubyte * (128 * len(self.srcs)))()
            for j, (s, t) in enumerate(zip(spec.segs, self.srcs)):
                _lib.call("fcn_encode_activation_map", C.addressof(self.maps) + 128 * j, _ptr(t),
                          1, t.shape[0] * t.shape[1], t.shape[2], s.stride)   # flattened padded rows
            a.tmaps = C.addressof(self.maps)
        a.out, a.ld_out, a.T_store, a.c_off = _ptr(self.out), self.out.shape[2], spec.T_store, spec.c_off
        a.P_m, a.P_store = spec.P_m, self.out.shape[1]
        self.args = a

    def run(self):
        from frustum_convnet_b200 import _lib
        _lib.call("fcn_conv_gemm", C.byref(self.args), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return self.out.cpu()


def bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Bit equality of two fp32 tensors (NaN sentinels compare equal to themselves)."""
    return a.shape == b.shape and torch.equal(a.float().contiguous().view(torch.int32),
                                              b.float().contiguous().view(torch.int32))


def describe_mismatch(got: torch.Tensor, exp: torch.Tensor, limit: int = 8) -> str:
    gi, ei = got.float().contiguous().view(torch.int32), exp.float().contiguous().view(torch.int32)
    bad = (gi != ei).nonzero()
    lines = ["%d of %d elements differ" % (bad.shape[0], got.numel())]
    for idx in bad[:limit].tolist():
        lines.append("  %s: got %r expected %r" % (tuple(idx), float(got[tuple(idx)]), float(exp[tuple(idx)])))
    return "\n".join(lines)
