"""Host-side engine of the H100 frustum hot path (eval / inference).

Owns (as torch tensors — the library itself allocates nothing, SURVEY.md section 8(b) "Ownership"):
  * the BN-folded, kernel-ready weight pack built from a reference-format state dict
    (BN folding happens here at eval()/load time, never inside the state dict);
  * per-shape workspaces (row records, tile tables, position-major activations, outputs);
  * an optional CUDA graph of the whole forward (no host sync exists on the path: the
    `indices.max()/min()` assert of /root/reference/models/det_base.py:70 is dropped because the
    kernels emit in-range indices by construction).

The sequence of C-ABI calls mirrors PointNetDet.forward (det_base.py:334-412):
  fcn_group_rows            QueryDepthPoint + gather + centre subtraction, all scales  (:68-80)
  fcn_pointnet_tiles  x S   conv1..3 + BN + ReLU + mask + max over K                  (:95-101,134-143)
  fcn_conv_gemm       x 14  ConvFeatNet + heads (cat == extra K segments)             (:196-224,367-368)
  fcn_decode_eval           softmax / argmax / box decode                             (:376-411)
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from . import mega as _mega
from .config import DATASET_INFO, ArchSpec, fcn_layers
from .synth import reg_out_size

BN_EPS = 1e-5


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def tf32_rna(x: torch.Tensor) -> torch.Tensor:
    """Round fp32 to TF32 (10-bit mantissa), nearest with ties away from zero == cvt.rna.tf32.f32."""
    i = x.contiguous().view(torch.int32)
    mag = ((i & 0x7FFFFFFF) + 0x1000) & ~0x1FFF
    return ((i & -0x80000000) | mag).view(torch.float32)


def pack_sw128(w: torch.Tensor, n_chunk: int) -> torch.Tensor:
    """(Cout, Cin) fp32 -> tensor-core stage images: for each n-chunk and each 32-wide K block a
    [n_chunk rows][128 B] tile in the K-major 128-byte-swizzle layout (16-byte chunk c of row n
    stored at chunk position c ^ (n & 7)), stages concatenated in consumption order (nc, kb)."""
    co, ci = w.shape
    assert co % n_chunk == 0 and ci % 32 == 0 and n_chunk % 8 == 0
    x = tf32_rna(w.float()).view(co // n_chunk, n_chunk, ci // 32, 8, 4).permute(0, 2, 1, 3, 4)
    n = torch.arange(n_chunk, device=w.device)
    src = torch.arange(8, device=w.device)[None, :] ^ (n[:, None] & 7)          # [n][pos] -> source chunk
    return x[:, :, n[:, None], src, :].contiguous().view(-1)


def _fold_bn(sd, prefix) -> Tuple[torch.Tensor, torch.Tensor]:
    """(scale, shift) in float64 of an eval-mode BatchNorm (models/common.py:38-63 factories)."""
    g = sd[prefix + ".weight"].double()
    b = sd[prefix + ".bias"].double()
    m = sd[prefix + ".running_mean"].double()
    v = sd[prefix + ".running_var"].double()
    s = g / torch.sqrt(v + BN_EPS)
    return s, b - m * s


def _out_map(L) -> str:
    """Activation map an FCN layer writes: its own, the concat (transposed convs) or the logits (heads)."""
    return {"deconv": "cat", "heads": "logits"}.get(L.kind, L.name)


class _ConvLayer:
    """One fcn_conv_gemm call: packed weights + symbolic segment/output description.
    `wt` / `bias` arrive as HOST tensors (BN folded in float64 on the CPU: one upload per operand instead of
    ~900 tiny device launches per pack); the device copies are made here."""

    def __init__(self, name, kind, segs, K_pad, n_cols, Cout, up, relu, wt, bias, out, c_off, device):
        self.name, self.kind, self.segs, self.K_pad, self.n_cols = name, kind, segs, K_pad, n_cols
        self.Cout, self.up, self.relu = Cout, up, relu
        self.out, self.c_off, self.device = out, c_off, device
        if K_pad % 64:   # tensor-core stages are 64 K elements wide: one extra all-zero K block
            wt = torch.cat([wt, torch.zeros(32, wt.shape[1], dtype=wt.dtype)], 0).contiguous()
            self.K_pad = K_pad + 32
        self._wt_host = wt
        self.wt = wt.to(device)
        self.bias = bias.to(device)
        self._tc = {}

    def tc_image(self, n_tile: int) -> torch.Tensor:
        """Pre-swizzled tensor-core stage images [n_tile][kb][n_tile rows x 128 B] (lazy, cached)."""
        if n_tile not in self._tc:
            self._tc[n_tile] = pack_sw128(self._wt_host.t().contiguous(), n_tile).to(self.device)
        return self._tc[n_tile]


class FrustumEngine:
    """Kernel-ready form of one PointNetDet (KITTI 4-scale or SUN-RGBD 5-scale)."""

    def __init__(self, arch: ArchSpec, num_vec: int, dataset: str, dists: Sequence[float],
                 num_bins: int, state_dict: Dict[str, torch.Tensor], device, precision: int = 0):
        self.arch, self.num_vec, self.dataset = arch, int(num_vec), dataset
        self.dists = [float(d) for d in dists]
        assert len(self.dists) == arch.num_scales
        self.num_bins = int(num_bins)
        self.num_size = DATASET_INFO[dataset].NUM_SIZE_CLUSTER
        self.device = torch.device(device)
        self.precision = int(precision)
        self.use_tma = os.environ.get("FCN_CONV_TMA", "1") != "0"   # conv A operand via TMA tensor maps
        # FCN_PN_CLUSTER=1: PointNet on 2-CTA clusters (precision 2: every weight stage is read from L2 once per
        # cluster and multicast to both CTAs) for the scales whose layer-1 width is >= FCN_PN_CLUSTER_MIN.  Off by
        # default: with overlapped wgmmas, on an H100 SXM (700 W limit, B=32, 200-step regions, two runs each) it
        # measured 2-3 % below the 1-CTA kernel on every workload (resident frustums/s: car 109.8-111.6 k vs
        # 113.5-114.7 k, people 66.9-67.7 k vs 69.1-69.3 k, SUN-RGBD 72.3-72.6 k vs 74.7-75.1 k).
        self.pn_cluster = os.environ.get("FCN_PN_CLUSTER", "0") == "1"
        self.pn_cluster_min = int(os.environ.get("FCN_PN_CLUSTER_MIN", "128"))
        self.group_scan = os.environ.get("FCN_GROUP_SCAN") is not None   # A/B: section-scan grouping kernels
        # persistent FCN kernel (all conv layers + heads + decode in one launch, csrc/fcn_mega.cu); FCN_MEGA=0
        # falls back to one fcn_conv_gemm launch per layer + fcn_decode_eval (kept as the A/B and module-API path)
        self.use_mega = (self.precision == 1 and self.use_tma and os.environ.get("FCN_MEGA", "1") != "0")
        # persistent CTAs per forward.  A CTA that waits for a producer tile holds its SM idle: FEW CTAs per forward
        # and several forwards in flight favour throughput; FCN_MEGA_GRID=<SM count> favours the latency of a single
        # forward instead.  0 = adaptive: 2/3 of the smallest per-layer tile count of the main chain, within [4, 48]
        # (B=32: car 24, people 30, SUN-RGBD 6)
        self.mega_grid = int(os.environ.get("FCN_MEGA_GRID", "0"))
        # 256-wide N tiles for the layers with >= 256 output columns: less shared-memory traffic per MAC (the A box
        # feeds twice as many MMA columns) but half as many jobs per layer.  "auto" uses them when every main-chain
        # layer still has >= 24 tiles (people, car at B >= 64); True / False force.
        v = os.environ.get("FCN_MEGA_NT256", "auto")
        self.mega_nt256 = "auto" if v == "auto" else (v == "1")
        self.tile_rows = 64 if self.precision == 0 else 128
        self.out_size = reg_out_size(dataset, self.num_bins)
        self.ld_logit = _round_up(2 + self.out_size, 64)
        self.c3 = [m[2] for m in arch.mlps]
        self.ld_feat = [_round_up(c + self.num_vec, 4) for c in self.c3]
        self.mean_size = torch.tensor(DATASET_INFO[dataset].MEAN_SIZE_ARRAY, dtype=torch.float32,
                                      device=self.device)
        self._plans: Dict[tuple, "_Plan"] = {}
        self.max_plans = int(os.environ.get("FCN_MAX_PLANS", "64"))   # (shape, stream) workspaces kept alive
        # optional `f(numel, device) -> fp32 tensor` supplying the result block of new plans (lets a caller
        # place the blocks of several in-flight plans in one buffer, e.g. for one all-gather over all of them)
        self.out_alloc = None
        self.pack(state_dict)

    # ------------------------------------------------------------------ weight packing
    def pack(self, state_dict: Dict[str, torch.Tensor]):
        # BN folding and operand packing run on the HOST in float64 (a few ms for 3.3 M parameters); only the
        # finished operands are uploaded.  (Folding on the device cost ~900 tiny torch launches per pack.)
        sd = {k: v.detach().cpu() for k, v in state_dict.items()}
        dev, f32 = self.device, torch.float32
        cpu = torch.device("cpu")
        self.pn = []
        self.layers: List[_ConvLayer] = []
        self._plans.clear()
        self.has_feat = "feat_net.pointnet1.conv1.0.weight" in sd
        self.has_fcn = "conv_net.block1_conv1.0.weight" in sd
        self.has_heads = "cls_out.weight" in sd
        for i, (c1, c2, c3) in enumerate(self.arch.mlps if self.has_feat else ()):
            p = "feat_net.pointnet%d" % (i + 1)
            lay = {}
            for j in (1, 2, 3):
                w = sd["%s.conv%d.0.weight" % (p, j)].double()[:, :, 0, 0]      # (Co,Ci)
                s, sh = _fold_bn(sd, "%s.conv%d.1" % (p, j))
                wf = (w * s[:, None]).to(f32)                                   # (Co,Ci) folded
                lay["w%dt" % j] = wf.t().contiguous().to(dev)                   # (Ci,Co)
                lay["b%d" % j] = sh.to(f32).contiguous().to(dev)
                if self.precision == 1 and j >= 2:
                    lay["w%d_tc" % j] = pack_sw128(wf, min(c2, 128) if j == 2 else 128).to(dev)
            self.pn.append(lay)
        if not self.has_fcn:
            return
        for L in fcn_layers(self.arch, self.num_vec):
            if L.kind == "heads" and not self.has_heads:
                return
            ci = sum(c for _, c in L.srcs)
            if L.kind == "heads":          # one K segment over the concat; columns [cls0, cls1, reg...]
                segs, n_cols, co, up = [("cat", ci, 0, 1)], self.ld_logit, self.ld_logit, 1
            elif L.kind == "deconv":       # taps laid out along N: column j * Cout + c is output position t * k + j
                segs, n_cols, co, up = [(L.srcs[0][0], ci, 0, 1)], _round_up(L.k * L.Cout, 64), L.Cout, L.k
            else:                          # conv taps (tap-major) and merge sources laid out along K
                segs = [(src, c, j - L.k // 2, L.stride) for j in range(L.k) for src, c in L.srcs]
                n_cols, co, up = _round_up(L.Cout, 64), L.Cout, 1
            k_off = np.cumsum([0] + [_round_up(c, 32) for _, c, _, _ in segs]).tolist()
            wt = torch.zeros(k_off[-1], n_cols, dtype=torch.float64, device=cpu)
            bias = torch.zeros(n_cols, dtype=torch.float64, device=cpu)
            if L.kind == "heads":          # det_base.py:250-251,367-368
                osz = self.out_size
                wt[:ci, 0:2] = sd["cls_out.weight"][:, :, 0].double().t()
                wt[:ci, 2:2 + osz] = sd["reg_out.weight"][:, :, 0].double().t()
                bias[0:2], bias[2:2 + osz] = sd["cls_out.bias"].double(), sd["reg_out.bias"].double()
            else:
                w = sd["conv_net.%s.0.weight" % L.name].double()     # conv / merge (Co,Ci,k), deconv (Ci,Co,k)
                s, sh = _fold_bn(sd, "conv_net.%s.1" % L.name)
                if L.kind == "deconv":
                    for j in range(L.k):
                        wt[:ci, j * co:(j + 1) * co] = w[:, :, j] * s[None, :]
                        bias[j * co:(j + 1) * co] = sh
                else:
                    n = 0
                    for j in range(L.k):
                        c0 = 0
                        for _, c in L.srcs:
                            wt[k_off[n]: k_off[n] + c, :co] = (w[:, c0:c0 + c, j] * s[:, None]).t()
                            c0, n = c0 + c, n + 1
                    bias[:co] = sh
            self.layers.append(_ConvLayer(L.name, L.kind, segs, k_off[-1], n_cols, co, up, int(L.kind != "heads"),
                                          wt.to(f32).contiguous(), bias.to(f32).contiguous(), _out_map(L), L.c_off,
                                          dev))

    # ------------------------------------------------------------------ shape plans
    def plan(self, B: int, N: int, T: Sequence[int]) -> "_Plan":
        """Workspace for one input shape ON THE CURRENT STREAM: forwards issued from different streams
        (``with torch.cuda.stream(s): model(x)``) get disjoint workspaces/graphs and may overlap."""
        shape = (int(B), int(N), tuple(int(t) for t in T))
        key = shape + (torch.cuda.current_stream(self.device).cuda_stream,)
        p = self._plans.pop(key, None)
        if p is None:
            if len(self._plans) >= self.max_plans:       # LRU eviction (dict order = recency of use)
                self._plans.pop(next(iter(self._plans)))
            p = _Plan(self, *shape)
        self._plans[key] = p
        return p

    # ------------------------------------------------------------------ public calls
    @torch.no_grad()
    def forward(self, pc: torch.Tensor, centers: Sequence[torch.Tensor], one_hot, use_graph=False,
                copy_out=True, trusted=False):
        """Eval forward -> the 6-tuple of det_base.py:411.  trusted: the caller validated these tensors before."""
        p = self.plan(pc.shape[0], pc.shape[2], [c.shape[2] for c in centers])
        return p.run(pc, centers, one_hot, use_graph=use_graph, copy_out=copy_out, trusted=trusted)

    @torch.no_grad()
    def pointnet_feat(self, pc, centers, one_hot):
        """API #3: PointNetFeat.forward -> tuple of channel-first (B, C3+V, T_i)."""
        p = self.plan(pc.shape[0], pc.shape[2], [c.shape[2] for c in centers])
        return p.run_feat(pc, centers, one_hot)

    @torch.no_grad()
    def conv_feat_net(self, feats_bct: Sequence[torch.Tensor]):
        """ConvFeatNet.forward on channel-first inputs -> (B, arch.reg_in, T2)."""
        B = feats_bct[0].shape[0]
        p = self.plan(B, 1, [f.shape[2] for f in feats_bct])
        return p.run_fcn_bct(feats_bct)

    @torch.no_grad()
    def pointnet_module(self, scale: int, pc, new_pc):
        """API #2: PointNetModule.forward -> masked, un-pooled (B, C3, T, K)."""
        return _run_module(self, scale, pc, new_pc)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _Plan:
    """Workspace + prebuilt C argument structs for one (B, N, T...) shape."""

    def __init__(self, eng: FrustumEngine, B: int, N: int, T: Tuple[int, ...]):
        self.eng, self.B, self.N, self.T = eng, B, N, T
        arch, dev = eng.arch, eng.device
        S = arch.num_scales
        assert len(T) == S, "expected %d section lists, got %d" % (S, len(T))
        for i in range(1, S):  # FCN length bookkeeping (k3 s2 p1): T_i == ceil(T_{i-1}/2)
            assert T[i] == (T[i - 1] + 1) // 2, \
                "section counts %s are not a /2 pyramid (ConvFeatNet cat would fail)" % (T,)
        f32 = torch.float32
        K = arch.nsample
        tr = eng.tile_rows
        # Row pitch of every position-major map: P_S = T_S + 1, P_i = 2 * P_{i+1}.  Each frustum is followed
        # by >= 1 zero pad row (never written), so the FCN GEMMs can run over the FLATTENED rows of the
        # whole batch (full 128-row tiles): k=3 taps read a zero row instead of the neighbouring frustum,
        # and stride-2 layers map flat row r to input rows 2r-1..2r+1 because the pitch halves per level.
        P = [0] * S
        P[S - 1] = T[S - 1] + 1
        for i in range(S - 2, -1, -1):
            P[i] = 2 * P[i + 1]
            assert P[i] >= T[i] + 1
        self.P = P
        self.buf: Dict[str, torch.Tensor] = {}
        self.rows, self.cnt, self.tiles, self.max_tiles, self.idx32 = [], [], [], [], []
        for s in range(S):
            cap = T[s] * K[s]
            self.rows.append(torch.empty((B, cap, 4), dtype=f32, device=dev))
            self.cnt.append(torch.empty((B, T[s]), dtype=torch.int32, device=dev))
            self.idx32.append(torch.empty((B, T[s], K[s]), dtype=torch.int32, device=dev))
            mt = B * ((cap + tr - 1) // tr)
            self.max_tiles.append(mt)
            self.tiles.append(torch.empty((max(mt, 1), 4), dtype=torch.int32, device=dev))
            self.buf["feat%d" % (s + 1)] = torch.zeros((B, P[s], eng.ld_feat[s]), dtype=f32, device=dev)
        self.ntiles = torch.zeros(_lib.MAX_SCALES, dtype=torch.int32, device=dev)
        self.valid_T = {"feat%d" % (s + 1): T[s] for s in range(S)}
        # one map per conv / merge layer; the transposed convs share the concat, the heads write the logits
        for L in fcn_layers(arch, eng.num_vec):
            name = _out_map(L)
            if name not in self.buf:
                C = {"cat": arch.reg_in, "logits": eng.ld_logit}.get(name, L.Cout)
                self.buf[name] = torch.zeros((B, P[L.level], C), dtype=f32, device=dev)
                self.valid_T[name] = T[L.level]
        T2 = T[1]
        # the six outputs of det_base.py:411 are views into one flat block (single all-gather / D2H)
        widths_out = (2, 3, 1, 3, eng.num_bins, eng.num_size)
        n_out = B * T2 * sum(widths_out)
        self.out_flat = (eng.out_alloc(n_out, dev) if eng.out_alloc is not None
                         else torch.empty(n_out, dtype=f32, device=dev))
        outs, off = [], 0
        for wd in widths_out:
            n = B * T2 * wd
            v = self.out_flat[off: off + n]
            outs.append(v.view(B, T2) if wd == 1 and len(outs) == 2 else v.view(B, T2, wd))
            off += n
        self.out = tuple(outs)
        # static inputs (graph replay reads these): views of ONE flat block [pc | centers... | one_hot],
        # so a packed batch is staged with a single copy and a caller may also fill them in place
        sizes = [B * 3 * max(N, 1)] + [B * 3 * T[s] for s in range(S)] + [B * max(eng.num_vec, 1)]
        offs = np.concatenate([[0], np.cumsum([(n + 63) // 64 * 64 for n in sizes])]).astype(int)
        self.in_flat = torch.zeros(int(offs[-1]), dtype=f32, device=dev)
        self._in_offs = [int(o) for o in offs[:-1]]
        self.in_pc = self.in_flat[offs[0]: offs[0] + sizes[0]].view(B, 3, max(N, 1))
        self.in_centers = [self.in_flat[offs[1 + s]: offs[1 + s] + sizes[1 + s]].view(B, 3, T[s]) for s in range(S)]
        self.in_onehot = self.in_flat[offs[1 + S]: offs[1 + S] + sizes[1 + S]].view(B, max(eng.num_vec, 1))
        self.graph = None
        self._sides = []
        self._build_args()

    def _tsize(self, name):
        return self.buf[name].shape[1]

    def _build_args(self):
        eng, S = self.eng, self.eng.arch.num_scales
        g = _lib.GroupArgs()
        g.num_scales, g.B, g.N, g.num_vec = S, self.B, self.N, eng.num_vec
        g.tile_rows, g.unique_rows = eng.tile_rows, 1
        for s in range(S):
            g.T[s], g.K[s], g.dis_z[s] = self.T[s], eng.arch.nsample[s], eng.dists[s]
            g.c3[s], g.ld_feat[s] = eng.c3[s], eng.ld_feat[s]
            g.row_cap[s] = self.T[s] * eng.arch.nsample[s]
            g.tile_cap[s] = max(self.max_tiles[s], 1)
            g.rows[s], g.cnt[s] = _ptr(self.rows[s]), _ptr(self.cnt[s])
            g.feat[s], g.tiles[s] = _ptr(self.buf["feat%d" % (s + 1)]), _ptr(self.tiles[s])
            g.idx_scratch[s] = _ptr(self.idx32[s])
            g.feat_pitch[s] = self.P[s]
        g.ntiles = _ptr(self.ntiles)
        g.force_scan = 1 if eng.group_scan else 0
        self.group_args = g
        self.pn_args = []
        for s in range(S if eng.has_feat else 0):
            c1, c2, c3 = eng.arch.mlps[s]
            a = _lib.PointnetArgs()
            a.C1, a.C2, a.C3, a.T, a.K = c1, c2, c3, self.T[s], eng.arch.nsample[s]
            a.ld_feat, a.row_cap, a.tile_rows = eng.ld_feat[s], self.T[s] * eng.arch.nsample[s], eng.tile_rows
            a.unpooled, a.precision, a.B = 0, eng.precision, self.B
            a.rows, a.tiles = _ptr(self.rows[s]), _ptr(self.tiles[s])
            a.ntiles = self.ntiles.data_ptr() + 4 * s
            a.max_tiles = self.max_tiles[s]
            w = eng.pn[s]
            a.w1t, a.b1, a.w2t, a.b2, a.w3t, a.b3 = (_ptr(w["w1t"]), _ptr(w["b1"]), _ptr(w["w2t"]),
                                                    _ptr(w["b2"]), _ptr(w["w3t"]), _ptr(w["b3"]))
            a.w2_tc, a.w3_tc = _ptr(w.get("w2_tc")), _ptr(w.get("w3_tc"))
            if eng.precision == 1 and eng.pn_cluster and c1 >= eng.pn_cluster_min:
                a.precision = 2
            a.out = _ptr(self.buf["feat%d" % (s + 1)])
            a.feat_pitch = self.P[s]
            self.pn_args.append(a)
        # GEMM geometry of every layer: (output positions T_out, row pitch P_m of the M space, N tile width)
        self.geom = []
        for L in eng.layers:
            src, _, _, stride = L.segs[0]
            T_in = self.valid_T[src]
            self.geom.append((T_in if stride == 1 else (T_in + 1) // 2, self.buf[src].shape[1] // stride,
                              128 if L.n_cols % 128 == 0 else 64))
        self.conv_args = []
        self._tmaps = []
        for L, (T_out, P_m, nt) in zip(eng.layers, self.geom):
            a = _lib.ConvArgs()
            out = self.buf[L.out]
            a.B, a.T_out, a.P_m = self.B, T_out, P_m
            a.n_seg = len(L.segs)
            for j, (src, c, tap, st) in enumerate(L.segs):
                t = self.buf[src]
                a.seg[j].src, a.seg[j].ld, a.seg[j].C = _ptr(t), t.shape[2], c
                a.seg[j].T_src, a.seg[j].tap, a.seg[j].stride = self.valid_T[src], tap, st
                a.seg[j].pitch = t.shape[1]
            a.K_pad, a.n_cols, a.Cout, a.up, a.relu = L.K_pad, L.n_cols, L.Cout, L.up, L.relu
            a.precision, a.w_tc = 0, None
            if eng.precision == 1 and L.Cout % 32 == 0:
                # The A operand feed is the limit, so the wider N tile (2x the MMA work per A byte) is used
                # whenever the layer has >= 128 columns.
                a.w_tc = _ptr(L.tc_image(nt))
                if eng.use_tma:
                    # fully TMA-fed variant: one 128-byte tensor map per A segment (host memory, kept alive here)
                    maps = (C.c_ubyte * (128 * a.n_seg))()
                    for j, (src, c, tap, st) in enumerate(L.segs):
                        t = self.buf[src]
                        _lib.call("fcn_encode_activation_map", C.addressof(maps) + 128 * j, _ptr(t),
                                  1, self.B * t.shape[1], t.shape[2], st)   # flattened padded rows
                    self._tmaps.append(maps)
                    a.tmaps = C.addressof(maps)
                    a.precision = 3 if nt == 128 else 4
                else:
                    a.precision = 1 if nt == 128 else 2
            a.round_out = 1 if (eng.precision == 1 and L.kind != "heads") else 0
            a.wt, a.bias = _ptr(L.wt), _ptr(L.bias)
            a.out, a.ld_out, a.T_store, a.c_off = _ptr(out), out.shape[2], self.valid_T[L.out], L.c_off
            a.P_store = out.shape[1]
            self.conv_args.append(a)

        self.mega_args = None
        self.mega_grid = 0
        if (eng.use_mega and eng.has_heads and self.heads_one_tile()
                and all(a.precision in (3, 4) for a in self.conv_args)):
            self._build_mega()

    def heads_one_tile(self):
        """The persistent kernel's heads epilogue decodes whole logit rows, so the heads layer must be ONE N tile
        (ld_logit <= 128).  Wider heads (e.g. 48 heading bins on SUN-RGBD, 64 on KITTI: ld_logit = 192, three
        64-column tiles) run the per-layer path: the GEMM per layer, then fcn_decode_eval."""
        return all(nt == L.n_cols for L, (_, _, nt) in zip(self.eng.layers, self.geom) if L.kind == "heads")

    def mega_descs(self):
        """Shape-level layer descriptions for the persistent FCN kernel (pure host arithmetic, testable on the CPU)."""
        eng = self.eng

        def build(wide):
            descs = []
            for L, (T_out, P_m, nt) in zip(eng.layers, self.geom):
                out = self.buf[L.out]
                if wide and L.n_cols % 256 == 0 and L.kind != "heads":
                    nt = 256
                descs.append(_mega.LayerDesc(L.name, L.kind, L.segs, L.K_pad, L.n_cols, L.Cout, L.up, L.relu, L.out,
                                             L.c_off, nt, int(L.kind != "heads"), P_m, T_out, self.B * P_m,
                                             out.shape[2], out.shape[1], self.valid_T[L.out]))
            return descs

        if eng.mega_nt256 == "auto":
            descs = build(True)
            if _mega.chain_tiles(descs) >= 24:
                return descs
            return build(False)
        return build(bool(eng.mega_nt256))

    def _build_mega(self):
        """Tables of the persistent FCN kernel (mega.py): tensor maps, layers, topologically ordered jobs."""
        eng, dev = self.eng, self.eng.device
        descs = self.mega_descs()
        map_keys, rows, jobs, nflags = _mega.build_tables(descs)
        maps = (C.c_ubyte * (128 * len(map_keys)))()
        for i, (kind, name, par) in enumerate(map_keys):
            t = self.buf[name]
            if kind == "load":      # A-operand boxes over the flattened padded rows, conv stride = par
                _lib.call("fcn_encode_activation_map", C.addressof(maps) + 128 * i, _ptr(t), 1, self.B * t.shape[1],
                          t.shape[2], par)
            else:                   # epilogue stores: one tensor row = `par` (= up) consecutive output rows
                _lib.call("fcn_encode_store_map", C.addressof(maps) + 128 * i, _ptr(t), self.B * t.shape[1] // par,
                          par * t.shape[2])
        ptrs = [(_ptr(L.tc_image(d.NT)), a.bias, a.out) for L, d, a in zip(eng.layers, descs, self.conv_args)]
        LA, JA = _mega.to_ctypes(descs, rows, jobs, ptrs)
        self._mega_host = (maps, LA)                   # HOST tables (copied into the kernel parameters per launch)
        self._mega_dev = torch.frombuffer(bytearray(bytes(JA)), dtype=torch.uint8).to(dev)
        self.mega_sync = torch.zeros(4 + nflags, dtype=torch.int32, device=dev)
        m = _lib.MegaArgs()
        grid = eng.mega_grid
        if grid <= 0:
            grid = max(4, min(48, (2 * _mega.chain_tiles(descs)) // 3))
        self.mega_grid = grid
        m.n_layers, m.n_jobs, m.n_flags, m.grid = len(descs), len(jobs), nflags, grid
        m.tmaps, m.n_maps = C.addressof(maps), len(map_keys)
        m.layers, m.jobs = C.addressof(LA), _ptr(self._mega_dev)
        m.sync = _ptr(self.mega_sync)
        m.B, m.T, m.NH, m.NS = self.B, self.T[1], eng.num_bins, eng.num_size
        m.center_ref, m.mean_size = _ptr(self.in_centers[1]), _ptr(eng.mean_size)
        m.n_out, m.n_flag_out = 1, 0
        self._set_decode_out(m.outs[0], self.out)
        self.mega_args = m
        self.mega_jobs = len(jobs)

    @staticmethod
    def _set_decode_out(slot, outs):
        (slot.cls_probs, slot.center, slot.heading, slot.size, slot.heading_probs, slot.size_probs) = \
            [_ptr(o) for o in outs]

    def set_peer_outputs(self, peer_block_ptrs, flag_ptrs=()):
        """Multi-GPU result exchange without a collective: `peer_block_ptrs` are device ADDRESSES of flat fp32
        blocks with the layout of ``out_flat`` (this rank's slot of every peer's gather buffer, peer memory mapped
        with fcn_ipc_open); the heads epilogue of the persistent FCN kernel stores the decoded rows into all of
        them over NVLink.  `flag_ptrs`: int32 device addresses that receive the forward's epoch number."""
        assert self.mega_args is not None, "peer outputs need the persistent FCN kernel (TF32 path)"
        assert self.graph is None, "set peer outputs before the first graph capture"
        m = self.mega_args
        assert 1 + len(peer_block_ptrs) <= _lib.MAX_PEERS and len(flag_ptrs) <= _lib.MAX_PEERS
        base = self.out_flat.data_ptr()
        offs = [o.data_ptr() - base for o in self.out]            # byte offsets of the six views in a block
        for i, ptr in enumerate(peer_block_ptrs):
            slot = m.outs[1 + i]
            (slot.cls_probs, slot.center, slot.heading, slot.size, slot.heading_probs, slot.size_probs) = \
                [int(ptr) + o for o in offs]
        m.n_out = 1 + len(peer_block_ptrs)
        for i, fp in enumerate(flag_ptrs):
            m.flag_out[i] = int(fp)
        m.n_flag_out = len(flag_ptrs)

    def _launch_mega(self, center_ref2):
        self.mega_args.center_ref = _ptr(center_ref2)
        _lib.call("fcn_mega_forward", C.byref(self.mega_args), _stream())

    def _launch_tail(self, center_ref2):
        """FCN + heads + decode: one persistent kernel, or (FCN_MEGA=0 / fp32) one launch per layer + decode."""
        if self.mega_args is not None:
            self._launch_mega(center_ref2)
        else:
            self._launch_fcn()
            self._launch_decode(center_ref2)

    # ---- launch sequences (all asynchronous on the current stream)
    def _launch_feat(self, pc, centers, one_hot):
        g = self.group_args
        g.pc = _ptr(pc)
        g.one_hot = _ptr(one_hot) if self.eng.num_vec > 0 else None
        for s, c in enumerate(centers):
            g.centers[s] = _ptr(c)
        main = torch.cuda.current_stream()
        _lib.call("fcn_group_rows", C.byref(g), main.cuda_stream)
        # the S scales are independent: fork them onto side streams (largest first, on the main stream)
        # so that the tile tail of one scale is filled by CTAs of the next (also inside the CUDA graph)
        S = len(self.pn_args)
        if S == 0:
            return
        if os.environ.get("FCN_NO_FORK", "0") == "1":      # diagnostics: everything on one stream
            for s_ in range(S - 1, -1, -1):
                _lib.call("fcn_pointnet_tiles", C.byref(self.pn_args[s_]), main.cuda_stream)
            return
        side = self._side_streams(S - 1)
        fork = torch.cuda.Event()
        fork.record(main)
        order = list(range(S - 1, -1, -1))
        joins = []
        for rank, s_ in enumerate(order):
            if rank == 0:
                _lib.call("fcn_pointnet_tiles", C.byref(self.pn_args[s_]), main.cuda_stream)
            else:
                st = side[rank - 1]
                st.wait_event(fork)
                _lib.call("fcn_pointnet_tiles", C.byref(self.pn_args[s_]), st.cuda_stream)
                ev = torch.cuda.Event()
                ev.record(st)
                joins.append(ev)
        for ev in joins:
            main.wait_event(ev)

    def _side_streams(self, n):
        while len(self._sides) < n:
            self._sides.append(torch.cuda.Stream(device=self.eng.device))
        return self._sides

    def _launch_fcn(self):
        """Main chain on the current stream; the transposed convs of all but the last block only
        feed the final concat, so they run on a side stream next to the following block."""
        main = torch.cuda.current_stream()
        layers = self.eng.layers
        deconvs = [i for i, L in enumerate(layers) if L.kind == "deconv"][:-1]
        side_of = {layers[i].segs[0][0]: self.conv_args[i] for i in deconvs}   # map read -> side deconv
        side = self._side_streams(1)[0] if side_of else None
        joins = []
        for i, (a, L) in enumerate(zip(self.conv_args, layers)):
            if i in deconvs:
                continue
            if L.kind == "heads":
                for ev in joins:
                    main.wait_event(ev)
                joins = []
            _lib.call("fcn_conv_gemm", C.byref(a), main.cuda_stream)
            da = side_of.get(L.out)
            if da is not None:
                ev = torch.cuda.Event()
                ev.record(main)
                side.wait_event(ev)
                _lib.call("fcn_conv_gemm", C.byref(da), side.cuda_stream)
                ev2 = torch.cuda.Event()
                ev2.record(side)
                joins.append(ev2)
        for ev in joins:
            main.wait_event(ev)

    def _launch_decode(self, center_ref2):
        eng = self.eng
        o = self.out
        _lib.call("fcn_decode_eval", self.B, self.T[1], self.P[1], eng.ld_logit, eng.num_bins, eng.num_size,
                  _ptr(self.buf["logits"]), _ptr(center_ref2), _ptr(eng.mean_size), _ptr(o[0]), _ptr(o[1]),
                  _ptr(o[2]), _ptr(o[3]), _ptr(o[4]), _ptr(o[5]), _stream())

    def _check_inputs(self, pc, centers, one_hot):
        assert pc.is_cuda and pc.dtype == torch.float32 and pc.is_contiguous()
        assert tuple(pc.shape) == (self.B, 3, self.N)
        for s, c in enumerate(centers):
            assert c.is_cuda and c.dtype == torch.float32 and c.is_contiguous()
            assert tuple(c.shape) == (self.B, 3, self.T[s])
        if self.eng.num_vec > 0:
            assert one_hot is not None and tuple(one_hot.shape) == (self.B, self.eng.num_vec)
            assert one_hot.dtype == torch.float32 and one_hot.is_contiguous()

    # ---- packed inputs (zero / single-copy staging for graph replay)
    def input_views(self):
        """The plan's own input tensors as a reference-style dict: fill them in place (e.g. H2D copy
        into ``in_flat``) and pass this dict to the model to skip the staging copy."""
        d = {"point_cloud": self.in_pc}
        for s, c in enumerate(self.in_centers):
            d["center_ref%d" % (s + 1)] = c
        if self.eng.num_vec > 0:
            d["one_hot"] = self.in_onehot
        return d

    def pack(self, data, pin=False, device=None):
        """Pack a reference-style dict into one flat tensor with this plan's input layout; returns
        (flat, dict of views).  Staging such a dict costs one device copy instead of S+2."""
        flat = torch.zeros(self.in_flat.numel(), dtype=torch.float32,
                           device=device if device is not None else "cpu")
        if pin:
            flat = flat.pin_memory()
        keys = ["point_cloud"] + ["center_ref%d" % (s + 1) for s in range(len(self.in_centers))] + ["one_hot"]
        views = {}
        for k, off, ref in zip(keys, self._in_offs, [self.in_pc] + self.in_centers + [self.in_onehot]):
            if k not in data:
                continue
            v = flat[off: off + ref.numel()].view(ref.shape)
            v.copy_(torch.as_tensor(data[k]))
            views[k] = v
        return flat, views

    def _stage(self, pc, centers, one_hot):
        base = self.in_flat.data_ptr()
        if pc.data_ptr() == base:
            return                                   # caller filled the plan's own input block
        off0 = pc.data_ptr()
        packed = all(c.data_ptr() - off0 == 4 * o for c, o in zip(centers, self._in_offs[1:1 + len(centers)]))
        if packed and self.eng.num_vec > 0:
            packed = one_hot.data_ptr() - off0 == 4 * self._in_offs[-1]
        if packed and pc.untyped_storage().nbytes() - pc.storage_offset() * 4 >= self.in_flat.numel() * 4:
            src = torch.as_strided(pc, (self.in_flat.numel(),), (1,))
            self.in_flat.copy_(src, non_blocking=True)   # one copy for the whole packed batch
            return
        self.in_pc.copy_(pc, non_blocking=True)
        for d, c in zip(self.in_centers, centers):
            d.copy_(c, non_blocking=True)
        if self.eng.num_vec > 0:
            self.in_onehot.copy_(one_hot, non_blocking=True)

    def _views(self, flat):
        outs, off = [], 0
        for o in self.out:
            outs.append(flat[off: off + o.numel()].view(o.shape))
            off += o.numel()
        return tuple(outs)

    def run(self, pc, centers, one_hot, use_graph=False, copy_out=True, trusted=False):
        """copy_out=True returns fresh tensors (reference semantics); False returns views of the
        plan's output block, which the next call overwrites (zero-copy serving / benchmarking)."""
        out = self._run(pc, centers, one_hot, use_graph, trusted)
        return self._views(self.out_flat.clone()) if copy_out else out

    def _run(self, pc, centers, one_hot, use_graph=False, trusted=False):
        own = use_graph and pc.data_ptr() == self.in_flat.data_ptr()   # the plan's own input views: valid by construction
        if not own and not trusted:
            self._check_inputs(pc, centers, one_hot)
        dev = self.eng.device
        if dev.index is not None and torch.cuda.current_device() != dev.index:
            with torch.cuda.device(dev):
                return self._run_on_device(pc, centers, one_hot, use_graph, own)
        return self._run_on_device(pc, centers, one_hot, use_graph, own)

    def _run_on_device(self, pc, centers, one_hot, use_graph, own):
        if not use_graph:
            self._launch_feat(pc, centers, one_hot)
            self._launch_tail(centers[1])
            return self.out
        if not own:
            self._stage(pc, centers, one_hot)
        if self.graph is None:
            self._capture()
        self.graph.replay()
        return self.out

    def _capture(self):
        skip = set(os.environ.get("FCN_DIAG_SKIP", "").split(","))   # timing diagnostics only

        def seq():
            if "feat" not in skip:
                self._launch_feat(self.in_pc, self.in_centers, self.in_onehot)
            if "fcn" not in skip:
                self._launch_tail(self.in_centers[1])

        seq()   # warm-up run outside capture (sets function attributes, loads modules)
        torch.cuda.current_stream().synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            seq()
        self.graph = g

    def forward_staged(self, pc, centers, one_hot):
        """Eval forward for a consumer of the head logits (``head_logits``): the inputs are copied into the plan's own
        block and the forward graph is replayed (captured on the first call, which synchronizes once).  While the
        current stream is being captured, the launch sequence itself is recorded into the caller's graph instead.
        No host sync otherwise; the decoded outputs are written as by ``run``."""
        self._check_inputs(pc, centers, one_hot)
        with torch.cuda.device(self.eng.device):
            self._stage(pc, centers, one_hot)
            if torch.cuda.is_current_stream_capturing():
                self._launch_feat(self.in_pc, self.in_centers, self.in_onehot)
                self._launch_tail(self.in_centers[1])
                return
            if self.graph is None:
                self._capture()
            self.graph.replay()

    def head_logits(self):
        """(logits, pitch, ld_logit, center_ref2) of the last ``forward_staged``: the pitched head-logit buffer
        (B, pitch, ld_logit) whose row (b, t < T2) is [cls0, cls1, regression...], and the staged (B, 3, T2) refs."""
        return self.buf["logits"], self.P[1], self.eng.ld_logit, self.in_centers[1]

    def run_feat(self, pc, centers, one_hot):
        self._check_inputs(pc, centers, one_hot)
        eng = self.eng
        with torch.cuda.device(eng.device):
            self._launch_feat(pc, centers, one_hot)
            outs = []
            for s in range(eng.arch.num_scales):
                c = eng.c3[s] + eng.num_vec
                o = torch.empty((self.B, c, self.T[s]), dtype=torch.float32, device=eng.device)
                _lib.call("fcn_btc_to_bct", self.B, c, self.T[s], self.P[s], eng.ld_feat[s],
                          _ptr(self.buf["feat%d" % (s + 1)]), _ptr(o), _stream())
                outs.append(o)
        return tuple(outs)

    def run_fcn_bct(self, feats_bct):
        eng = self.eng
        with torch.cuda.device(eng.device):
            for s, f in enumerate(feats_bct):
                c = eng.c3[s] + eng.num_vec
                assert f.is_cuda and f.dtype == torch.float32 and f.is_contiguous()
                assert tuple(f.shape) == (self.B, c, self.T[s]), "feat%d has shape %s" % (s + 1, tuple(f.shape))
                _lib.call("fcn_bct_to_btc", self.B, c, self.T[s], self.P[s], eng.ld_feat[s], _ptr(f),
                          _ptr(self.buf["feat%d" % (s + 1)]), _stream())
            st = _stream()
            for a, L in zip(self.conv_args, eng.layers):
                if L.kind == "heads":
                    continue
                _lib.call("fcn_conv_gemm", C.byref(a), st)
            cat = self.buf["cat"]
            T2 = self.T[1]
            o = torch.empty((self.B, cat.shape[2], T2), dtype=torch.float32, device=eng.device)
            _lib.call("fcn_btc_to_bct", self.B, cat.shape[2], T2, cat.shape[1], cat.shape[2], _ptr(cat), _ptr(o), st)
        return o

    def time_kernels(self, dev_pool, iters=20):
        """Per-kernel device time, measured live with CUDA events on the launching stream: each
        C-ABI call is captured `iters` times back to back into one CUDA graph, which is replayed
        between two events (hot L2, no host launch overhead; includes the inter-kernel gap exactly
        like the whole-forward graph does).  Also returns executed/nominal FLOPs per launch."""
        eng, S = self.eng, self.eng.arch.num_scales
        mega = self.mega_args is not None
        names = ["group_rows"] + ["pointnet_s%d" % (s + 1) for s in range(S)] + \
            (["fcn_mega"] if mega else [L.name for L in eng.layers] + ["decode_eval"])
        d = dev_pool[0]
        self.in_pc.copy_(d["point_cloud"])
        for dst, i in zip(self.in_centers, range(S)):
            dst.copy_(d["center_ref%d" % (i + 1)])
        if eng.num_vec > 0:
            self.in_onehot.copy_(d["one_hot"])
        g = self.group_args
        g.pc, g.one_hot = _ptr(self.in_pc), _ptr(self.in_onehot) if eng.num_vec > 0 else None
        for s_, c in enumerate(self.in_centers):
            g.centers[s_] = _ptr(c)

        def call_group():
            _lib.call("fcn_group_rows", C.byref(g), _stream())

        calls = [call_group]
        calls += [(lambda a=a: _lib.call("fcn_pointnet_tiles", C.byref(a), _stream())) for a in self.pn_args]
        if mega:
            calls += [lambda: self._launch_mega(self.in_centers[1])]
        else:
            calls += [(lambda a=a: _lib.call("fcn_conv_gemm", C.byref(a), _stream())) for a in self.conv_args]
            calls += [lambda: self._launch_decode(self.in_centers[1])]
        acc = np.zeros(len(names))
        with torch.cuda.device(eng.device):
            for fn in calls:       # eager warm-up of the whole sequence (valid tiles/feats for later kernels)
                fn()
            torch.cuda.synchronize()
            for i, fn in enumerate(calls):
                gr = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gr):     # `iters` back-to-back launches of the same kernel in ONE graph
                    for _ in range(iters):
                        fn()
                gr.replay()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                reps = 3
                e0.record()
                for _ in range(reps):
                    gr.replay()
                e1.record()
                torch.cuda.synchronize()
                acc[i] = e0.elapsed_time(e1) / (iters * reps)
                del gr
        rows_exec = [int(c.sum().item()) for c in self.cnt]
        rows_nom = [self.B * self.T[s] * eng.arch.nsample[s] for s in range(S)]
        kern = [dict(name="group_rows", ms=float(acc[0]), executed_gflop=0.0, nominal_gflop=0.0)]
        sm = torch.cuda.get_device_properties(eng.device).multi_processor_count
        ntiles = self.ntiles.cpu().tolist()

        def balanced(n, slots):          # csrc/wgmma.cuh balanced_stride
            rounds = -(-n // slots)
            return -(-n // rounds) if n > 0 else 0

        for s in range(S):
            c1, c2, c3 = eng.arch.mlps[s]
            mac = 3 * c1 + c1 * c2 + c2 * c3
            a = self.pn_args[s]
            nt = min(int(ntiles[s]), int(a.max_tiles))
            if a.precision == 2:         # 2-CTA clusters, one tile pair per cluster and round
                sms = 2 * balanced((nt + 1) // 2, sm // 2)
            elif a.precision == 1:       # persistent 1-CTA kernel, two CTAs per SM at <= 64 channels
                per_sm = 2 if c1 <= 64 else 1
                sms = min(sm, -(-balanced(nt, sm * per_sm) // per_sm))
            else:
                sms = sm
            kern.append(dict(name="pointnet_s%d" % (s + 1), ms=float(acc[1 + s]), sms=int(sms), tiles=nt,
                             executed_gflop=2e-9 * mac * rows_exec[s], nominal_gflop=2e-9 * mac * rows_nom[s]))
        fcn_gf = []
        for j, (L, a) in enumerate(zip(eng.layers, self.conv_args)):
            kreal = sum(sg[1] for sg in L.segs)
            nreal = (2 + eng.out_size) if L.kind == "heads" else L.up * L.Cout
            fcn_gf.append(2e-9 * a.B * a.T_out * kreal * nreal)
        if mega:
            kern.append(dict(name="fcn_mega", ms=float(acc[1 + S]), executed_gflop=sum(fcn_gf), nominal_gflop=sum(fcn_gf)))
        else:
            for j, L in enumerate(eng.layers):
                kern.append(dict(name=L.name, ms=float(acc[1 + S + j]), executed_gflop=fcn_gf[j], nominal_gflop=fcn_gf[j]))
            kern.append(dict(name="decode_eval", ms=float(acc[-1]), executed_gflop=0.0, nominal_gflop=0.0))
        for k_ in kern:
            k_["executed_tflops"] = k_["executed_gflop"] / max(k_["ms"], 1e-9)  # GFLOP/ms == TFLOP/s
        return dict(kernels=kern, launches_per_step=len(names) + 1,   # group_rows = count + emit kernels
                    unique_row_fraction=float(sum(rows_exec)) / float(max(sum(rows_nom), 1)))

    def logits(self):
        """(B*T2, 2) class scores and (B*T2, out) regression rows of the last run (views)."""
        lg = self.buf["logits"][:, :self.T[1], :].reshape(-1, self.eng.ld_logit)
        return lg[:, 0:2], lg[:, 2:2 + self.eng.out_size]


def _run_module(eng: FrustumEngine, scale: int, pc, new_pc):
    """PointNetModule.forward (det_base.py:62-103): un-pooled masked (B,C3,T,K)."""
    assert pc.is_cuda and pc.is_contiguous() and new_pc.is_contiguous()
    B, N, T = pc.shape[0], pc.shape[2], new_pc.shape[2]
    K = eng.arch.nsample[scale]
    c1, c2, c3 = eng.arch.mlps[scale]
    dev, f32 = eng.device, torch.float32
    tr = 64
    with torch.cuda.device(dev):
        rows = torch.empty((B, T * K, 4), dtype=f32, device=dev)
        cnt = torch.empty((B, T), dtype=torch.int32, device=dev)
        mt = B * ((T * K + tr - 1) // tr)
        tiles = torch.empty((max(mt, 1), 4), dtype=torch.int32, device=dev)
        ntiles = torch.zeros(_lib.MAX_SCALES, dtype=torch.int32, device=dev)
        out = torch.empty((B, c3, T, K), dtype=f32, device=dev)
        g = _lib.GroupArgs()
        g.num_scales, g.B, g.N, g.num_vec, g.tile_rows, g.unique_rows = 1, B, N, 0, tr, 0
        g.pc, g.one_hot = _ptr(pc), None
        g.centers[0], g.T[0], g.K[0], g.dis_z[0] = _ptr(new_pc), T, K, eng.dists[scale]
        g.c3[0], g.ld_feat[0], g.row_cap[0], g.tile_cap[0] = c3, 0, T * K, max(mt, 1)
        g.rows[0], g.cnt[0], g.feat[0], g.tiles[0] = _ptr(rows), _ptr(cnt), None, _ptr(tiles)
        idx32 = torch.empty((B, T, K), dtype=torch.int32, device=dev)
        g.idx_scratch[0] = _ptr(idx32)
        g.ntiles = _ptr(ntiles)
        st = _stream()
        _lib.call("fcn_group_rows", C.byref(g), st)
        a = _lib.PointnetArgs()
        a.C1, a.C2, a.C3, a.T, a.K = c1, c2, c3, T, K
        a.ld_feat, a.row_cap, a.tile_rows, a.unpooled, a.precision, a.B = 0, T * K, tr, 1, 0, B
        a.rows, a.tiles, a.ntiles, a.max_tiles = _ptr(rows), _ptr(tiles), _ptr(ntiles), mt
        w = eng.pn[scale]
        a.w1t, a.b1, a.w2t, a.b2, a.w3t, a.b3 = (_ptr(w["w1t"]), _ptr(w["b1"]), _ptr(w["w2t"]),
                                                _ptr(w["b2"]), _ptr(w["w3t"]), _ptr(w["b3"]))
        a.out = _ptr(out)
        _lib.call("fcn_pointnet_tiles", C.byref(a), st)
    return out
