"""Host side of the training step on hand-written kernels (config 5: cfgs/refine_car.yaml).

Mirrors what PointNetDet does in train() mode (/root/reference/models/det_base.py:334-375 up to the head logits;
layer factories models/common.py:38-63) as a table of ``fcn_train_layer`` records over dense position-major
tensors, executed by csrc/train.cu:

    grouping (fcn_group_rows, all T*K rows incl. the reference's back-fill duplicates - they weight the batch
    statistics)  ->  per scale conv1..3 (+BN batch stats) -> mask + max over K -> FCN -> deconvs -> heads

``TrainStep`` takes the losses and dlogits of the (B*T2, 2+39) logits from the fused loss kernels (csrc/loss.cu), the
drop-in ``model(data)`` path from PyTorch ops and their autograd (train_path.losses_from_logits); from dlogits
``backward`` runs the hand-written backward kernels.  Parameters live in ONE flat fp32 buffer (every
``nn.Parameter`` is a view), gradients in ONE flat bucket written in the parameter layout by the kernels:
one ``all_reduce`` per step (SURVEY.md 8(e)) and one fused optimizer launch (``fcn_adam_step`` or ``fcn_sgd_step``).
BatchNorm statistics are per rank (the reference's DataParallel semantics: per-replica BN, no SyncBN).  In
deterministic mode the gradient is summed over the ranks in rank order (all-to-all, ``fcn_rank_fold``, all-gather)
and every rank adopts rank 0's BN running statistics after each step, DataParallel's replica-0 buffers.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence

import numpy as np
import torch

from . import _lib
from .config import fcn_layers


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _stream():
    return torch.cuda.current_stream().cuda_stream


class FlatParams:
    """All parameters of a module as views of one flat fp32 buffer (+ a flat gradient bucket of the same layout)."""

    def __init__(self, module: torch.nn.Module):
        ps = [p for p in module.parameters()]
        assert all(p.dtype == torch.float32 and p.is_cuda for p in ps), "fp32 CUDA parameters expected"
        n = sum(p.numel() for p in ps)
        dev = ps[0].device
        self.param = torch.empty(n, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(n, dtype=torch.float32, device=dev)
        self.offsets: Dict[int, int] = {}
        off = 0
        for p in ps:
            k = p.numel()
            self.param[off: off + k].copy_(p.data.reshape(-1))
            p.data = self.param[off: off + k].view(p.shape)
            self.offsets[id(p)] = off
            off += k
        self.numel = n

    @staticmethod
    def of(model) -> "FlatParams":
        """The model's bucket: created on first use and cached on the model, so every TrainStep and TrainEngine of
        one model shares it."""
        flat = getattr(model, "_flat_params", None)
        if flat is None:
            flat = model._flat_params = FlatParams(model)
        return flat

    def gptr(self, p) -> int:
        return self.grad.data_ptr() + 4 * self.offsets[id(p)]

    def grad_view(self, p) -> torch.Tensor:
        off = self.offsets[id(p)]
        return self.grad[off: off + p.numel()].view(p.shape)

    def expose_grads(self, module):
        """``p.grad`` = view of the flat bucket (what an optimizer or a test reads after TrainStep.forward_backward)."""
        for p in module.parameters():
            p.grad = self.grad_view(p)


class LogitsFn(torch.autograd.Function):
    """autograd bridge for the reference's own training loop (``losses, _ = model(data); loss.backward();
    optimizer.step()``, train/train_net_det.py:121-128): forward = the kernel forward up to the head logits,
    backward = the kernel backward; parameter gradients are returned to autograd as copies of the flat bucket."""

    @staticmethod
    def forward(ctx, eng, pc, one_hot, ncent, *rest):
        centers, params = rest[:ncent], rest[ncent:]
        cls, reg = eng.forward(pc, list(centers), one_hot)
        ctx.eng, ctx.params, ctx.ncent = eng, params, ncent
        return cls.clone(), reg.clone()

    @staticmethod
    def backward(ctx, dcls, dreg):
        eng = ctx.eng
        eng.flat.grad.zero_()
        eng.backward(dcls.contiguous(), dreg.contiguous())
        grads = tuple(eng.flat.grad_view(p).clone() for p in ctx.params)
        return (None, None, None, None) + (None,) * ctx.ncent + grads


class TrainEngine:
    """Kernel tables + workspaces of one PointNetDet for one input shape (B, N, T...).  ``deterministic``: the
    layers run on ``fcn_train_forward_deterministic`` / ``fcn_train_backward_deterministic`` (bit-reproducible)."""

    def __init__(self, model, B: int, N: int, T: Sequence[int], deterministic: bool = False):
        self.model = model
        self.deterministic = bool(deterministic)
        arch = model.ARCH
        S = arch.num_scales
        assert len(T) == S
        self.B, self.N, self.T = int(B), int(N), tuple(int(t) for t in T)
        self.dev = next(model.parameters()).device
        self.V = model.num_vec
        self.flat = FlatParams.of(model)
        dev, f32 = self.dev, torch.float32
        K = arch.nsample
        self.K = K
        # ---- grouping workspace (all T*K rows per section: unique_rows = 0)
        self.rows = [torch.empty((B * T[s] * K[s], 4), dtype=f32, device=dev) for s in range(S)]
        self.cnt = [torch.empty((B, T[s]), dtype=torch.int32, device=dev) for s in range(S)]
        self.tiles = [torch.empty((B * ((T[s] * K[s] + 63) // 64) + 1, 4), dtype=torch.int32, device=dev) for s in range(S)]
        self.idx32 = [torch.empty((B, T[s], K[s]), dtype=torch.int32, device=dev) for s in range(S)]
        self.ntiles = torch.zeros(_lib.MAX_SCALES, dtype=torch.int32, device=dev)
        # ---- layer list: (name, ctypes layer, out key); activations keyed by name
        self.layers: List[_lib.TrainLayer] = []
        self.names: List[str] = []
        self.dx_mask: List[int] = []
        self.act: Dict[str, dict] = {}
        self._zero_fwd: List[torch.Tensor] = []     # fp64 Sum(y), Sum(y^2)
        self._zero_bwd: List[torch.Tensor] = []     # fp64 Sum(dz), Sum(dz*xh) and all dA / dfeat buffers
        self._keep = []

        def new_act(name, rows, cols, T_pos, up=1, cout=None, bn=None, relu=1, grad=True):
            a = dict(rows=rows, cols=cols, T=T_pos, up=up, cout=cout or cols, relu=relu)
            a["Y"] = torch.empty((rows, cols), dtype=f32, device=dev)
            a["dA"] = torch.zeros((rows, cols), dtype=f32, device=dev) if grad else None
            if grad:
                self._zero_bwd.append(a["dA"])
            if bn is not None:
                a["bn"] = bn
                a["sums"] = torch.zeros(2 * a["cout"], dtype=torch.float64, device=dev)
                a["dsums"] = torch.zeros(2 * a["cout"], dtype=torch.float64, device=dev)
                self._zero_fwd.append(a["sums"])
                self._zero_bwd.append(a["dsums"])
            self.act[name] = a
            return a

        def src_of(name, c0=0):
            a = self.act[name]
            s = _lib.TrainSrc()
            s.raw, s.grad = _ptr(a["Y"]), _ptr(a.get("dA"))
            bn = a.get("bn")
            if bn is not None:
                s.sums, s.gamma, s.beta = _ptr(a["sums"]), _ptr(bn.weight), _ptr(bn.bias)
                s.count = float(a["rows"] * a["up"])
                s.Cstat, s.coff, s.relu = a["cout"], 0, a["relu"]
            else:
                s.sums = None
                s.count, s.Cstat, s.coff, s.relu = 1.0, 1, 0, 0
            s.ld, s.T, s.up, s.cup, s.c0 = a["cols"], a["T"], a["up"], a["cout"], c0
            return s

        def add_layer(name, out, segs, conv, bn, N_cols, cout, up, s_co, s_j, T_out, bias=None, dx=True):
            L = _lib.TrainLayer()
            L.B, L.T_out, L.n_seg, L.N, L.Cout, L.up = B, T_out, len(segs), N_cols, cout, up
            L.s_co, L.s_j, L.has_bn, L.relu = s_co, s_j, (1 if bn is not None else 0), (1 if bn is not None else 0)
            mask = 0
            for i, (srcname, Cc, tap, stride, s_ci, w_off) in enumerate(segs):
                g = L.seg[i]
                g.src = src_of(srcname)
                g.C, g.tap, g.stride, g.s_ci, g.w_off = Cc, tap, stride, s_ci, w_off
                if dx and self.act[srcname].get("dA") is not None:
                    mask |= 1 << i
            a = self.act[out]
            L.W, L.dW = _ptr(conv.weight), self.flat.gptr(conv.weight)
            if bias is not None:
                L.bias, L.dbias = _ptr(bias), self.flat.gptr(bias)
            L.Y, L.dA = _ptr(a["Y"]), _ptr(a["dA"])
            if bn is not None:
                L.sums, L.dsums = _ptr(a["sums"]), _ptr(a["dsums"])
                L.gamma, L.beta = _ptr(bn.weight), _ptr(bn.bias)
                L.dgamma, L.dbeta = self.flat.gptr(bn.weight), self.flat.gptr(bn.bias)
                L.run_mean, L.run_var = _ptr(bn.running_mean), _ptr(bn.running_var)
            else:
                a["dsums"] = torch.zeros(2 * N_cols, dtype=torch.float64, device=dev)
                self._zero_bwd.append(a["dsums"])
                L.dsums = _ptr(a["dsums"])
            self.layers.append(L)
            self.names.append(name)
            self.dx_mask.append(mask)

        # ---- PointNet scales
        self.pools = []
        fn = model.feat_net
        for s in range(S):
            c1, c2, c3 = arch.mlps[s]
            pm = getattr(fn, "pointnet%d" % (s + 1))
            TK = T[s] * K[s]
            rname = "rows%d" % (s + 1)
            self.act[rname] = dict(rows=B * TK, cols=4, T=TK, up=1, cout=4, relu=0, Y=self.rows[s], dA=None)
            prev, pc = rname, 3
            for j, co in enumerate((c1, c2, c3)):
                blk = getattr(pm, "conv%d" % (j + 1))
                nm = "pn%d_%d" % (s + 1, j + 1)
                new_act(nm, B * TK, co, TK, bn=blk[1])
                add_layer(nm, nm, [(prev, pc, 0, 1, 1, 0)], blk[0], blk[1], co, co, 1, pc, 0, TK, dx=(j > 0))
                prev, pc = nm, co
            # pooled feature (+ one-hot columns): identity source for the FCN
            fname = "feat%d" % (s + 1)
            fa = dict(rows=B * T[s], cols=c3 + self.V, T=T[s], up=1, cout=c3 + self.V, relu=0)
            fa["Y"] = torch.zeros((B * T[s], c3 + self.V), dtype=f32, device=dev)
            fa["dA"] = torch.zeros((B * T[s], c3 + self.V), dtype=f32, device=dev)
            self._zero_bwd.append(fa["dA"])
            self.act[fname] = fa
            P = _lib.TrainPool()
            last = self.act[prev]
            P.B, P.T, P.K, P.C, P.V, P.ld_feat = B, T[s], K[s], c3, self.V, c3 + self.V
            P.Y, P.cnt, P.sums = _ptr(last["Y"]), _ptr(self.cnt[s]), _ptr(last["sums"])
            P.gamma, P.beta = _ptr(last["bn"].weight), _ptr(last["bn"].bias)
            argmax = torch.zeros((B * T[s], c3), dtype=torch.int32, device=dev)
            self._keep.append(argmax)
            P.feat, P.argmax, P.dfeat, P.dA = _ptr(fa["Y"]), _ptr(argmax), _ptr(fa["dA"]), _ptr(last["dA"])
            self.pools.append(P)
        self.n_pn_layers = len(self.layers)
        # ---- ConvFeatNet + heads.  Weight index of (co, ci, tap j): conv / merge co * Ci * k + ci * k + j,
        # transposed conv ci * Cout * k + co * k + j
        for i in range(1, S):
            assert T[i] == (T[i - 1] + 1) // 2, "section counts are not a /2 pyramid"
        table = {L.name: L for L in fcn_layers(arch, self.V)}
        for L in table.values():
            ci = sum(c for _, c in L.srcs)
            if L.kind == "heads":     # on the cropped concat of the transposed-conv outputs (det_base.py:222-224,367-368)
                segs = [(src, c, 0, 1, 1, table[src].c_off) for src, c in L.srcs]
                for nm, conv in (("cls_out", model.cls_out), ("reg_out", model.reg_out)):
                    co = conv.weight.shape[0]
                    new_act(nm, B * T[L.level], co, T[L.level], bn=None)
                    add_layer(nm, nm, segs, conv, None, co, co, 1, ci, 0, T[L.level], bias=conv.bias)
                continue
            blk = getattr(model.conv_net, L.name)
            if L.kind == "deconv":    # one row per input position, k output positions per row
                src, Tin = L.srcs[0][0], self.act[L.srcs[0][0]]["T"]
                new_act(L.name, B * Tin, L.k * L.Cout, Tin, up=L.k, cout=L.Cout, bn=blk[1])
                add_layer(L.name, L.name, [(src, ci, 0, 1, L.Cout * L.k, 0)], blk[0], blk[1], L.k * L.Cout, L.Cout,
                          L.k, L.k, 1, Tin)
            else:
                c0 = np.cumsum([0] + [c for _, c in L.srcs]).tolist()
                segs = [(src, c, j - L.k // 2, L.stride, L.k, c0[n] * L.k + j)
                        for j in range(L.k) for n, (src, c) in enumerate(L.srcs)]
                new_act(L.name, B * T[L.level], L.Cout, T[L.level], bn=blk[1])
                add_layer(L.name, L.name, segs, blk[0], blk[1], L.Cout, L.Cout, 1, ci * L.k, 0, T[L.level])
        self.T2 = T[1]
        # device copy of the layer table for the end-of-step kernel
        arr = (_lib.TrainLayer * len(self.layers))(*self.layers)
        self._table_host = arr
        self.table_dev = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev)
        self._bn_counters = [b for n, b in model.named_buffers() if n.endswith("num_batches_tracked")]
        # static inputs (the launch sequences are captured into CUDA graphs)
        self.in_pc = torch.zeros((B, 3, N), dtype=f32, device=dev)
        self.in_centers = [torch.zeros((B, 3, T[s]), dtype=f32, device=dev) for s in range(S)]
        self.in_onehot = torch.zeros((B, max(self.V, 1)), dtype=f32, device=dev)
        for P in self.pools:
            P.one_hot = _ptr(self.in_onehot) if self.V > 0 else None
        self.group_args = self._group_args()
        self._graphs = {}
        self.use_graph = True
        lib = _lib.load()
        query = lib.fcn_train_deterministic_workspace_floats if self.deterministic else lib.fcn_train_workspace_floats
        need = max([int(query(C.byref(L))) for L in self.layers] + [1])
        # K-split partial sums of the skinny FCN layers; deterministic mode: also the slots and slices of its sums
        self.workspace = torch.empty(need, dtype=f32, device=dev)

    # ------------------------------------------------------------------
    def _group_args(self):
        g = _lib.GroupArgs()
        arch = self.model.ARCH
        S = arch.num_scales
        g.num_scales, g.B, g.N, g.num_vec, g.tile_rows, g.unique_rows = S, self.B, self.N, 0, 64, 0
        dists = self.model.feat_net.dists
        for s in range(S):
            g.T[s], g.K[s], g.dis_z[s] = self.T[s], self.K[s], float(dists[s])
            g.c3[s], g.ld_feat[s] = arch.mlps[s][2], 0
            g.row_cap[s] = self.T[s] * self.K[s]
            g.tile_cap[s] = self.tiles[s].shape[0]
            g.rows[s], g.cnt[s], g.feat[s], g.tiles[s] = _ptr(self.rows[s]), _ptr(self.cnt[s]), None, _ptr(self.tiles[s])
            g.idx_scratch[s] = _ptr(self.idx32[s])
            g.feat_pitch[s] = 0
        g.ntiles = _ptr(self.ntiles)
        g.force_scan = 0
        g.pc, g.one_hot = _ptr(self.in_pc), None
        for s in range(S):
            g.centers[s] = _ptr(self.in_centers[s])
        return g

    # ---- launch sequences (all pointers are static: the step is CUDA-graph capturable)
    def _layer_forward(self, li, st):
        if self.deterministic:
            _lib.call("fcn_train_forward_deterministic", C.byref(self.layers[li]), _ptr(self.workspace),
                      self.workspace.numel(), st)
        else:
            _lib.call("fcn_train_forward", C.byref(self.layers[li]), _ptr(self.workspace), self.workspace.numel(), st)

    def _layer_backward(self, li, st):
        if self.deterministic:
            _lib.call("fcn_train_backward_deterministic", C.byref(self.layers[li]), self.dx_mask[li],
                      _ptr(self.workspace), self.workspace.numel(), st)
        else:
            _lib.call("fcn_train_backward", C.byref(self.layers[li]), self.dx_mask[li], st)

    def _seq_forward(self):
        S = len(self.T)
        st = _stream()
        torch._foreach_zero_(self._zero_fwd)
        _lib.call("fcn_group_rows", C.byref(self.group_args), st)
        li = 0
        for s in range(S):
            for _ in range(3):
                self._layer_forward(li, st)
                li += 1
            _lib.call("fcn_train_pool", C.byref(self.pools[s]), 0, st)
        while li < len(self.layers):
            self._layer_forward(li, st)
            li += 1

    def _seq_backward(self, stage, update_running):
        st = _stream()
        S = len(self.T)
        if stage in ("all", "fcn"):
            # FCN + heads in reverse creation order (a topological order of the backward graph: every consumer of
            # a tensor was created after it)
            for li in range(len(self.layers) - 1, self.n_pn_layers - 1, -1):
                self._layer_backward(li, st)
            # BN bookkeeping of the FCN layers: their dgamma / dbeta belong to the first gradient bucket
            nf = len(self.layers) - self.n_pn_layers
            _lib.call("fcn_train_finalize", _ptr(self.table_dev) + self.n_pn_layers * C.sizeof(_lib.TrainLayer), nf,
                      1 if update_running else 0, st)
        if stage in ("all", "pointnet"):
            for s in range(S - 1, -1, -1):
                _lib.call("fcn_train_pool", C.byref(self.pools[s]), 1, st)
                for j in (2, 1, 0):
                    li = 3 * s + j
                    self._layer_backward(li, st)
            _lib.call("fcn_train_finalize", _ptr(self.table_dev), self.n_pn_layers, 1 if update_running else 0, st)
            if update_running and self._bn_counters:
                torch._foreach_add_(self._bn_counters, 1)

    def _graph(self, key, fn):
        """Capture `fn` once (after an eager warm-up run, whose effects are the first execution) and replay it."""
        g = self._graphs.get(key)
        if g is None:
            fn()                                   # eager: this call's work
            try:
                torch.cuda.current_stream().synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    fn()
                self._graphs[key] = g
            except Exception as e:                 # stay functional without graphs
                import sys
                sys.stderr.write("TrainEngine: CUDA-graph capture of %r failed (%r); launching eagerly\n" % (key, e))
                self._graphs[key] = False
                torch.cuda.synchronize()
            return
        if g is False:
            fn()
        else:
            g.replay()

    @torch.no_grad()
    def forward(self, pc, centers, one_hot):
        """-> (cls logits (B*T2, 2), reg logits (B*T2, out)) as views of the engine's buffers."""
        assert tuple(pc.shape) == (self.B, 3, self.N) and pc.dtype == torch.float32
        self.in_pc.copy_(pc)
        for s, c in enumerate(centers):
            assert tuple(c.shape) == (self.B, 3, self.T[s])
            self.in_centers[s].copy_(c)
        if self.V > 0:
            self.in_onehot.copy_(one_hot)
        if self.use_graph:
            self._graph("fwd", self._seq_forward)
        else:
            self._seq_forward()
        return self.act["cls_out"]["Y"], self.act["reg_out"]["Y"]

    @torch.no_grad()
    def backward(self, dcls, dreg, update_running=True, stage="all"):
        """dlogits -> gradients of every parameter, ACCUMULATED into the flat bucket ``self.flat.grad``.
        stage = "fcn" (heads + ConvFeatNet: everything the feat_net gradients depend on), "pointnet" (the rest +
        BN bookkeeping) or "all"."""
        if stage in ("all", "fcn"):
            torch._foreach_zero_(self._zero_bwd)
            self.act["cls_out"]["dA"].copy_(dcls.reshape(self.act["cls_out"]["dA"].shape))
            self.act["reg_out"]["dA"].copy_(dreg.reshape(self.act["reg_out"]["dA"].shape))
        if self.use_graph:
            self._graph(("bwd", stage, bool(update_running)), lambda: self._seq_backward(stage, update_running))
        else:
            self._seq_backward(stage, update_running)

    def kernel_launches_per_step(self):
        """Launches of one step in the DEFAULT mode (the layer GEMMs, pools, grouping, finalize and the optimizer).
        The deterministic mode adds its ordered-sum launches (slots, dW and dX slices), which this does not count."""
        n_fwd = len(self.layers) + len(self.pools) + 2
        n_bwd = sum(1 + L.n_seg + bin(m).count("1") for L, m in zip(self.layers, self.dx_mask)) + len(self.pools) + 1
        return n_fwd + n_bwd + 1      # + fused Adam or SGD


def piece_split(model) -> int:
    """Where the flat bucket is cut in two for the reduction over ranks: [0, split) is the PointNet (feat_net) piece,
    [split, n) the ConvFeatNet + heads piece, whose gradient is complete first."""
    first = next(model.conv_net.parameters())
    off = 0
    for p in model.parameters():
        if p is first:
            return off
        off += p.numel()
    raise ValueError("the model's conv_net parameters are not among its parameters")


def shard_plan(n: int, world: int):
    """The cut of a gradient piece of `n` floats for the rank-ordered reduction over `world` ranks -> (shard,
    padded): rank r reduces floats [r*shard, (r+1)*shard) of the piece padded to padded = world*shard floats (the
    padding's sums are never copied back).
    `shard` is a multiple of 4, so every shard starts 16 bytes apart in the staging buffers and the fold takes its
    float4 path.  Depends on (n, world) only, so every rank cuts alike."""
    if n < 1 or world < 1:
        raise ValueError("shard_plan: n = %d and world = %d must be >= 1" % (n, world))
    shard = ((n + world - 1) // world + 3) // 4 * 4
    return shard, world * shard


class _RankOrderedReduce:
    """The deterministic mode's sum of the gradient over the ranks.  Each piece is cut by `shard_plan`; one
    ``all_to_all_single`` hands every rank its shard of every rank's piece as [world][shard], ``fcn_rank_fold`` sums
    them in rank order and one ``all_gather_into_tensor`` writes the summed shards back.  The collectives only copy,
    so the bits do not depend on the transport's algorithm.  Per rank the two copies move 2 (world-1)/world of the
    piece, as a ring all-reduce does.  The staging buffers are allocated once, for the larger piece."""

    def __init__(self, pieces, world, device):
        self.world = world
        plans = [shard_plan(n, world) for n in pieces]
        padded = max(p for _, p in plans)
        self.send = torch.zeros(padded, dtype=torch.float32, device=device)
        self.recv = torch.zeros(padded, dtype=torch.float32, device=device)
        self.out = torch.zeros(max(s for s, _ in plans), dtype=torch.float32, device=device)

    def __call__(self, piece):
        """Sum `piece` (contiguous float32) over the ranks in place, on the current stream."""
        import torch.distributed as dist
        n = piece.numel()
        shard, padded = shard_plan(n, self.world)
        send, recv, out = self.send[:padded], self.recv[:padded], self.out[:shard]
        send[:n].copy_(piece)
        dist.all_to_all_single(recv, send)
        _lib.call("fcn_rank_fold", _ptr(recv), shard, self.world, shard, _ptr(out), _stream())
        dist.all_gather_into_tensor(send, out)
        piece.copy_(send[:n])


class _BufferBroadcast:
    """Rank 0's BatchNorm buffers (running_mean, running_var, num_batches_tracked of every BN) to every rank in one
    broadcast of one packed byte buffer, on the current stream."""

    def __init__(self, model, device):
        bns = [m for m in model.modules()
               if isinstance(m, torch.nn.modules.batchnorm._BatchNorm) and m.track_running_stats]
        counters = [m.num_batches_tracked.view(-1) for m in bns]
        stats = [b for m in bns for b in (m.running_mean, m.running_var)]
        assert all(b.dtype == torch.float32 for b in stats) and all(c.dtype == torch.int64 for c in counters)
        nc, nf = 8 * len(counters), 4 * sum(b.numel() for b in stats)
        self.packed = torch.zeros(nc + nf, dtype=torch.uint8, device=device)
        views = list(self.packed[:nc].view(torch.int64).split([1] * len(counters))) + \
            list(self.packed[nc:].view(torch.float32).split([b.numel() for b in stats]))
        self.bufs, self.views = counters + stats, views

    def __call__(self):
        import torch.distributed as dist
        torch._foreach_copy_(self.views, self.bufs)
        dist.broadcast(self.packed, src=0)
        torch._foreach_copy_(self.bufs, self.views)


class _FlatOptimizer:
    """What FlatAdam and FlatSGD share, mixed in before their torch optimizer class: one parameter group over all of
    a model's parameters (FlatParams order) whose state lives in flat buffers of the bucket's layout, a
    `load_state_dict` that checks the loaded state before the subclass adopts it into those buffers, and a `step`
    that is ONE fused launch over the whole bucket.  A subclass supplies its flat buffers (`_flat_state`), the checks
    of the group settings (`_check_group`) and of the loaded per-parameter state (`_check_states`), `_adopt_loaded`
    and the launch (`_launch`)."""

    def __init__(self, model, flat, **hyper):
        super().__init__(list(model.parameters()), **hyper)
        self.model, self.flat = model, flat
        self.step_count = 0
        self.grad_scale = 1.0          # multiplies the gradient first: 1/world after a summing all-reduce
        self.register_load_state_dict_pre_hook(type(self)._check_loaded)
        self.register_load_state_dict_post_hook(type(self)._adopt_loaded)

    def _views(self):
        """-> (parameter, its view of each flat state buffer) for every parameter."""
        bufs = self._flat_state()
        for p in self.param_groups[0]["params"]:
            off, n = self.flat.offsets[id(p)], p.numel()
            yield (p,) + tuple(b[off: off + n].view(p.shape) for b in bufs)

    def _check_loaded(self, state_dict):
        """ValueError unless the loaded state has the one parameter group over all of the model's parameters that a
        fused step over the flat bucket takes, with settings and per-parameter state that step can continue."""
        groups = state_dict["param_groups"]
        if len(groups) != 1:
            raise ValueError("TrainStep.optimizer: the loaded state has %d parameter groups; the fused step takes "
                             "exactly one (all parameters of the model)" % len(groups))
        ids, params = groups[0]["params"], self.param_groups[0]["params"]
        if len(ids) != len(params):
            raise ValueError("TrainStep.optimizer: the loaded state has %d parameters, the model has %d"
                             % (len(ids), len(params)))
        self._check_group(groups[0])
        self._check_states(state_dict["state"], ids, params)

    @torch.no_grad()
    def step(self, closure=None):
        """One step of every parameter from the gradient in the flat bucket (``TrainStep.forward_backward`` leaves it
        there)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        g = self.param_groups[0]
        self._check_group(g)
        self.model.refresh()       # parameters change behind autograd's version counters: eval pack must rebuild
        self._launch(g)
        return loss


class FlatAdam(_FlatOptimizer, torch.optim.Adam):
    """``torch.optim.Adam`` over a model's parameters (one param group, FlatParams order) whose state is the flat
    bucket: each parameter's ``exp_avg`` / ``exp_avg_sq`` are views of two flat buffers and the step count is shared,
    so `state_dict` / `load_state_dict` speak torch's own format (the reference's checkpoints,
    train_net_det.py:345-361,384-398) while `step` is ONE ``fcn_adam_step`` launch over the whole bucket.  `step`
    reads lr, betas, eps and weight_decay from ``param_groups[0]`` on every call, where lr schedulers and the
    reference's MIN_LR clamp write.  The per-parameter ``state[p]["step"]`` tensors are brought up to date by
    `state_dict`; ``step_count`` is the live value."""

    def __init__(self, model, flat, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(model, flat, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        self.exp_avg = torch.zeros_like(flat.param)
        self.exp_avg_sq = torch.zeros_like(flat.param)
        self._bind()
        self.register_state_dict_pre_hook(FlatAdam._sync_steps)

    def _flat_state(self):
        return self.exp_avg, self.exp_avg_sq

    def _bind(self):
        for p, m, v in self._views():
            self.state[p] = {"step": torch.tensor(float(self.step_count)), "exp_avg": m, "exp_avg_sq": v}

    @staticmethod
    def _check_group(g):
        bad = [k for k in ("amsgrad", "maximize", "decoupled_weight_decay") if g.get(k)]
        if bad:
            raise ValueError("TrainStep.optimizer: %s is set; the fused step (fcn_adam_step) is plain Adam with L2 "
                             "weight decay" % " / ".join(bad))

    @staticmethod
    def _sync_steps(opt):
        for p in opt.param_groups[0]["params"]:
            opt.state[p]["step"] = torch.tensor(float(opt.step_count))

    def _check_states(self, states, ids, params):
        steps = set()
        for i, (k, p) in enumerate(zip(ids, params)):
            st = states.get(k)
            if not st:
                steps.add(0.0)
                continue
            for key in ("exp_avg", "exp_avg_sq"):
                if key not in st:
                    raise ValueError("TrainStep.optimizer: parameter %d: the loaded state has no %s (not an Adam "
                                     "state)" % (i, key))
                if tuple(st[key].shape) != tuple(p.shape):
                    raise ValueError("TrainStep.optimizer: parameter %d: loaded %s has shape %s, the parameter %s"
                                     % (i, key, tuple(st[key].shape), tuple(p.shape)))
            steps.add(float(st["step"]))
        if len(steps) > 1:
            raise ValueError("TrainStep.optimizer: the loaded per-parameter step counts differ (%s); the fused step "
                             "keeps one count for all parameters" % sorted(steps))

    @torch.no_grad()
    def _adopt_loaded(self):
        step = 0
        for p, m, v in self._views():
            st = self.state.get(p)
            if st:
                m.copy_(st["exp_avg"])
                v.copy_(st["exp_avg_sq"])
                step = int(float(st["step"]))
            else:
                m.zero_()
                v.zero_()
        self.step_count = step
        self._bind()

    def _launch(self, g):
        b1, b2 = g["betas"]
        self.step_count += 1
        f = self.flat
        _lib.call("fcn_adam_step", _ptr(f.param), _ptr(f.grad), _ptr(self.exp_avg), _ptr(self.exp_avg_sq), f.numel,
                  float(g["lr"]), float(b1), float(b2), float(g["eps"]), float(g["weight_decay"]), self.step_count,
                  float(self.grad_scale), _stream())


class FlatSGD(_FlatOptimizer, torch.optim.SGD):
    """``torch.optim.SGD`` over a model's parameters (one param group, FlatParams order) whose state is the flat
    bucket: each parameter's ``momentum_buffer`` is a view of one flat buffer, so `state_dict` / `load_state_dict`
    speak torch's own format while `step` is ONE ``fcn_sgd_step`` launch over the whole bucket.  `step` reads lr,
    momentum and weight_decay from ``param_groups[0]`` on every call.  torch creates a parameter's buffer on its first
    step with momentum; the fused step keeps one flag for the bucket (``has_buffers``), so the state is empty before
    that step and holds every parameter's buffer after it, as torch's does.  nesterov, dampening and maximize are
    rejected (the reference uses none of them).  ``step_count`` counts the steps this object took; torch's SGD state
    has no step count to restore it from."""

    def __init__(self, model, flat, lr=1e-3, momentum=0.0, weight_decay=0.0):
        super().__init__(model, flat, lr=lr, momentum=momentum, weight_decay=weight_decay)
        self.momentum_buffer = torch.zeros_like(flat.param)
        self.has_buffers = False

    def _flat_state(self):
        return (self.momentum_buffer,)

    def _bind(self):
        self.state.clear()
        if self.has_buffers:
            for p, b in self._views():
                self.state[p] = {"momentum_buffer": b}

    @staticmethod
    def _check_group(g):
        if "momentum" not in g:
            raise ValueError("TrainStep.optimizer: the parameter group has no momentum (not an SGD state)")
        bad = [k for k in ("nesterov", "maximize") if g.get(k)] + (["dampening"] if g.get("dampening", 0) else [])
        if bad:
            raise ValueError("TrainStep.optimizer: %s is set; the fused step (fcn_sgd_step) is plain SGD with momentum "
                             "and L2 weight decay" % " / ".join(bad))

    def _check_states(self, states, ids, params):
        with_buffer = 0
        for i, (k, p) in enumerate(zip(ids, params)):
            st = states.get(k) or {}
            other = sorted(set(st) - {"momentum_buffer"})
            if other:
                raise ValueError("TrainStep.optimizer: parameter %d: the loaded state has %s (not an SGD state)"
                                 % (i, " / ".join(other)))
            buf = st.get("momentum_buffer")      # torch < 2 wrote None when momentum was 0
            if buf is None:
                continue
            if tuple(buf.shape) != tuple(p.shape):
                raise ValueError("TrainStep.optimizer: parameter %d: loaded momentum_buffer has shape %s, the "
                                 "parameter %s" % (i, tuple(buf.shape), tuple(p.shape)))
            with_buffer += 1
        if 0 < with_buffer < len(params):
            raise ValueError("TrainStep.optimizer: the loaded state has momentum buffers on %d of %d parameters; the "
                             "fused step keeps buffers for all parameters or none" % (with_buffer, len(params)))

    @torch.no_grad()
    def _adopt_loaded(self):
        loaded = [self.state.get(p, {}).get("momentum_buffer") for p in self.param_groups[0]["params"]]
        self.has_buffers = loaded[0] is not None       # _check_loaded admits buffers on all parameters or on none
        if self.has_buffers:
            # each source onto its own view: a source may BE that view (torch keeps a loaded tensor that already has
            # the parameter's dtype and device, as in opt.load_state_dict(opt.state_dict())), so nothing is zeroed first
            for (p, b), src in zip(self._views(), loaded):
                b.copy_(src)
        else:
            self.momentum_buffer.zero_()
        self._bind()

    def _launch(self, g):
        momentum = float(g["momentum"])
        first = not self.has_buffers
        f = self.flat
        _lib.call("fcn_sgd_step", _ptr(f.param), _ptr(f.grad), _ptr(self.momentum_buffer), f.numel, float(g["lr"]),
                  momentum, float(g["weight_decay"]), int(first), float(self.grad_scale), _stream())
        self.step_count += 1
        if momentum != 0 and first:
            self.has_buffers = True
            self._bind()


class TrainStep:
    """One optimizer step of PointNetDet on the hand-written kernels: forward -> fused losses and d/dlogits
    (``fcn_det_loss``) -> backward kernels -> ONE all-reduce of the flat gradient bucket (when torch.distributed is
    initialised and world > 1) -> fused Adam or SGD.  Mirrors train/train_net_det.py:121-134 (zero_grad / backward /
    step and the TrainingStates update).  ``optimizer`` ("adam" or "sgd", the values of cfg.TRAIN.OPTIMIZER,
    train_net_det.py:321-328) selects a torch.optim.Adam (FlatAdam) or torch.optim.SGD (FlatSGD, with ``momentum``)
    for lr schedulers and checkpoints; ``states`` (validate.TrainStates) collects every step's losses and metrics on
    the device.  ``deterministic`` (settable): True runs the step bit-reproducibly (deterministic layer kernels and
    fused loss; one build, same inputs and hyper-parameters; with world > 1 a rank-ordered gradient sum and rank 0's
    BN buffers on every rank, so every rank holds the same model), False the default kernels, None follows
    ``torch.use_deterministic_algorithms`` at every step."""

    def __init__(self, model, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, comm_stream=None,
                 states_capacity=None, optimizer="adam", momentum=0.0, deterministic=None):
        from .validate import TrainStates
        if optimizer not in ("adam", "sgd"):
            raise ValueError("TrainStep: optimizer %r is not supported; the fused steps are 'adam' and 'sgd'"
                             % (optimizer,))
        self.model = model
        self.engines: Dict[tuple, TrainEngine] = {}
        self.flat = FlatParams.of(model)
        if optimizer == "adam":
            self.optimizer = FlatAdam(model, self.flat, lr, betas, eps, weight_decay)
        else:
            self.optimizer = FlatSGD(model, self.flat, lr, momentum, weight_decay)
        self.states = TrainStates(self.flat.param.device, states_capacity, deterministic=self._deterministic_now)
        self._comm = None
        self._split = 0
        self._ordered = None           # _RankOrderedReduce and _BufferBroadcast, built on the first such step
        self._bn_bcast = None
        self._fused_losses = {}        # train_path.FusedLoss per (deterministic, B, T2)
        self.deterministic = deterministic

    @property
    def loss_impl(self):
        """How the losses and d/dlogits are computed: "kernel", the fused kernels of csrc/loss.cu."""
        return "kernel"

    @property
    def lr(self):
        return self.optimizer.param_groups[0]["lr"]

    @lr.setter
    def lr(self, value):
        self.optimizer.param_groups[0]["lr"] = value

    def _adam(self, name):
        if not isinstance(self.optimizer, FlatAdam):
            raise AttributeError("TrainStep.%s exists for Adam only; this TrainStep steps with SGD" % name)
        return self.optimizer

    @property
    def m(self):
        return self._adam("m").exp_avg

    @property
    def v(self):
        return self._adam("v").exp_avg_sq

    @property
    def betas(self):
        return self._adam("betas").param_groups[0]["betas"]

    @property
    def eps(self):
        return self._adam("eps").param_groups[0]["eps"]

    @property
    def wd(self):
        return self.optimizer.param_groups[0]["weight_decay"]

    @property
    def step_count(self):
        return self.optimizer.step_count

    def _deterministic_now(self) -> bool:
        from .train_path import deterministic_mode
        return deterministic_mode(self.deterministic)

    def engine(self, B, N, T, deterministic=False) -> TrainEngine:
        key = (int(B), int(N), tuple(int(t) for t in T), bool(deterministic))
        e = self.engines.get(key)
        if e is None:
            e = self.engines[key] = TrainEngine(self.model, *key[:3], deterministic=key[3])
        return e

    def _fused_loss(self, eng):
        from .train_path import FusedLoss
        key = (eng.deterministic, eng.B, eng.T2)
        fl = self._fused_losses.get(key)
        if fl is None:
            fl = self._fused_losses[key] = FusedLoss(self.model, eng.B, eng.T2, eng.act["reg_out"]["cols"], eng.dev,
                                                     eng.deterministic)
        return fl

    def _losses(self, eng, cls, reg, center_ref2, data):
        """-> (losses, metrics, dcls, dreg)."""
        return self._fused_loss(eng).run(cls, reg, center_ref2, data)

    def _forward_losses(self, data):
        """This step's engine (shape and mode), a zeroed gradient bucket, the forward and the losses -> (engine,
        losses, metrics, dcls, dreg)."""
        from .train_path import deterministic_mode
        S = self.model.ARCH.num_scales
        pc = data["point_cloud"][:, :3, :].contiguous()
        centers = [data["center_ref%d" % (i + 1)].contiguous() for i in range(S)]
        eng = self.engine(pc.shape[0], pc.shape[2], [c.shape[2] for c in centers],
                          deterministic_mode(self.deterministic))
        self.flat.grad.zero_()
        cls, reg = eng.forward(pc, centers, data.get("one_hot"))
        return (eng,) + self._losses(eng, cls, reg, centers[1], data)

    def forward_backward(self, data, update_running=True):
        """-> (losses, metrics); gradients (this rank's) are left in the flat bucket."""
        eng, losses, metrics, dcls, dreg = self._forward_losses(data)
        eng.backward(dcls, dreg, update_running=update_running)
        self.flat.expose_grads(self.model)
        return losses, metrics

    def step(self, data):
        """forward + losses + backward + gradient all-reduce + Adam or SGD.  With world > 1 the flat bucket is reduced in
        TWO pieces on a communication stream: the FCN + heads part (92 % of the parameters, complete after the
        first ~15 % of the backward) overlaps the PointNet backward; the PointNet part follows.  In deterministic mode
        each piece is summed in rank order (`_RankOrderedReduce`) and rank 0's BN buffers are then broadcast on the
        same stream, so every rank ends the step with the same parameters, optimizer state and buffers."""
        import torch.distributed as dist
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        eng, losses, metrics, dcls, dreg = self._forward_losses(data)
        self.states.append(self._fused_loss(eng).out, eng.B)     # fcn_det_loss's 16-float result block as it stands
        if world > 1:
            if self._comm is None:
                self._comm = torch.cuda.Stream(device=self.flat.grad.device)
                self._split = piece_split(self.model)       # [0, split): feat_net, [split, n): conv_net + heads
            if eng.deterministic and (self._ordered is None or self._ordered.world != world):
                dev = self.flat.grad.device
                self._ordered = _RankOrderedReduce((self._split, self.flat.numel - self._split), world, dev)
                self._bn_bcast = _BufferBroadcast(self.model, dev)
            reduce = self._ordered if eng.deterministic else dist.all_reduce
            cur = torch.cuda.current_stream()
            eng.backward(dcls, dreg, stage="fcn")
            ev = torch.cuda.Event()
            ev.record(cur)
            self._comm.wait_event(ev)
            with torch.cuda.stream(self._comm):
                reduce(self.flat.grad[self._split:])
            eng.backward(None, None, stage="pointnet")
            ev2 = torch.cuda.Event()
            ev2.record(cur)
            self._comm.wait_event(ev2)
            with torch.cuda.stream(self._comm):
                reduce(self.flat.grad[: self._split])
                if eng.deterministic:
                    self._bn_bcast()
            cur.wait_stream(self._comm)
        else:
            eng.backward(dcls, dreg)
        self.optimizer.grad_scale = 1.0 / world
        self.optimizer.step()
        return losses, metrics
