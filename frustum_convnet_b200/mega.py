"""Host-side tables of the persistent FCN kernel (csrc/fcn_mega.cu, C entry ``fcn_mega_forward``).

Turns the engine's per-layer GEMM descriptions (``_ConvLayer`` + the plan's buffers) into
  * one tensor map per distinct (source map, conv stride),
  * a layer table (``fcn_mega_layer``),
  * a job table (``fcn_mega_job``): one [128 rows x NT columns] output tile each (NT = 256 | 128 | 64), in TOPOLOGICAL order, with the
    completion counters of the producer tiles it reads.
The order interleaves the side transposed convs with the next block's first layer, so CTAs that would wait on
a dependency find independent work first.  Replaces the launch sequence of ConvFeatNet.forward + heads + decode
(/root/reference/models/det_base.py:196-224,367-411) with one call.

Pure index arithmetic: ``build_tables`` runs (and is tested) without a GPU.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence

from . import _lib

ROWS = 128
EPI_WARPS = 1          # completion counts per finished tile (the store warp publishes each tile once)


class LayerDesc:
    """Shape-level description of one GEMM layer (no pointers): what ``build_tables`` needs."""

    def __init__(self, name, kind, segs, K_pad, n_cols, Cout, up, relu, out, c_off, NT, round_out,
                 P_m, T_out, n_rows, ld_out, P_store, T_store):
        self.name, self.kind, self.segs, self.K_pad, self.n_cols = name, kind, segs, K_pad, n_cols
        self.Cout, self.up, self.relu, self.out, self.c_off = Cout, up, relu, out, c_off
        self.NT, self.round_out = NT, round_out
        self.P_m, self.T_out, self.n_rows = P_m, T_out, n_rows
        self.ld_out, self.P_store, self.T_store = ld_out, P_store, T_store
        self.m_tiles = (n_rows + ROWS - 1) // ROWS
        self.n_tiles = n_cols // NT
        self.k_atoms = 1 if NT == 256 else 2       # 32-wide K atoms per stage of the packed weight image


def chain_tiles(layers: Sequence[LayerDesc]) -> int:
    """Fewest output tiles of a main-chain layer (the conv and merge layers)."""
    return min(L.m_tiles * L.n_tiles for L in layers if L.kind in ("conv", "merge"))


def job_order(layers: Sequence[LayerDesc]) -> List[int]:
    """Layer order of the job table: main chain in network order; every side transposed conv right after the
    layer it reads.  (eng.layers lists the deconvs after all blocks; moving them up keeps the order topological -
    a deconv only reads its own block's merge output - and lets them overlap the next block.)"""
    order = []
    for i, L in enumerate(layers):
        if L.kind in ("conv", "merge"):
            order.append(i)
            order += [j for j, D in enumerate(layers) if D.kind == "deconv" and D.segs[0][0] == L.out]
    order += [i for i, L in enumerate(layers) if L.kind == "heads"]
    assert sorted(order) == list(range(len(layers)))
    return order


def build_tables(layers: Sequence[LayerDesc], interleave: bool = True):
    """-> (map_keys, layer_rows, jobs, nflags).  map_keys: tensor maps in index order - ("load", buffer, stride) for
    the A-operand boxes and ("store", buffer, up) for the epilogue stores; layer_rows: dict per layer with map
    indices / flag bases; jobs: list of dicts {layer, m, n, deps: [(first_flag, count, target)]} in execution order."""
    producers: Dict[str, List[int]] = {}
    for i, L in enumerate(layers):
        producers.setdefault(L.out, []).append(i)
    map_keys, map_idx = [], {}
    flag_base, nflags = [], 0
    for L in layers:
        flag_base.append(nflags)
        nflags += L.m_tiles
    rows = []
    for i, L in enumerate(layers):
        segs = []
        for (src, c, tap, st) in L.segs:
            key = ("load", src, st)
            if key not in map_idx:
                map_idx[key] = len(map_keys)
                map_keys.append(key)
            segs.append(dict(map_idx=map_idx[key], kblocks=(c + 31) // 32, tap=tap, stride=st))
        okey = ("store", L.out, L.up)
        if L.kind != "heads" and okey not in map_idx:
            map_idx[okey] = len(map_keys)
            map_keys.append(okey)
        rows.append(dict(segs=segs, flag_base=flag_base[i], out_map=map_idx.get(okey, 0)))

    def deps_of(li, m):
        L = layers[li]
        r0, r1 = m * ROWS, min(m * ROWS + ROWS, L.n_rows) - 1
        want = {}                                        # producer layer -> (lo tile, hi tile)
        for (src, c, tap, st) in L.segs:
            for pi in producers.get(src, ()):
                Pr = layers[pi]
                lo_row, hi_row = r0 * st + tap, r1 * st + tap          # flat rows of the source map
                lo = max(0, lo_row // Pr.up // ROWS)
                hi = min(Pr.m_tiles - 1, hi_row // Pr.up // ROWS)
                if hi < lo:
                    continue
                a, b = want.get(pi, (lo, hi))
                want[pi] = (min(a, lo), max(b, hi))
        out = [(flag_base[pi] + lo, hi - lo + 1, EPI_WARPS * layers[pi].n_tiles) for pi, (lo, hi) in sorted(want.items())]
        assert len(out) <= _lib.MEGA_MAX_DEPS, "layer %s reads more than %d producers" % (L.name, _lib.MEGA_MAX_DEPS)
        return out

    order = job_order(layers)
    jobs = []

    def emit(li):
        L = layers[li]
        return [dict(layer=li, m=m, n=n, deps=deps_of(li, m)) for m in range(L.m_tiles) for n in range(L.n_tiles)]

    k = 0
    while k < len(order):
        li = order[k]
        if interleave and layers[li].kind == "deconv" and k + 1 < len(order) and layers[order[k + 1]].kind != "heads":
            # deconv of block i  x  first conv of block i+1: both only read merge_i -> interleave their tiles
            a, b = emit(li), emit(order[k + 1])
            na, nb = len(a), len(b)
            ia = ib = 0
            while ia < na or ib < nb:      # proportional merge keeps each list's internal order
                if ib >= nb or (ia < na and ia * nb <= ib * na):
                    jobs.append(a[ia]); ia += 1
                else:
                    jobs.append(b[ib]); ib += 1
            k += 2
        else:
            jobs.extend(emit(li))
            k += 1
    # topological check: every dependency counter belongs to a layer whose tiles all appear earlier
    done = set()
    pos = {}
    for j, jb in enumerate(jobs):
        pos.setdefault((jb["layer"], jb["m"]), []).append(j)
    flag_owner = {}
    for i, L in enumerate(layers):
        for m in range(L.m_tiles):
            flag_owner[flag_base[i] + m] = (i, m)
    for j, jb in enumerate(jobs):
        for first, cnt, target in jb["deps"]:
            for f in range(first, first + cnt):
                assert max(pos[flag_owner[f]]) < j, "job table is not topologically ordered"
    return map_keys, rows, jobs, nflags


def to_ctypes(layers: Sequence[LayerDesc], rows, jobs, ptrs):
    """ptrs[i] = (w_tc, bias, out) device pointers of layer i -> (ctypes layer array, ctypes job array)."""
    LA = (_lib.MegaLayer * len(layers))()
    for i, (L, row) in enumerate(zip(layers, rows)):
        a = LA[i]
        a.n_seg = len(row["segs"])
        for j, sg in enumerate(row["segs"]):
            a.seg[j].map_idx, a.seg[j].kblocks, a.seg[j].tap, a.seg[j].stride = (sg["map_idx"], sg["kblocks"],
                                                                                  sg["tap"], sg["stride"])
        a.n_stage, a.NT, a.n_tiles_n, a.k_atoms = L.K_pad // (32 * L.k_atoms), L.NT, L.n_tiles, L.k_atoms
        a.relu, a.round_out, a.up, a.Cout = L.relu, L.round_out, L.up, L.Cout
        a.P_m, a.T_out, a.n_rows = L.P_m, L.T_out, L.n_rows
        a.ld_out, a.P_store, a.T_store, a.c_off = L.ld_out, L.P_store, L.T_store, L.c_off
        a.is_heads, a.flag_base, a.out_map = int(L.kind == "heads"), row["flag_base"], row["out_map"]
        a.w_tc, a.bias, a.out = ptrs[i]
    JA = (_lib.MegaJob * max(len(jobs), 1))()
    for j, jb in enumerate(jobs):
        a = JA[j]
        a.layer, a.m_tile, a.n_tile, a.n_dep = jb["layer"], jb["m"], jb["n"], len(jb["deps"])
        for d, (first, cnt, target) in enumerate(jb["deps"]):
            a.dep[d].first, a.dep[d].count, a.dep[d].target = first, cnt, target
    return LA, JA
