"""Restatement of fcn_group_rows (include/frustum_b200.h section 2) on the CPU, for bit-exact tests.

Built on ``oracle.qdp.qdp_c`` (pinned to the reference's own grouping kernel) plus the gather and centre
subtraction of models/det_base.py:75-80.  For one frustum b and scale s with T sections of K slots:

  cnt[t]        = min(hits, K), hits = #{k : fabsf(fp32(zc[t] - z[k])) < dis_z};
  unique_rows=1 : the sections end to end, cnt[t] rows each (empty sections contribute nothing);
  unique_rows=0 : exactly T*K rows in (t, l) order; slot l >= cnt repeats the first hit, an empty section
                  gathers point 0;
  record        : {x - cx, y - cy, z - cz} as IEEE fp32 round-to-nearest subtractions, then the section index t
                  as int bits, with the sign bit set when the section is empty;
  tiles         : {(b, i*tile_rows, min(tile_rows, total_b - i*tile_rows))} for i < ceil(total_b / tile_rows);
  feature map   : rows [0, T) of the frustum's block zero, the one-hot values in columns [c3, c3 + num_vec),
                  every other element unchanged.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np

SIGN = np.int32(-0x80000000)


@dataclass
class ScaleRef:
    cnt: np.ndarray               # (B, T) int32
    idx: np.ndarray               # (B, T, K) int64, the reference's idx tensor (back-fill included)
    rows: List[np.ndarray]        # per frustum: (n_b, 4) float32 records, column 3 holds the tag bits
    tiles: List[tuple]            # (b, row0, nrows), frustum-major, row0 ascending

    def total(self, b):
        return self.rows[b].shape[0]


def records(pc: np.ndarray, cen: np.ndarray, b: int, k: np.ndarray, t: np.ndarray, empty: np.ndarray) -> np.ndarray:
    """(n, 4) float32 records of point indices k in sections t of frustum b (numpy fp32 arithmetic: IEEE round to
    nearest, one rounding per subtraction)."""
    pc = np.asarray(pc, dtype=np.float32)
    cen = np.asarray(cen, dtype=np.float32)
    out = np.empty((k.shape[0], 4), dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for c in range(3):
            out[:, c] = pc[b, c, k] - cen[b, c, t]
    tag = t.astype(np.int32) | np.where(empty, SIGN, np.int32(0)).astype(np.int32)
    out.view(np.int32)[:, 3] = tag
    return out


def records_f64(pc, cen, b, k, t):
    """The same coordinates computed in float64 and then rounded to fp32.  Rounding twice is harmless for one
    subtraction of fp32 operands because 53 >= 2*24 + 2, so this equals the fp32 subtraction (tests assert it)."""
    pc = np.asarray(pc, dtype=np.float64)
    cen = np.asarray(cen, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return np.stack([(pc[b, c, k] - cen[b, c, t]).astype(np.float32) for c in range(3)], 1)


def group_scale(pc, cen, dis_z: float, K: int, unique_rows: int, tile_rows: int, qdp=None) -> ScaleRef:
    """One scale of fcn_group_rows.  pc (B,3,N), cen (B,3,T) float32.  `qdp` replaces the query (default
    oracle.qdp.qdp_c), e.g. with oracle.qdp.qdp_loops for cross-checks."""
    from oracle import qdp as Q
    pc = np.ascontiguousarray(pc, dtype=np.float32)
    cen = np.ascontiguousarray(cen, dtype=np.float32)
    idx, cnt = (qdp or Q.qdp_c)(pc, cen, np.float32(dis_z), K)
    B, T = cnt.shape
    rows, tiles = [], []
    for b in range(B):
        c = cnt[b].astype(np.int64)
        if unique_rows:
            t = np.repeat(np.arange(T), c)
            l = np.arange(t.shape[0]) - np.repeat(np.cumsum(c) - c, c)
        else:
            t = np.repeat(np.arange(T), K)
            l = np.tile(np.arange(K), T)
        k = idx[b, t, l]
        rows.append(records(pc, cen, b, k, t, c[t] == 0))
        n = rows[-1].shape[0]
        tiles += [(b, r0, min(tile_rows, n - r0)) for r0 in range(0, n, tile_rows)]
    return ScaleRef(cnt, idx, rows, tiles)


def feat_ref(feat_init: np.ndarray, T: int, c3: int, one_hot: Optional[np.ndarray], num_vec: int) -> np.ndarray:
    """Expected feature map of one scale: feat_init (B, feat_pitch, ld_feat) with rows [0, T) zeroed and the
    one-hot values written (when one_hot is given and num_vec > 0)."""
    f = np.array(feat_init, dtype=np.float32, copy=True)
    f[:, :T, :] = 0.0
    if one_hot is not None and num_vec > 0:
        f[:, :T, c3:c3 + num_vec] = np.asarray(one_hot, dtype=np.float32)[:, None, :num_vec]
    return f


def rounding_edges(zc, dis_z, steps: int = 64) -> List[np.float32]:
    """fp32 depths z near zc - dis_z and zc + dis_z whose exact distance |zc - z| is below dis_z while the fp32
    difference rounds up onto dis_z: the kernels' strict `<` on the rounded difference rejects them, an exact
    comparison would accept them.  Found where z has a finer ulp than the distance, i.e. |z| < dis_z / 2."""
    zc, D = np.float32(zc), np.float32(dis_z)
    out = set()
    for target in (float(zc) - float(D), float(zc) + float(D)):
        for direction in (-np.inf, np.inf):
            z = np.float32(target)
            for _ in range(steps):
                if abs(float(zc) - float(z)) < float(D) and abs(np.float32(zc - z)) >= D:
                    out.add(z)
                z = np.nextafter(z, np.float32(direction))
    return sorted(out)


# ------------------------------------------------------------------ the bit-matrix / section-scan rule
SMEM_LIMIT = 200 * 1024


def bitmask_bytes(N: int, Ts, Ks) -> int:
    """Shared memory of the single-launch bit-matrix kernel: the largest scale's T x ceil(N/32) bit matrix plus
    3T words (centres, counts, offsets) plus T*K parked point indices."""
    return max(4 * (T * ((N + 31) // 32) + 3 * T + T * K) for T, K in zip(Ts, Ks))


def uses_bitmask(N: int, Ts, Ks, force_scan: int = 0) -> bool:
    return not force_scan and bitmask_bytes(N, Ts, Ks) <= SMEM_LIMIT


# ------------------------------------------------------------------ bit comparisons
def same_bits(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Element-wise bit equality of two float32 arrays, any NaN equal to any NaN (the device returns the
    canonical NaN where x86 propagates a payload)."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    return (a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))


def record_bits_equal(got: np.ndarray, exp: np.ndarray) -> np.ndarray:
    """Per-row equality of (n, 4) records: coordinates by same_bits, the tag by its int bits."""
    ok = same_bits(got[:, :3], exp[:, :3]).all(1)
    return ok & (np.ascontiguousarray(got).view(np.int32)[:, 3] == np.ascontiguousarray(exp).view(np.int32)[:, 3])
