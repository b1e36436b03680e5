"""ORACLE: the reference's depth-to-cloud conversion (sunrgbd/read_3d_points.py, a port of the SUNRGBD toolbox's
read3dPoints.m) restated in numpy with every operation's order and precision explicit, independent of the BLAS that
numpy links:

    valid = raw != 0 (row-major)        r = (raw >> 3) | (raw << 13) in uint16
    d = float32(r) / 1000 in float32, then d[d > 8] = 8
    x3 = ((u - cx) * d) / fx, y3 = ((v - cy) * d) / fy in float64 (u, v: 0-based column and row)
    point (x3, d, -y3) times Rtilt in float64 as np.matmul(Rtilt, points.T) sums it, rounded to float32 once
    colour float32(rgb) / 255 in float32

The port's `depth[depthpath > 8] = 8` compares the path string (a TypeError in Python 3); the line meant, and what the
MATLAB original does, is the clamp above.

np.matmul of (3, 3) by (3, n) goes to OpenBLAS's dgemm for n >= 2: each row is a0 b0 rounded, then one FMA per
further term (dot_fma of csrc/input_builder.cuh).  For n = 1 it goes to dgemv, which rounds a1 b1 first, then adds
term 0 and term 2 by FMA.  Both orders are restated with an exactly rounded FMA emulated in float64 (`fma`)."""
from __future__ import annotations

import numpy as np


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _two_prod(a, b):
    """a * b = p + e exactly (Veltkamp's split; no overflow or underflow in this use)."""
    p = a * b
    sa = 134217729.0 * a
    ah = sa - (sa - a)
    al = a - ah
    sb = 134217729.0 * b
    bh = sb - (sb - b)
    bl = b - bh
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _add_odd(a, b):
    """a + b rounded to odd: the rounded-to-nearest sum, moved to its odd neighbour towards the exact sum when it is
    inexact and even."""
    s, e = _two_sum(a, b)
    even = (s.view(np.int64) & 1) == 0
    return np.where((e != 0) & even, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)


def fma(a, b, c):
    """a * b + c rounded once (float64 arrays): Boldo and Melquiond's emulation, RN(th + RO(tl + ul)) with
    a * b = uh + ul and c + uh = th + tl exactly.  An exact zero takes the sign a hardware FMA gives it, which the
    plain a * b + c has then too."""
    a, b, c = (np.asarray(x, np.float64) for x in (a, b, c))
    uh, ul = _two_prod(a, b)
    th, tl = _two_sum(c, uh)
    z = th + _add_odd(tl, ul)
    return np.where(z == 0, a * b + c, z)


def rtilt_rows(R, p):
    """np.matmul(R, p.T).T for p (n, 3) float64, in the order OpenBLAS sums it (see the module note)."""
    R = np.asarray(R, np.float64)
    out = np.empty_like(p)
    for k in range(3):
        if len(p) == 1:
            out[:, k] = fma(R[k, 2], p[:, 2], fma(R[k, 0], p[:, 0], R[k, 1] * p[:, 1]))
        else:
            out[:, k] = fma(R[k, 2], p[:, 2], fma(R[k, 1], p[:, 1], R[k, 0] * p[:, 0]))
    return out


def depth_cloud(depth, rgb, Rtilt, K):
    """depth (h, w) uint16, rgb (h, w, 3) uint8 in RGB order or None, Rtilt and K (3, 3) -> float32 (n, 6): x, y, z,
    r, g, b of the valid pixels in row-major order (colour 0 when rgb is None)."""
    raw = np.asarray(depth, np.uint16)
    h, w = raw.shape
    valid = (raw != 0).ravel()
    r = (raw >> np.uint16(3)) | (raw << np.uint16(13))
    d = r.astype(np.float32) / np.float32(1000)
    d[d > np.float32(8)] = np.float32(8)
    K = np.asarray(K, np.float64)
    cx, cy, fx, fy = K[0, 2], K[1, 2], K[0, 0], K[1, 1]
    v, u = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    z = d.astype(np.float64)
    x3 = ((u - cx) * z) / fx
    y3 = ((v - cy) * z) / fy
    p = np.stack([x3.ravel(), z.ravel(), -y3.ravel()], 1)[valid]
    out = np.zeros((len(p), 6), np.float32)
    out[:, :3] = rtilt_rows(Rtilt, p).astype(np.float32)
    if rgb is not None:
        out[:, 3:] = np.asarray(rgb, np.uint8).astype(np.float32).reshape(-1, 3)[valid] / np.float32(255)
    return out


def frame_cloud(depth, rgb, image_hw, calib, H, W, P):
    """The device entry's frame (C ABI section (24)): the top-left min(h, H) x min(w, W) crop of depth (H, W) (and of
    rgb), calib (18,) = Rtilt, K; -> (cloud (min(n, P), 6), n, status bits)."""
    h, w = (int(x) for x in image_hw)
    hc, wc = min(max(h, 0), H), min(max(w, 0), W)
    calib = np.asarray(calib, np.float64)
    cloud = depth_cloud(depth[:hc, :wc], None if rgb is None else rgb[:hc, :wc], calib[:9].reshape(3, 3),
                        calib[9:].reshape(3, 3))
    bits = (1 if len(cloud) > P else 0) | (128 if h > H or w > W else 0)
    return cloud[:P], len(cloud), bits
