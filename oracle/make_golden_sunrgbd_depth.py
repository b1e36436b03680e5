"""Writes tests/golden/sunrgbd_depth.npz: what the reference's own, unmodified read_3d_points
(sunrgbd/read_3d_points.py) returns for hand-built depth and RGB images.  Needs the reference tree
(oracle/ref_import.REF); the tests read only the fixture.

    python -m oracle.make_golden_sunrgbd_depth

Two stand-ins make the port run here: `skimage` (not installed) is a module whose io.imread(x) returns x.image, and
the depth "path" is an object whose `> 8` gives the decoded-depth mask, which is what the port's
`depth[depthpath > 8] = 8` means (it compares the path string, a TypeError in Python 3).  Cases, each under two
calibrations with a tilted Rtilt, fx != fy and fractional cx, cy:
  edges     7 x 11: raw 0, raw with low bits 1..7 (which rotate past 8 m), r = 8000 and 8001, raw 65535 and random
            depths under a random valid mask;
  random    23 x 31: random depths under a random valid mask;
  single    1 x 1;
  invalid   4 x 5, every pixel 0.
Asserted: oracle/sunrgbd_depth.py equals every result rounded to float32, bit for bit."""
from __future__ import annotations

import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import sunrgbd_depth as osd  # noqa: E402
from oracle.ref_import import REF  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "sunrgbd_depth.npz")
SEED = 11


def rot_left3(r):
    """The raw value that decodes (rotate right by 3) to r."""
    r = np.asarray(r, np.uint32)
    return (((r << 3) | (r >> 13)) & 0xFFFF).astype(np.uint16)


def calibs():
    def rot(axis, t):
        c, s = np.cos(t), np.sin(t)
        m = np.eye(3)
        i, j = [k for k in range(3) if k != axis]
        m[i, i], m[i, j], m[j, i], m[j, j] = c, -s, s, c
        return m
    R0 = rot(0, 0.137) @ rot(1, -0.061)
    K0 = np.array([[529.5, 0.0, 365.3125], [0.0, 527.25, 265.75], [0.0, 0.0, 1.0]])
    R1 = rot(0, -0.212) @ rot(1, 0.093) @ rot(2, 0.018)
    K1 = np.array([[518.857901, 0.0, 284.582449], [0.0, 519.469611, 208.736166], [0.0, 0.0, 1.0]])
    return [(R0, K0), (R1, K1)]


def cases(rng):
    out = {}
    e = rng.integers(500, 7500, size=(7, 11))
    raw = rot_left3(e)
    raw[rng.random((7, 11)) < 0.3] = 0
    raw[0, :7] = np.arange(1, 8)                         # low bits 1..7 set: r = raw << 13, past 8 m
    raw[1, 0], raw[1, 1], raw[1, 2], raw[1, 3] = rot_left3(8000), rot_left3(8001), 65535, 0
    raw[6, 10] = rot_left3(1)
    out["edges"] = raw
    raw = rot_left3(rng.integers(300, 9000, size=(23, 31)))
    raw[rng.random((23, 31)) < 0.45] = 0
    out["random"] = raw
    out["single"] = rot_left3([[2345]])
    out["invalid"] = np.zeros((4, 5), np.uint16)
    return out


class _Image:
    def __init__(self, image):
        self.image = image


class _DepthPath(_Image):
    def __gt__(self, x):
        r = (self.image >> np.uint16(3)) | (self.image << np.uint16(13))
        return r.astype(np.float32) / 1000 > x


def reference_read_3d_points():
    io = types.ModuleType("skimage.io")
    io.imread = lambda x: x.image
    sk = types.ModuleType("skimage")
    sk.io = io
    sys.modules["skimage"], sys.modules["skimage.io"] = sk, io
    spec = importlib.util.spec_from_file_location("ref_read_3d_points", os.path.join(REF, "sunrgbd",
                                                                                     "read_3d_points.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.read_3d_points


def main():
    rng = np.random.default_rng(SEED)
    read = reference_read_3d_points()
    z, names = {}, []
    for name, raw in cases(rng).items():
        rgb = rng.integers(0, 256, size=raw.shape + (3,), dtype=np.uint8)
        rgb[0, 0], rgb[-1, -1] = (0, 128, 255), (255, 1, 254)
        for c, (R, K) in enumerate(calibs()):
            key = "%s_%d" % (name, c)
            ref = read(_Image(rgb), _DepthPath(raw), R, K)
            assert ref.dtype == np.float64 and ref.shape == (int((raw != 0).sum()), 6), (key, ref.dtype, ref.shape)
            mine = osd.depth_cloud(raw, rgb, R, K)
            assert np.array_equal(mine.view(np.uint32), ref.astype(np.float32).view(np.uint32)), key
            z["depth_" + key], z["rgb_" + key] = raw, rgb
            z["calib_" + key] = np.concatenate([R.reshape(-1), K.reshape(-1)])
            z["ref_" + key] = ref
            names.append(key)
    z["cases"] = np.array(names)
    np.savez_compressed(OUT, **z)
    print("wrote", OUT, names)


if __name__ == "__main__":
    main()
