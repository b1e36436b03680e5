"""CPU: the SUN-RGBD depth-cloud conversion (C ABI section (24)) without a GPU: the numpy oracle against the
reference's own read_3d_points (tests/golden/sunrgbd_depth.npz), its emulated FMA against exact arithmetic, the
entry's argument checks and the ptxas usage of its kernels."""
import ctypes as C
import os
from fractions import Fraction

import numpy as np
import pytest

from conftest import ROOT
from toolchain import compile_cuda

GOLDEN = os.path.join(ROOT, "tests", "golden", "sunrgbd_depth.npz")


def _golden():
    z = np.load(GOLDEN)
    return z, [str(c) for c in z["cases"]]


def _decode(raw):
    return ((raw.astype(np.uint32) >> 3) | (raw.astype(np.uint32) << 13)) & 0xFFFF


def test_oracle_equals_the_reference_bit_for_bit():
    from oracle import sunrgbd_depth as osd
    z, cases = _golden()
    for c in cases:
        cal = z["calib_" + c]
        ref = z["ref_" + c]
        got = osd.depth_cloud(z["depth_" + c], z["rgb_" + c], cal[:9].reshape(3, 3), cal[9:].reshape(3, 3))
        assert got.dtype == np.float32 and got.shape == ref.shape, c
        assert np.array_equal(got.view(np.uint32), ref.astype(np.float32).view(np.uint32)), c
        nocolour = osd.depth_cloud(z["depth_" + c], None, cal[:9].reshape(3, 3), cal[9:].reshape(3, 3))
        assert np.array_equal(nocolour[:, :3].view(np.uint32), got[:, :3].view(np.uint32)) and not nocolour[:, 3:].any()


def test_the_fixture_covers_every_rule():
    z, cases = _golden()
    raws = {c: z["depth_" + c] for c in cases}
    allraw = np.concatenate([r.ravel() for r in raws.values()])
    r = _decode(allraw)
    assert (allraw == 0).any() and (allraw == 65535).any()
    assert np.isin(np.arange(1, 8), allraw).all()                   # low bits only: rotate to >= 8.192 m
    assert (r == 8000).any() and (r == 8001).any()
    assert ((r > 0) & (r < 8000)).sum() > 100
    shapes = {raws[c].shape for c in cases}
    assert (1, 1) in shapes and any(h != w for h, w in shapes)
    assert any(not raws[c].any() for c in cases) and any(raws[c].shape == (1, 1) and raws[c].all() for c in cases)
    assert any(0 < (raws[c] != 0).mean() < 1 for c in cases)
    calibs = {z["calib_" + c].tobytes() for c in cases}
    assert len(calibs) == 2
    for cal in map(lambda b: np.frombuffer(b), calibs):
        R, K = cal[:9].reshape(3, 3), cal[9:].reshape(3, 3)
        assert not np.allclose(R, np.eye(3)) and K[0, 0] != K[1, 1]
        assert K[0, 2] != np.floor(K[0, 2]) and K[1, 2] != np.floor(K[1, 2])


def _exact_fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def test_emulated_fma_is_exactly_rounded():
    from oracle.sunrgbd_depth import fma
    rng = np.random.default_rng(5)
    n = 4000
    a = rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6, n)
    b = rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6, n)
    c = -a * b * (1 + rng.standard_normal(n) * 2.0 ** -rng.integers(20, 60, n))   # cancellation
    c[: n // 2] = rng.standard_normal(n // 2) * 10.0 ** rng.integers(-8, 8, n // 2)
    c[:50] = 0.0
    a[50:60] = 0.0
    got = fma(a, b, c)
    want = np.array([_exact_fma(x, y, w) for x, y, w in zip(a, b, c)])
    assert np.array_equal(got, want)
    # halfway cases, where a plain product-then-sum rounds twice
    x = 1.0 + 2.0 ** -30
    assert fma(np.array([x]), np.array([x]), np.array([-1.0]))[0] == _exact_fma(x, x, -1.0)
    assert fma(np.array([1.0 + 2.0 ** -52]), np.array([1.0 - 2.0 ** -53]), np.array([2.0 ** -54]))[0] == \
        _exact_fma(1.0 + 2.0 ** -52, 1.0 - 2.0 ** -53, 2.0 ** -54)
    # signed zeros: -0 only from (-0) + (-0)
    for s in ((0.0, 1.0, -0.0), (-0.0, 1.0, -0.0), (2.0, 3.0, -6.0)):
        assert np.signbit(fma(*(np.array([v]) for v in s))[0]) == np.signbit(s[0] * s[1] + s[2]), s


def test_the_oracle_matmul_orders_are_exact_fma_chains():
    """rtilt_rows restates np.matmul(R, p.T): the dgemm order for n >= 2 and gemv's for n = 1, term by term."""
    from oracle import sunrgbd_depth as osd
    z, cases = _golden()
    cal = z["calib_" + cases[0]]
    R = cal[:9].reshape(3, 3)
    p = np.random.default_rng(2).standard_normal((40, 3)) * 4
    many, one = osd.rtilt_rows(R, p), osd.rtilt_rows(R, p[:1])
    for k in range(3):
        for i in range(len(p)):
            t = float(Fraction(R[k, 0]) * Fraction(p[i, 0]))
            assert many[i, k] == _exact_fma(R[k, 2], p[i, 2], _exact_fma(R[k, 1], p[i, 1], t))
        t = float(Fraction(R[k, 1]) * Fraction(p[0, 1]))
        assert one[0, k] == _exact_fma(R[k, 2], p[0, 2], _exact_fma(R[k, 0], p[0, 0], t))


def test_frame_cloud_crops_and_flags():
    from oracle import sunrgbd_depth as osd
    z, cases = _golden()
    c = [c for c in cases if c.startswith("random")][0]
    raw, rgb, cal = z["depth_" + c], z["rgb_" + c], z["calib_" + c]
    full = osd.depth_cloud(raw, rgb, cal[:9].reshape(3, 3), cal[9:].reshape(3, 3))
    n = len(full)
    cloud, cnt, bits = osd.frame_cloud(raw, rgb, raw.shape, cal, *raw.shape, n)
    assert cnt == n and bits == 0 and np.array_equal(cloud, full)
    cloud, cnt, bits = osd.frame_cloud(raw, rgb, raw.shape, cal, *raw.shape, n - 1)
    assert cnt == n and bits == 1 and np.array_equal(cloud, full[:n - 1])
    cloud, cnt, bits = osd.frame_cloud(raw, rgb, (raw.shape[0] + 3, raw.shape[1]), cal, *raw.shape, n)
    assert bits == 128 and np.array_equal(cloud, full)
    h, w = raw.shape[0] - 5, raw.shape[1] - 7
    cloud, cnt, bits = osd.frame_cloud(raw, rgb, (h, w), cal, *raw.shape, n)
    want = osd.depth_cloud(raw[:h, :w], rgb[:h, :w], cal[:9].reshape(3, 3), cal[9:].reshape(3, 3))
    assert bits == 0 and cnt == len(want) and np.array_equal(cloud, want)
    assert osd.frame_cloud(raw, rgb, (-1, w), cal, *raw.shape, n)[1:] == (0, 0)


def _args():
    from frustum_convnet_b200 import _lib
    a = _lib.SunrgbdDepthArgs()
    a.num_frames, a.height, a.width, a.point_capacity = 2, 530, 730, 386900
    return a


def test_entry_argument_checks_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    assert _lib.FRAME_PIXELS == 128
    assert lib.fcn_sunrgbd_depth_cloud(None, None) == -1
    assert lib.fcn_sunrgbd_depth_cloud_workspace_bytes(None) == -1
    for field in ("num_frames", "height", "width", "point_capacity"):
        a = _args()
        setattr(a, field, 0)
        assert lib.fcn_sunrgbd_depth_cloud_workspace_bytes(C.byref(a)) == -1, field
        assert b">= 1" in lib.fcn_last_error(), field
    for field, value in (("num_frames", 65536), ("height", 1 << 16)):
        a = _args()
        setattr(a, field, value)
        a.width = 1 << 15
        assert lib.fcn_sunrgbd_depth_cloud_workspace_bytes(C.byref(a)) == -1, field
        assert b"too large" in lib.fcn_last_error(), field
    a = _args()
    assert lib.fcn_sunrgbd_depth_cloud_workspace_bytes(C.byref(a)) == 1536 + 256   # 2 * 189 tile counts, 2 totals
    assert lib.fcn_sunrgbd_depth_cloud(C.byref(a), None) == -1
    assert b"NULL input" in lib.fcn_last_error()
    a.depth, a.image_hw, a.calibs, a.status = 256, 256, 256, 256
    assert lib.fcn_sunrgbd_depth_cloud(C.byref(a), None) == -1
    assert b"NULL output" in lib.fcn_last_error()
    a.clouds, a.counts = 256, 256
    for field, value in (("depth", 257), ("calibs", 260), ("clouds", 258)):
        setattr(a, field, value)
        assert lib.fcn_sunrgbd_depth_cloud(C.byref(a), None) == -1, field
        assert b"aligned" in lib.fcn_last_error(), field
        setattr(a, field, 256)
    assert lib.fcn_sunrgbd_depth_cloud(C.byref(a), None) == -1                  # no workspace (rgb NULL is fine)
    assert b"workspace" in lib.fcn_last_error()


def test_python_entries_refuse_cpu():
    from frustum_convnet_b200.sunrgbd_depth import depth_clouds
    with pytest.raises(RuntimeError):
        depth_clouds([np.zeros((2, 2), np.uint16)], None, [{"Rtilt": np.eye(3), "K": np.eye(3)}], [0], device="cpu")


@pytest.mark.parametrize("kernel,max_regs", [("sd_count_kernel", 32), ("sd_scan_kernel", 32),
                                             ("sd_write_kernel", 64)])
def test_new_kernels_do_not_spill(kernel, max_regs):
    found = [(n, k) for n, k in compile_cuda("sunrgbd_depth.cu").kernels.items() if kernel in n]
    assert len(found) == 1
    name, k = found[0]
    assert k.local_memory == (0, 0, 0), (name, k.report)
    assert k.registers <= max_regs, (name, k.registers)
