"""CPU: the rank-ordered gradient sum's pieces that need no device - the fcn_rank_fold entry (declared, exported,
argument checks before any launch, a kernel without stack frame or spills), the shard plan of the deterministic
multi-rank step, and the float32 fold reference the GPU tests compare against."""
import os
import re

import numpy as np
import pytest

from frustum_convnet_b200 import build
from rank_fold_ref import F32, left_fold, order_sensitive, same_bits
from toolchain import compile_cuda


def test_the_entry_is_declared_and_exported():
    from frustum_convnet_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(build.HERE), "include", "frustum_b200.h")).read()
    assert re.search(r"FCN_API int fcn_rank_fold\(const float \*src, long long ld, int G, long long n, float \*dst, "
                     r"fcn_stream_t stream\);", hdr)
    assert "fcn_rank_fold" in _lib.SIGNATURES
    assert hasattr(_lib.load(), "fcn_rank_fold")


def test_bad_arguments_are_rejected_before_any_launch():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    buf = np.zeros(256, dtype=np.float32)
    src, dst = buf.ctypes.data, buf.ctypes.data + 4 * 128
    cases = [((None, 8, 2, 8, dst), b"NULL"), ((src, 8, 2, 8, None), b"NULL"), ((src, 8, 0, 8, dst), b"G < 1"),
             ((src, 8, -1, 8, dst), b"G < 1"), ((src, 8, 2, -1, dst), b"n < 0"), ((src, 7, 2, 8, dst), b"ld < n"),
             ((src, 8, 2, 8, src), b"overlaps"), ((src, 8, 2, 8, src + 4 * 15), b"overlaps"),
             ((src, 64, 3, 8, src + 4 * 64), b"overlaps"), ((dst, 8, 2, 8, dst - 4 * 7), b"overlaps"),
             ((src, 1 << 62, 3, 8, dst), b"overflows")]
    for args, word in cases:
        assert lib.fcn_rank_fold(*args, None) == -1, args
        assert word in lib.fcn_last_error(), (args, lib.fcn_last_error())
    assert lib.fcn_rank_fold(src, 8, 2, 0, dst, None) == 0                 # n == 0: nothing to launch
    assert lib.fcn_rank_fold(src, 8, 2, 0, src, None) == 0
    with pytest.raises(RuntimeError, match="ld < n"):
        _lib.call("fcn_rank_fold", src, 3, 2, 4, dst, None)


def test_fold_kernels_have_no_stack_frame_or_spills():
    usage = {m: k.local_memory for m, k in compile_cuda("train.cu").kernels.items()}
    found = [v for k, v in usage.items() if "rank_fold_kernel" in k]
    assert found == [(0, 0, 0), (0, 0, 0)], usage          # the float4 and the scalar kernel


# ----------------------------------------------------------------------------------------------- the shard plan
KITTI_PIECES = (275968, 3040809)          # PointNet, ConvFeatNet + heads: 3 316 777 floats
SUNRGBD_PIECES = (475392, 6192197)        # 6 667 589 floats


@pytest.mark.parametrize("n", (1, 3, 4, 5) + KITTI_PIECES + SUNRGBD_PIECES + (3316777, 6667589))
@pytest.mark.parametrize("world", range(1, 9))
def test_shard_plan_covers_the_piece_in_aligned_equal_shards(n, world):
    from frustum_convnet_b200.train_engine import shard_plan
    shard, padded = shard_plan(n, world)
    assert shard % 4 == 0 and padded == world * shard
    assert padded >= n and padded - n < 4 * world               # the least multiple-of-4 shard that covers n
    assert (shard - 4) * world < n
    offsets = [r * shard for r in range(world)]
    assert offsets[0] == 0 and all(o % 4 == 0 for o in offsets) and offsets[-1] + shard == padded
    assert shard_plan(n, world) == (shard, padded)


def test_shard_plan_small_cases_and_errors():
    from frustum_convnet_b200.train_engine import shard_plan
    assert shard_plan(1, 1) == (4, 4) and shard_plan(1, 8) == (4, 32) and shard_plan(5, 1) == (8, 8)
    assert shard_plan(5, 2) == (4, 8) and shard_plan(9, 2) == (8, 16) and shard_plan(3316777, 8) == (414600, 3316800)
    for n, w in ((0, 2), (4, 0), (-1, 1)):
        with pytest.raises(ValueError):
            shard_plan(n, w)


@pytest.mark.parametrize("wl,pieces", [("refine_car", KITTI_PIECES), ("car", KITTI_PIECES),
                                       ("sunrgbd", SUNRGBD_PIECES)])
def test_the_real_buckets_split_where_the_step_cuts_them(wl, pieces):
    from frustum_convnet_b200 import config
    from frustum_convnet_b200.train_engine import piece_split
    cfg, w = config.load_workload(wl)
    if w["arch"].num_scales == 5:
        from frustum_convnet_b200.det_base_sunrgbd import PointNetDet
    else:
        from frustum_convnet_b200.det_base import PointNetDet
    m = PointNetDet(3, num_vec=w["num_vec"])
    n = sum(p.numel() for p in m.parameters())
    split = piece_split(m)
    assert (split, n - split) == pieces


# ----------------------------------------------------------------------------------------------- the reference
def test_left_fold_is_the_rank_order():
    rows = np.array([[2.0 ** 24, 1.0, -0.0, np.inf], [1.0, 2.0 ** -149, -0.0, -1.0], [1.0, -(2.0 ** -149), -0.0, 1.0]],
                    dtype=F32)
    got = left_fold(rows)
    assert got[0] == F32(2.0 ** 24)                       # (2^24 + 1) rounds to even, then again
    assert got[1] == F32(1.0) and np.signbit(got[2]) and got[3] == np.inf
    assert same_bits(left_fold(rows[:1]), rows[0])        # G == 1 is a copy


@pytest.mark.parametrize("G", [3, 4, 7, 8, 16])
def test_the_order_sensitive_input_tells_the_rank_order_from_others(G):
    rows = order_sensitive(G, 1023, seed=G)
    want = left_fold(rows)
    assert not same_bits(want, left_fold(rows[::-1]))
    assert not same_bits(want, left_fold(rows[np.r_[1:G, 0]]))
    with np.errstate(invalid="ignore", over="ignore"):
        f64 = rows.astype(np.float64).sum(0).astype(F32)
    assert not same_bits(want, f64)
    assert np.isnan(want).any() and np.isinf(want).any()
    assert (np.abs(rows) < np.finfo(F32).tiny).any()      # subnormals
