"""CPU: the counter-based resampling draw of csrc/resample.cu restated in numpy (tests/resample_ref.py), the argument
checks of the frame-detection entries (C ABI section (21)) and the ptxas usage of their kernels."""
import numpy as np
import pytest

from resample_ref import choice_row, philox4x32_10
from toolchain import compile_cuda


def test_philox_known_answers():
    """Random123's known-answer vectors for philox4x32_10."""
    got = [int(w) for w in philox4x32_10(0, 0, 0, 0, 0, 0)]
    assert got == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    m = 0xFFFFFFFF
    got = [int(w) for w in philox4x32_10(m, m, m, m, m, m)]
    assert got == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    pi = [0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344, 0xA4093822, 0x299F31D0]
    got = [int(w) for w in philox4x32_10(*pi)]
    assert got == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


@pytest.mark.parametrize("n,N", [(1024, 1024), (1025, 1024), (5000, 1024), (70000, 2048), (3, 1)])
def test_without_replacement_draws_distinct_indices(n, N):
    for slot in (0, 7, 123):
        c = choice_row(n, N, seed=11, slot=slot, call=5)
        assert c.shape == (N,) and c.dtype == np.int32
        assert c.min() >= 0 and c.max() < n
        assert len(np.unique(c)) == N


@pytest.mark.parametrize("n,N", [(1, 1024), (7, 1024), (1023, 1024)])
def test_with_replacement_draws_in_range(n, N):
    c = choice_row(n, N, seed=3, slot=2, call=0)
    assert c.shape == (N,) and c.min() >= 0 and c.max() < n
    if n == 1:
        assert (c == 0).all()
    else:
        assert len(np.unique(c)) > 1


def test_key_repeats_and_every_key_part_matters():
    base = choice_row(4000, 1024, seed=9, slot=5, call=2)
    assert np.array_equal(base, choice_row(4000, 1024, seed=9, slot=5, call=2))
    for kw in (dict(seed=10, slot=5, call=2), dict(seed=9, slot=6, call=2), dict(seed=9, slot=5, call=3),
               dict(seed=9, slot=5, call=2 + (1 << 32)), dict(seed=9 + (1 << 32), slot=5, call=2)):
        assert not np.array_equal(base, choice_row(4000, 1024, **kw)), kw
    assert (choice_row(0, 16, 1, 1, 1) == 0).all()


def test_without_replacement_is_uniform_over_positions():
    """The first index of permutation(n)[:N] is uniform over [0, n): a chi-square over 4000 keys."""
    n, N = 40, 32
    first = np.array([choice_row(n, N, seed=1, slot=s, call=0)[0] for s in range(4000)])
    counts = np.bincount(first, minlength=n)
    chi2 = float(((counts - 100.0) ** 2 / 100.0).sum())
    assert chi2 < 80.0, chi2           # 39 degrees of freedom: p < 1e-4 above 80


def test_entry_argument_checks_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    assert lib.fcn_frame_extract(None, None) == -1
    a = _lib.FrameExtractArgs()
    a.num_frames, a.scan_capacity, a.det_capacity, a.out_capacity = 1, 16, 4, 1 << 24
    assert lib.fcn_frame_extract_workspace_bytes(C_ref(a)) == -1
    assert b"too large" in lib.fcn_last_error()
    a.out_capacity = 16
    assert lib.fcn_frame_extract(C_ref(a), None) == -1
    assert b"NULL" in lib.fcn_last_error()
    r = _lib.ResampleArgs()
    r.B, r.N = 1, 2049
    assert lib.fcn_resample_choice(C_ref(r), None) == -1
    r.B, r.N = 0, 1024
    assert lib.fcn_resample_choice(C_ref(r), None) == 0
    r.B = 2
    assert lib.fcn_resample_choice(C_ref(r), None) == -1
    assert lib.fcn_det_candidates_valid(None, None, None) == -1
    d = _lib.DetCandidateArgs()
    d.B, d.T2, d.num_frustums, d.capacity = 1, 4, 1, 8
    for name in ("cls_probs", "center", "heading", "size", "rot_angle", "seg_of_frustum", "counter", "records"):
        setattr(d, name, 256)
    assert lib.fcn_det_candidates_valid(C_ref(d), None, None) == -1
    assert b"valid" in lib.fcn_last_error()
    assert lib.fcn_det_finalize_capacity(None, None, None) == -1


def C_ref(s):
    import ctypes
    return ctypes.byref(s)


@pytest.mark.parametrize("src,kernels", [
    ("resample.cu", ["resample_choice_kernel"]),
    ("frame_extract.cu", ["frame_setup_kernel", "frame_pack_kernel", "frame_slots_kernel"]),
])
def test_new_kernels_do_not_spill(src, kernels):
    seen = set()
    for name, k in compile_cuda(src).kernels.items():
        for want in kernels:
            if want in name:
                seen.add(want)
                assert (k.spill_stores, k.spill_loads) == (0, 0), (name, k.report)
                assert k.registers <= 64, (name, k.registers)          # 1024-thread CTAs need <= 64 registers a thread
    assert seen == set(kernels)
