"""GPU: fcn_rank_fold against the float32 left fold of tests/rank_fold_ref.py, bit for bit (NaN as NaN), on inputs
where another add order gives other bits: both kernel paths (float4 and scalar), offsets that break 16-byte
alignment, ld > n, and argument errors that return a status without launching anything."""
import numpy as np
import pytest
import torch

from rank_fold_ref import left_fold, order_sensitive, same_bits

pytestmark = pytest.mark.gpu


def _fold(src, ld, G, n, dst):
    from frustum_convnet_b200 import _lib
    _lib.call("fcn_rank_fold", src.data_ptr(), ld, G, n, dst.data_ptr(), torch.cuda.current_stream().cuda_stream)


def _run(rows, ld, src_off, dst_off):
    """rows (G, n) placed at src_off floats into a device buffer with row pitch ld; result read from dst_off."""
    G, n = rows.shape
    buf = torch.full((src_off + (G - 1) * ld + n,), float("nan"), device="cuda")
    view = buf[src_off:]
    for r in range(G):
        view[r * ld: r * ld + n].copy_(torch.from_numpy(rows[r]))
    out = torch.full((dst_off + n + 1,), 7.0, device="cuda")
    _fold(view, ld, G, n, out[dst_off:])
    got = out.cpu().numpy()
    assert got[-1] == 7.0 and (dst_off == 0 or got[dst_off - 1] == 7.0)        # nothing written outside dst
    return got[dst_off: dst_off + n]


@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 3316777])
@pytest.mark.parametrize("G", [1, 2, 3, 4, 7, 8, 16])
def test_fold_matches_the_float32_left_fold(G, n):
    rows = order_sensitive(G, n, seed=G * 1009 + n)
    want = left_fold(rows)
    assert same_bits(_run(rows, n, 0, 0), want)
    if G >= 3 and n >= 8:
        assert not same_bits(left_fold(rows[::-1]), want)       # the input can tell the orders apart


@pytest.mark.parametrize("G", [1, 3, 8])
@pytest.mark.parametrize("n", [5, 1023, 1024, 4097])
@pytest.mark.parametrize("ld_extra,src_off,dst_off", [(0, 1, 0), (0, 0, 1), (0, 2, 3), (3, 0, 0), (4, 0, 0),
                                                      (4, 4, 4), (5, 1, 2)])
def test_misaligned_pointers_and_padded_rows(G, n, ld_extra, src_off, dst_off):
    rows = order_sensitive(G, n, seed=n + 17 * G + ld_extra)
    assert same_bits(_run(rows, n + ld_extra, src_off, dst_off), left_fold(rows))


def test_zero_signs_infinities_and_nan():
    rows = np.array([[-0.0, -0.0, 0.0, np.inf, np.inf, np.nan, 1.0, 2.0 ** -149],
                     [-0.0, 0.0, -0.0, -np.inf, 1.0, 1.0, 2.0 ** 24, -(2.0 ** -149)],
                     [-0.0, -0.0, -0.0, 1.0, np.inf, 0.0, 2.0 ** 24, 2.0 ** -149]], dtype=np.float32)
    got = _run(rows, 8, 0, 0)
    assert np.signbit(got[0]) and got[0] == 0 and not np.signbit(got[1]) and not np.signbit(got[2])
    assert np.isnan(got[3]) and got[4] == np.inf and np.isnan(got[5])
    assert got[6] == np.float32(2.0 ** 25) and got[7] == np.float32(2.0 ** -149)
    assert same_bits(got, left_fold(rows))


def test_argument_errors_launch_nothing():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    src = torch.arange(64, dtype=torch.float32, device="cuda")
    dst = torch.full((16,), 7.0, device="cuda")
    s, d = src.data_ptr(), dst.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    for args in ((None, 16, 2, 16, d), (s, 16, 2, 16, None), (s, 16, 0, 16, d), (s, 16, 2, -1, d), (s, 15, 2, 16, d),
                 (s, 16, 2, 16, s + 4 * 20), (d, 4, 2, 4, d + 4 * 4), (s, 1 << 62, 4, 16, d)):
        assert lib.fcn_rank_fold(*args, st) == -1, args
        assert b"fcn_rank_fold: invalid argument" in lib.fcn_last_error()
    torch.cuda.synchronize()
    assert bool((dst == 7.0).all()) and torch.equal(src, torch.arange(64, dtype=torch.float32, device="cuda"))
    assert lib.fcn_rank_fold(s, 16, 2, 0, d, st) == 0
    torch.cuda.synchronize()
    assert bool((dst == 7.0).all())
