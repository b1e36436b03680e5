"""The host helpers every two-phase device entry uses (frustum_convnet_b200/_host.py): CSR offsets, the packed upload's
layout and the device check, on the CPU."""
import ctypes

import numpy as np
import pytest

from frustum_convnet_b200 import _host, _lib


def test_offsets():
    for counts, want in (([], [0]), ([0], [0, 0]), ([3, 0, 2], [0, 3, 3, 5]), (np.array([1, 4], np.int64), [0, 1, 5])):
        off = _host.csr_offsets(counts)
        assert off.dtype == np.int32
        assert off.tolist() == want


def test_pack_places_every_part_at_a_256_byte_boundary():
    frames = (_lib.FrustumFrame * 3)()
    frames[1].P[5], frames[2].height = 2.5, 7
    box = np.zeros(2, dtype=np.dtype(_lib.RefineBox))
    box["cs"] = [0.5, -1.0]
    parts = [bytes(frames),                                       # ctypes records, as bytes
             np.arange(12, dtype=np.float64).reshape(3, 4).T,     # not contiguous: packed in C order
             np.array([0, 4, 10], np.int32),
             np.zeros((0, 4), np.float64),                        # empty part: no bytes, still a start
             box,                                                 # structured records
             np.array([-1], np.int32)]
    buf, starts = _host.pack(parts)
    assert buf.dtype == np.uint8 and buf.ndim == 1
    want = [bytes(frames), np.ascontiguousarray(parts[1]).tobytes(), parts[2].tobytes(), b"", box.tobytes(),
            parts[5].tobytes()]
    end = 0
    for s, w in zip(starts, want):
        assert s % _host.ALIGN == 0 and s == end
        assert buf[s:s + len(w)].tobytes() == w
        end = s + -(-len(w) // _host.ALIGN) * _host.ALIGN
    assert buf.size == end
    assert not buf[starts[0] + ctypes.sizeof(frames):starts[1]].any()   # padding is zero


def test_cpu_device_raises_naming_the_caller():
    with pytest.raises(RuntimeError, match="SomeEvaluator: a CUDA device is required"):
        _host.cuda_device("cpu", "SomeEvaluator")
