"""CPU: the frame detection store (C ABI section (25)) without a GPU: its numpy restatement (tests/frame_store_ref.py)
against the merge of per-call dicts on random call tables (segment order, rebasing, the whole-call capacity rule and
the status words), the entry's argument checks and the ptxas usage of its kernels."""
import ctypes as C

import numpy as np
import pytest

from frame_store_ref import STORE_ROWS, STORE_SEGMENTS, Store, call_dict, call_tables
from toolchain import compile_cuda

CLASSES = ("Car", "Pedestrian", "Cyclist")


def _same(a, b):
    assert list(a) == list(b)
    for i in a:
        assert list(a[i]) == list(b[i]), i
        for c in a[i]:
            assert a[i][c].shape == b[i][c].shape and np.array_equal(a[i][c].view(np.int32), b[i][c].view(np.int32))


def _split(seed, K, F, C=3, R=64, **kw):
    """K calls with ids numbered through the split; some slots -1, the last call partially filled."""
    rng = np.random.default_rng(seed)
    calls, nxt = [], 0
    for k in range(K):
        tables = call_tables(rng, F, C, R, **kw)
        ids = np.arange(nxt, nxt + F, dtype=np.int64)
        nxt += F
        ids[rng.random(F) < 0.2] = -1
        if k == K - 1:
            ids[F // 2 + 1:] = -1
        calls.append((tables, ids, int(rng.choice([0, 0, 4, 8, 32]))))
    return calls


def _needs(calls):
    """Per call: (segments, rows) it appends."""
    out = []
    for (rows, off, kc, cls), ids, _ in calls:
        d = call_dict(rows, off, kc, cls, ids, range(cls.shape[1]))
        out.append((sum(len(v) for v in d.values()), sum(len(r) for v in d.values() for r in v.values())))
    return out


@pytest.mark.parametrize("F", [1, 4, 8])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_store_equals_the_merged_call_dicts(F, seed):
    calls = _split(seed, 6, F)
    st = Store(4096, 1024)
    want, status = {}, 0
    for (rows, off, kc, cls), ids, call_status in calls:
        assert st.append(rows, off, kc, cls, call_status, ids)
        want.update(call_dict(rows, off, kc, cls, ids, CLASSES))
        status |= call_status
    _same(st.to_dict(CLASSES), want)
    n_seg, n_row = (int(v) for v in st.cursor[:2])
    # segment order: frame slot, then class by first appearance; zero-row segments kept
    order = [(i, c) for i, by in want.items() for c in by]
    assert [(int(i), CLASSES[c]) for i, c in zip(st.image[:n_seg], st.cls[:n_seg])] == order
    assert F == 1 or (st.keep[:n_seg] == 0).any()
    # offsets rebased onto the store: a CSR over the appended rows
    assert st.offset[0] == 0 and np.array_equal(np.diff(st.offset[:n_seg + 1]), st.keep[:n_seg])
    assert st.offset[n_seg] == n_row
    assert list(st.cursor[2:]) == [len(calls), 0, status]
    # frames: the call number times F plus the slot
    frames = [k * F + f for k, (_, ids, _) in enumerate(calls) for f in range(F) if ids[f] >= 0]
    assert set(st.frame[:n_seg].tolist()) <= set(frames)


def test_empty_calls_and_unused_slots_add_nothing():
    rng = np.random.default_rng(3)
    st = Store(64, 16)
    rows, off, kc, cls = call_tables(rng, 4, 3, 32)
    assert (cls >= 0).any()
    assert st.append(rows, off, kc, cls, 8, np.full(4, -1))                     # every slot unused
    empty = np.full((4, 3), -1, np.int32)
    assert st.append(rows, np.zeros(13, np.int32), np.zeros(12, np.int32), empty, 0, np.arange(4))   # no segment
    assert list(st.cursor) == [0, 0, 2, 0, 8] and st.offset[0] == 0 and st.to_dict(CLASSES) == {}


def test_rows_are_cut_to_the_call_capacity():
    rows = np.arange(8 * 12, dtype=np.float32).reshape(8, 12)
    cls = np.array([[0, 1, 2]], np.int32)
    st = Store(64, 16)
    assert st.append(rows, np.array([-3, 6, 9, 9], np.int32), np.array([2, 5, 1], np.int32), cls, 0, [7])
    assert list(st.keep[:3]) == [2, 2, 0] and list(st.offset[:4]) == [0, 2, 4, 4]
    assert np.array_equal(st.rows[:2], rows[:2]) and np.array_equal(st.rows[2:4], rows[6:8])
    assert st.append(rows, np.zeros(4, np.int32), np.array([-1, 0, 1], np.int32), cls, 0, [8])
    assert list(st.keep[3:6]) == [0, 0, 1]


@pytest.mark.parametrize("short", ["rows", "segments"])
@pytest.mark.parametrize("by", [0, 1])
def test_whole_call_capacity_rule(short, by):
    """Capacities at exact fit (by = 0) and one short (by = 1) for the last call: a call that does not fit is absent,
    the bit of what was short is set and every earlier call is intact."""
    calls = _split(11, 5, 4)
    needs = _needs(calls)
    segs, rows = sum(n for n, _ in needs), sum(m for _, m in needs)
    assert needs[-1][0] > 0 and needs[-1][1] > 0
    cap = {"rows": rows - by, "segments": segs - by}
    st = Store(cap["rows"] if short == "rows" else rows + 100, cap["segments"] if short == "segments" else segs + 100)
    ok = [st.append(*tables, call_status, ids) for tables, ids, call_status in calls]
    assert ok == [True] * 4 + [by == 0]
    kept = calls if by == 0 else calls[:-1]
    want = {}
    for (r, o, k, c), ids, _ in kept:
        want.update(call_dict(r, o, k, c, ids, CLASSES))
    _same(st.to_dict(CLASSES), want)
    bit = STORE_ROWS if short == "rows" else STORE_SEGMENTS
    assert st.cursor[3] == (bit if by else 0)
    assert st.cursor[2] == len(kept)
    status = 0
    for _, _, s in kept:
        status |= s
    assert st.cursor[4] == status
    # a later call that fits is still stored after a refused one
    if by:
        tables = call_tables(np.random.default_rng(5), 1, 3, 8, p_frame=0.0)
        assert st.append(*tables, 16, [99]) and st.cursor[2] == len(kept) + 1 and st.cursor[4] == status | 16


def test_both_bits_when_both_are_short():
    calls = _split(12, 1, 4, p_frame=1.0)
    (n, m), = _needs(calls)
    st = Store(m - 1, n - 1)
    assert not st.append(*calls[0][0], 0, calls[0][1])
    assert list(st.cursor) == [0, 0, 0, STORE_ROWS | STORE_SEGMENTS, 0]


# ------------------------------------------------------------------------------------------------ the C entry
def _args():
    from frustum_convnet_b200 import _lib
    a = _lib.FrameStoreArgs()
    a.num_frames, a.num_classes, a.num_rows, a.row_capacity, a.segment_capacity = 8, 3, 600, 10000, 1000
    return a


def test_header_constants_and_cursor_layout():
    from frustum_convnet_b200 import _lib
    assert (_lib.STORE_ROWS, _lib.STORE_SEGMENTS) == (STORE_ROWS, STORE_SEGMENTS)
    assert [f for f, _ in _lib.FrameStoreCursor._fields_] == ["segments", "rows", "calls", "status", "frame_status"]
    assert C.sizeof(_lib.FrameStoreCursor) == 20


def test_entry_argument_checks_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    assert lib.fcn_frame_store_append(None, None) == -1
    assert lib.fcn_frame_store_append_workspace_bytes(None) == -1
    for field in ("num_frames", "num_classes", "num_rows", "row_capacity", "segment_capacity"):
        for value in (0, -1):
            a = _args()
            setattr(a, field, value)
            assert lib.fcn_frame_store_append_workspace_bytes(C.byref(a)) == -1, field
            assert b">= 1" in lib.fcn_last_error(), field
            assert lib.fcn_frame_store_append(C.byref(a), None) == -1, field
    for field, value in (("num_frames", _lib.STORE_MAX_FRAMES + 1), ("num_classes", _lib.STORE_MAX_CLASSES + 1)):
        a = _args()
        setattr(a, field, value)
        assert lib.fcn_frame_store_append_workspace_bytes(C.byref(a)) == -1, field
        assert b"out of range" in lib.fcn_last_error(), field
    a = _args()
    assert lib.fcn_frame_store_append_workspace_bytes(C.byref(a)) == 256 + 256        # the plan, 24 source offsets
    a.num_frames, a.num_classes = _lib.STORE_MAX_FRAMES, 10
    assert lib.fcn_frame_store_append_workspace_bytes(C.byref(a)) == 256 + (4 * 655350 + 255) // 256 * 256
    a = _args()
    assert lib.fcn_frame_store_append(C.byref(a), None) == -1
    assert b"NULL input" in lib.fcn_last_error()
    for field in ("rows", "seg_offsets", "keep_count", "seg_class", "status", "ids"):
        setattr(a, field, 256)
    assert lib.fcn_frame_store_append(C.byref(a), None) == -1
    assert b"NULL store" in lib.fcn_last_error()
    stores = ("store_rows", "store_image", "store_class", "store_frame", "store_offset", "store_keep", "cursor")
    for field in stores:
        setattr(a, field, 256)
    for field in stores[1:]:
        setattr(a, field, None)
        assert lib.fcn_frame_store_append(C.byref(a), None) == -1, field
        assert b"NULL store" in lib.fcn_last_error(), field
        setattr(a, field, 256)
    for field in ("rows", "store_rows"):
        setattr(a, field, 264)
        assert lib.fcn_frame_store_append(C.byref(a), None) == -1, field
        assert b"16-byte aligned" in lib.fcn_last_error(), field
        setattr(a, field, 256)
    assert lib.fcn_frame_store_append(C.byref(a), None) == -1                       # no workspace
    assert b"workspace" in lib.fcn_last_error()


def test_python_store_refuses_bad_capacities():
    from frustum_convnet_b200.frame_detect import FrameStore

    class Stage:
        F, classes, dataset, R, device = 1, CLASSES, 0, 8, None
    for rows, segments in ((0, 4), (4, 0), (2 ** 31, 4)):
        with pytest.raises(ValueError):
            FrameStore(Stage(), rows, segments)


@pytest.mark.parametrize("kernel,max_regs", [("fs_plan_kernel", 40), ("fs_copy_kernel", 32)])
def test_new_kernels_have_no_stack_frame_or_spills(kernel, max_regs):
    found = [(n, k) for n, k in compile_cuda("frame_store.cu").kernels.items() if kernel in n]
    assert len(found) == 1
    name, k = found[0]
    assert k.local_memory == (0, 0, 0), (name, k.report)
    assert k.registers <= max_regs, (name, k.registers)
