"""GPU: the frame detection store (frame_detect.FrameStore, C ABI section (25)).  The entry against its numpy
restatement (tests/frame_store_ref.py) on random call tables inside guard bands, at exact-fit and one-short
capacities; the store of K frame calls against the merge of each call's to_dict taken right after it; graph replay of
detect (+ refine) + append against eager calls; and the evaluators and the refinement extractor fed from the store
against the merged dict."""
import ctypes as C

import numpy as np
import pytest
import torch

from frame_store_ref import STORE_ROWS, STORE_SEGMENTS, Store, call_tables
from test_gpu_frame_detect import _frames, _model, _same

pytestmark = pytest.mark.gpu

TYPES = ("Car", "Pedestrian", "Cyclist")
GUARD = 4096


# ------------------------------------------------------------------------------------------------ the entry
class _Guarded:
    """A device buffer of `shape` with GUARD bytes of a fixed pattern on each side."""

    def __init__(self, shape, dtype):
        n = int(np.prod(shape))
        item = torch.empty(0, dtype=dtype).element_size()
        g = GUARD // item
        self.raw = torch.empty(n + 2 * g, dtype=dtype, device="cuda")
        self.raw.view(torch.uint8).fill_(0xA5)
        self.t = self.raw[g:g + n].view(shape)
        self.g = g

    def intact(self):
        b = self.raw.view(torch.uint8)
        return bool((b[:GUARD] == 0xA5).all()) and bool((b[-GUARD:] == 0xA5).all())


def _entry_store(F, Cn, R, rows, segments):
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200._host import workspace
    bufs = {"rows": _Guarded((rows, 12), torch.float32), "image": _Guarded((segments,), torch.int64),
            "cls": _Guarded((segments,), torch.int32), "frame": _Guarded((segments,), torch.int32),
            "offset": _Guarded((segments + 1,), torch.int32), "keep": _Guarded((segments,), torch.int32),
            "cursor": _Guarded((5,), torch.int32)}
    bufs["cursor"].t.zero_()
    call = {"rows": _Guarded((R, 12), torch.float32), "off": _Guarded((Cn * F + 1,), torch.int32),
            "keep": _Guarded((Cn * F,), torch.int32), "cls": _Guarded((F, Cn), torch.int32),
            "status": _Guarded((1,), torch.int32), "ids": _Guarded((F,), torch.int64)}
    a = _lib.FrameStoreArgs()
    a.num_frames, a.num_classes, a.num_rows, a.row_capacity, a.segment_capacity = F, Cn, R, rows, segments
    a.rows, a.seg_offsets, a.keep_count = call["rows"].t.data_ptr(), call["off"].t.data_ptr(), call["keep"].t.data_ptr()
    a.seg_class, a.status, a.ids = call["cls"].t.data_ptr(), call["status"].t.data_ptr(), call["ids"].t.data_ptr()
    a.store_rows, a.store_image, a.store_class = (bufs[k].t.data_ptr() for k in ("rows", "image", "cls"))
    a.store_frame, a.store_offset, a.store_keep = (bufs[k].t.data_ptr() for k in ("frame", "offset", "keep"))
    a.cursor = bufs["cursor"].t.data_ptr()
    ws, a.workspace_bytes = workspace("fcn_frame_store_append_workspace_bytes", torch.device("cuda"), C.byref(a))
    a.workspace = ws.data_ptr()
    return a, bufs, call, ws


def _entry_append(a, call, tables, status, ids):
    from frustum_convnet_b200 import _lib
    rows, off, kc, cls = tables
    for k, v in (("rows", rows), ("off", off), ("keep", kc), ("cls", cls)):
        call[k].t.copy_(torch.from_numpy(np.ascontiguousarray(v)))
    call["status"].t.fill_(status)
    call["ids"].t.copy_(torch.from_numpy(np.asarray(ids, np.int64)))
    _lib.call("fcn_frame_store_append", C.byref(a), torch.cuda.current_stream().cuda_stream)


def _check_entry(bufs, ref):
    torch.cuda.synchronize()
    assert all(b.intact() for b in bufs.values())
    cur = bufs["cursor"].t.cpu().numpy()
    assert list(cur) == list(ref.cursor)
    n, m = int(cur[0]), int(cur[1])
    for k, want in (("image", ref.image), ("cls", ref.cls), ("frame", ref.frame), ("keep", ref.keep)):
        assert np.array_equal(bufs[k].t[:n].cpu().numpy(), want[:n]), k
    if n:
        assert np.array_equal(bufs["offset"].t[:n + 1].cpu().numpy(), ref.offset[:n + 1])
    assert np.array_equal(bufs["rows"].t[:m].cpu().numpy().view(np.int32), ref.rows[:m].view(np.int32))


def _entry_calls(seed, K, F, Cn, R, cut=False):
    rng = np.random.default_rng(seed)
    calls = []
    for k in range(K):
        tables = call_tables(rng, F, Cn, R, max_keep=9)
        if cut:                     # tables no stage writes: offsets and counts outside the call's rows
            rows, off, kc, cls = tables
            off = rng.integers(-5, R + 6, len(off)).astype(np.int32)
            kc = rng.integers(-2, 12, len(kc)).astype(np.int32)
            tables = (rows, off, kc, cls)
        ids = np.arange(k * F, (k + 1) * F, dtype=np.int64)
        ids[rng.random(F) < 0.25] = -1
        calls.append((tables, int(rng.choice([0, 1, 8, 16])), ids))
    return calls


@pytest.mark.parametrize("F,Cn,R,cut", [(1, 3, 40, False), (8, 3, 200, False), (64, 10, 3000, False),
                                        (5, 3, 32, True)])
def test_entry_equals_the_restatement(F, Cn, R, cut):
    calls = _entry_calls(F * 7 + Cn, 6, F, Cn, R, cut)
    calls.insert(2, ((calls[0][0][0], np.zeros(Cn * F + 1, np.int32), np.zeros(Cn * F, np.int32),
                      np.full((F, Cn), -1, np.int32)), 4, np.arange(F)))               # a call with no segment
    calls.insert(3, (calls[1][0], 2, np.full(F, -1)))                                  # every slot unused
    a, bufs, call, _ = _entry_store(F, Cn, R, 20000, 4000)
    ref = Store(20000, 4000)
    for tables, status, ids in calls:
        _entry_append(a, call, tables, status, ids)
        ref.append(*tables, status, ids)
    _check_entry(bufs, ref)
    assert ref.cursor[0] > 0 and ref.cursor[2] == len(calls)


@pytest.mark.parametrize("short", ["rows", "segments"])
@pytest.mark.parametrize("by", [0, 1])
def test_entry_capacity_edges(short, by):
    """The last of four calls at exact fit (by = 0) or one short: absent, the bit set, earlier calls intact, every
    guard band whole; a later call that fits is still stored."""
    F, Cn, R = 6, 3, 120
    calls = _entry_calls(40, 5, F, Cn, R)
    probe = Store(100000, 10000)
    for tables, status, ids in calls[:4]:
        probe.append(*tables, status, ids)
    segs, rows = int(probe.cursor[0]), int(probe.cursor[1])
    cap_rows, cap_segs = (rows - by, segs + 50) if short == "rows" else (rows + 50, segs - by)
    a, bufs, call, _ = _entry_store(F, Cn, R, cap_rows, cap_segs)
    ref = Store(cap_rows, cap_segs)
    results = []
    for tables, status, ids in calls[:4]:
        _entry_append(a, call, tables, status, ids)
        results.append(ref.append(*tables, status, ids))
    assert results == [True] * 3 + [by == 0]
    assert ref.cursor[3] == (0 if by == 0 else STORE_ROWS if short == "rows" else STORE_SEGMENTS)
    _check_entry(bufs, ref)
    if by:
        rows0, off0, kc0, cls0 = calls[4][0]
        small = (rows0, off0, np.minimum(kc0, 0), cls0)                               # zero rows, a few segments
        ids = calls[4][2] if short == "rows" else np.full(F, -1)                   # rows short: no row; else no segment
        _entry_append(a, call, small, 8, ids)
        assert ref.append(*small, 8, ids)
        _check_entry(bufs, ref)


# ------------------------------------------------------------------------------------------------ FrameStore
def _split_frames(seed, K, F, types=TYPES):
    """K calls of at most F frames: frame 1 of call 0 has no detection, call 1 has one class only, the last call is
    partially filled (F > 1).  -> [(frames, ids)]."""
    out, nxt = [], 0
    for k in range(K):
        frames = _frames(seed + k, F, types=types)
        if k == 0 and F > 1:
            frames[1] = frames[1][:3] + ([],)
        if k == 1:
            frames = [fr[:3] + ([d for d in fr[3] if d[0] == fr[3][0][0]],) for fr in frames]
        if k == K - 1 and F > 1:
            frames = frames[:F - 1]
        out.append((frames, list(range(nxt, nxt + len(frames)))))
        nxt += len(frames)
    return out


def _per_call(fd, store, inp, split, call=None):
    """Eager calls of the detector fd (or of `call`, which reads fd's inputs), each appended; -> the merge of each
    call's to_dict(ids) taken right after it, and the OR of the calls' status words."""
    want, status = {}, 0
    call = call or (lambda: fd.detect(*inp))
    for frames, ids in split:
        fd.stage(inp, frames)
        store.stage_ids(ids)
        out = call()
        store.append(out)
        full = list(ids) + [-1] * (fd.F - len(ids))
        want.update({i: v for i, v in out.to_dict(full).items() if i >= 0})
        status |= out.status_bits()
    return want, status


@pytest.mark.parametrize("method", ["nms", "top"])
@pytest.mark.parametrize("F", [1, 4])
def test_store_equals_the_merged_per_call_dicts(F, method):
    from frustum_convnet_b200.frame_detect import FrameDetector, FrameStore
    fd = FrameDetector(_model("car"), TYPES, method=method, seed=7, frames=F, points=120000, dets=8)
    store = FrameStore(fd, rows=50000, segments=2000)
    inp = fd.inputs()
    want, status = _per_call(fd, store, inp, _split_frames(500 + F, 4, F))
    assert want and any(len(v) < 3 for v in want.values())
    _same(store.to_dict(), want)
    assert store.status_bits() == (0, status)
    c = store.collected()
    assert c.dataset == "KITTI" and list(c.order) == list(range(c.num_segments))
    assert c.num_rows == sum(len(r) for v in want.values() for r in v.values())


def test_graph_replay_equals_eager_calls():
    from frustum_convnet_b200.frame_detect import FrameDetector, FrameStore
    F = 2
    fd = FrameDetector(_model("car"), TYPES, seed=7, frames=F, points=120000, dets=8)
    store = FrameStore(fd, rows=20000, segments=1000)
    inp = fd.inputs()
    split = _split_frames(520, 4, F)
    fd.stage(inp, split[0][0])
    store.stage_ids(split[0][1])
    store.append(fd.detect(*inp))                        # the eager call before capture
    g, g_reset = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            store.append(fd.detect(*inp))
        with torch.cuda.graph(g_reset, stream=s):
            store.reset()
    torch.cuda.current_stream().wait_stream(s)
    assert store.status_bits() == (0, 0) and store.collected().num_segments > 0
    g_reset.replay()
    assert store.collected().num_segments == 0 and int(store.cursor[2].item()) == 0
    c0 = fd.call.clone()
    for frames, ids in split:
        fd.stage(inp, frames)
        store.stage_ids(ids)
        g.replay()
    got, bits = store.to_dict(), store.status_bits()
    store.reset()
    fd.call.copy_(c0)
    want, status = _per_call(fd, store, inp, split)
    assert got and bits == (0, status)
    _same(got, want)
    _same(store.to_dict(), want)


def test_graph_replay_of_detect_refine_and_append():
    from frustum_convnet_b200.frame_detect import FrameDetector, FrameRefiner, FrameStore
    F = 2
    fd = FrameDetector(_model("car"), TYPES, seed=7, frames=F, points=120000, dets=8)
    fr = FrameRefiner(fd, _model("refine_car"), type_whitelist=TYPES, jobs=64, seed=1)
    store = FrameStore(fr, rows=20000, segments=1000)
    inp = fd.inputs()
    split = _split_frames(540, 3, F)
    fd.stage(inp, split[0][0])
    store.append(fr.refine(inp, fd.detect(*inp)))
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            store.append(fr.refine(inp, fd.detect(*inp)))
    torch.cuda.current_stream().wait_stream(s)
    store.reset()
    c1, c2 = fd.call.clone(), fr.call.clone()
    for frames, ids in split:
        fd.stage(inp, frames)
        store.stage_ids(ids)
        g.replay()
    got, bits = store.to_dict(), store.status_bits()
    store.reset()
    fd.call.copy_(c1)
    fr.call.copy_(c2)
    want, status = _per_call(fd, store, inp, split, call=lambda: fr.refine(inp, fd.detect(*inp)))
    assert got and bits == (0, status)
    _same(got, want)


def test_kitti_evaluator_and_refinement_from_the_store():
    from det_feed_sets import kitti_set
    from test_gpu_det_eval_feed import compare_kitti_results, kitti_gt
    from frustum_convnet_b200 import refine_extract as rx
    from frustum_convnet_b200.frame_detect import FrameDetector, FrameStore
    F = 2
    fd = FrameDetector(_model("car"), TYPES, seed=7, frames=F, points=120000, dets=8)
    store = FrameStore(fd, rows=20000, segments=1000)
    inp = fd.inputs()
    split = _split_frames(560, 3, F)
    x = rx.RefineFrustumExtractor(TYPES)
    scans, calibs, hws = {}, {}, {}
    per_call, want = [], {}
    for frames, ids in split:
        for i, fr_ in zip(ids, frames):
            scans[i], calibs[i], hws[i] = fr_[0], fr_[1], fr_[2]
        fd.stage(inp, frames)
        store.stage_ids(ids)
        out = fd.detect(*inp)
        store.append(out)
        full = list(ids) + [-1] * (F - len(ids))
        want.update({i: v for i, v in out.to_dict(full).items() if i >= 0})
        per_call.append(x.from_collected({i: scans[i] for i in ids}, {i: calibs[i] for i in ids},
                                         {i: hws[i] for i in ids}, list(ids), out.collected(full)))
    n = len(scans)
    gts, _ = kitti_set(n, seed=5)
    ev = kitti_gt(list(range(n)), gts)
    collected = store.collected()
    compare_kitti_results(ev.evaluate_collected(collected), ev.evaluate(want))
    ids = sorted(scans)
    b = x.from_collected(scans, calibs, hws, ids, collected)
    assert len(b) > 0
    # bit for bit: the store's frustums are the per-call device frustums one after another
    assert b.id_list == [i for p in per_call for i in p.id_list]
    assert b.type_list == [t for p in per_call for t in p.type_list]
    assert torch.equal(b.points, torch.cat([p.points for p in per_call]))
    for name in ("frustum_angle_list", "pred_box3d_list", "pred_box3d_size_list", "pred_box3d_angle_list",
                 "prob_list", "box2d_list"):
        got = np.array(getattr(b, name))
        cat = np.concatenate([np.array(getattr(p, name)).reshape((-1,) + got.shape[1:]) for p in per_call])
        assert got.tobytes() == cat.tobytes(), name
    # and the same jobs, points and row-copied values as the dict path on the merged dict
    a = x.from_detections(scans, calibs, hws, ids, want)
    assert len(a) == len(b) and a.id_list == b.id_list and a.type_list == b.type_list
    assert torch.equal(a.offsets, b.offsets) and torch.equal(a.points, b.points)
    assert np.array_equal(a.counts, b.counts) and a.prob_list == b.prob_list
    assert np.array(a.box2d_list).tobytes() == np.array(b.box2d_list).tobytes()


def test_sunrgbd_evaluator_from_the_store():
    from test_gpu_sunrgbd_frame import _detector, _frames as sun_frames, _model as sun_model
    from frustum_convnet_b200.frame_detect import FrameStore
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator, SunrgbdGroundTruth, det_corners
    F = 2
    fd = _detector(sun_model(), F, method="nms")
    store = FrameStore(fd, rows=20000, segments=1000)
    inp = fd.inputs()
    split = [(sun_frames(31 + k, F), [2 * k, 2 * k + 1]) for k in range(2)]
    want, status = _per_call(fd, store, inp, split)
    assert want and store.status_bits() == (0, status)
    _same(store.to_dict(), want)
    rng = np.random.default_rng(0)
    gt = {}
    for f, by_class in want.items():
        for c, rows in by_class.items():
            r = rows[::2]
            corners, ids = gt.setdefault(c, ([], []))
            corners.append(det_corners(r) + rng.uniform(-0.05, 0.05, (len(r), 1, 3)))
            ids += [f] * len(r)
    ev = SunrgbdEvaluator(SunrgbdGroundTruth({c: (np.concatenate(v[0]), np.array(v[1])) for c, v in gt.items()}))
    collected = store.collected()
    assert collected.dataset == "SUNRGBD"
    a, b = ev.evaluate_collected(collected), ev.evaluate(want)
    assert a.ap == b.ap
    for c in a.ap:
        assert np.array_equal(a.rec[c], b.rec[c]) and np.array_equal(a.prec[c], b.prec[c]), c


@pytest.mark.parametrize("short", ["rows", "segments"])
@pytest.mark.parametrize("by", [0, 1])
def test_store_capacities(short, by):
    from frustum_convnet_b200.frame_detect import FrameDetector, FrameStore
    F = 2
    fd = FrameDetector(_model("car"), TYPES, seed=7, frames=F, points=120000, dets=8)
    inp = fd.inputs()
    split = _split_frames(580, 3, F)
    probe = FrameStore(fd, rows=20000, segments=1000)
    c0 = fd.call.clone()
    sizes = []
    for frames, ids in split:
        fd.stage(inp, frames)
        probe.stage_ids(ids)
        probe.append(fd.detect(*inp))
        sizes.append((int(probe.cursor[0].item()), int(probe.cursor[1].item())))
    segs, rows = sizes[-1]
    assert sizes[-1][0] > sizes[-2][0] and sizes[-1][1] > sizes[-2][1]
    store = FrameStore(fd, rows=rows - by if short == "rows" else rows + 10,
                       segments=segs - by if short == "segments" else segs + 10)
    fd.call.copy_(c0)
    want, _ = _per_call(fd, store, inp, split[:-1])
    fd.stage(inp, split[-1][0])
    store.stage_ids(split[-1][1])
    out = fd.detect(*inp)
    store.append(out)
    if by == 0:
        full = list(split[-1][1]) + [-1] * (F - len(split[-1][1]))
        want.update({i: v for i, v in out.to_dict(full).items() if i >= 0})
        _same(store.to_dict(), want)
        assert store.status_bits()[0] == 0
        return
    bit = STORE_ROWS if short == "rows" else STORE_SEGMENTS
    assert store.status_bits()[0] == bit
    with pytest.raises(RuntimeError, match="did not fit"):
        store.collected()
    assert [int(v) for v in store.cursor[:3].tolist()] == [sizes[-2][0], sizes[-2][1], len(split) - 1]
    store.cursor[3] = 0                                  # read the earlier calls past the bit: intact
    _same(store.to_dict(), want)


def test_frame_status_and_duplicate_ids():
    from frustum_convnet_b200.frame_detect import FrameDetector, FrameStore
    fd = FrameDetector(_model("car"), TYPES, seed=7, frames=2, points=120000, dets=8, rows=4)
    store = FrameStore(fd, rows=1000, segments=100)
    inp = fd.inputs()
    fd.stage(inp, _frames(600, 2))
    store.stage_ids([3, 5])
    out = fd.detect(*inp)
    store.append(out)
    assert out.status_bits() & 8
    assert store.status_bits() == (0, out.status_bits())
    store.collected()
    fd.stage(inp, _frames(601, 2))
    store.stage_ids([7, 5])
    store.append(fd.detect(*inp))
    with pytest.raises(ValueError, match="image id 5 "):
        store.collected()
    store.reset()
    assert store.status_bits() == (0, 0) and store.to_dict() == {}
    store.stage_ids([9, 9])
    store.append(fd.detect(*inp))
    with pytest.raises(ValueError, match="image id 9 "):
        store.collected()
