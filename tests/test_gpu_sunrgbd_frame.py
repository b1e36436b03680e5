"""GPU: SunrgbdFrameDetector (frame_detect.py, C ABI section (23)) against the offline chain on the same frames, the
same cap draws and the same resampling indices; its device draws against tests/resample_ref.py; every output of all B
entries against tests/sunrgbd_frame_ref.py at the capacity edges, each output buffer inside guard regions; its replay
from a captured CUDA graph; and the evaluator on its collected rows.

The offline chain is SunrgbdFrustumExtractor.from_rgb_detections (its rng's choice returns the frame path's cap rows
in job order) -> TrainBatchBuilder.from_frustums(.., "sunrgbd", labels=False) fed the frame path's choice -> the model
-> DetectionCollector(dataset="SUNRGBD") -> finalize().  The forward runs on the K kept frustums alone (B = K): every
kernel of the eval forward works per frustum, so a frustum's outputs do not depend on the batch size."""
import numpy as np
import pytest
import torch

from resample_ref import choice_row

pytestmark = pytest.mark.gpu

CAP = 2048


def _frames(seed, F, H=240, W=320, n_objects=6):
    """F synthetic SUN-RGBD frames with one detection per label box (jittered, plus the lamp no model class covers);
    the first box is cut to 30 x 30 px, so each frame has frustums on both sides of the 2048-point cap."""
    from oracle import sunrgbd_scene_synth as ss
    from frustum_convnet_b200 import sunrgbd_extract as sx
    rng = np.random.default_rng(seed)
    out = []
    for f in range(F):
        cloud, cal, lines = ss.large_frame(seed * 10 + f, H, W, n_objects)
        dets = [(o.classname, float(np.float32(rng.uniform(0.1, 1.0))), o.box2d + rng.uniform(-4, 4, 4))
                for o in (sx.SUNObject3d(ln) for ln in lines)]
        c = (dets[0][2][:2] + dets[0][2][2:]) / 2          # one frustum under the cap: a 30 x 30 px box
        dets[0] = (dets[0][0], dets[0][1], np.concatenate([c - 15, c + 15]))
        out.append((cloud, cal, dets))
    return out


def _model():
    from frustum_convnet_b200 import config
    from train_ref import make_model
    config.load_workload("sunrgbd")
    return make_model("sunrgbd", 5).eval()


class _CapRng:
    """An rng whose choice(n, 2048, replace=False) returns the given rows in order (checking n)."""

    def __init__(self, rows):
        self.rows = list(rows)

    def choice(self, n, size, replace=True):
        want_n, row = self.rows.pop(0)
        assert (int(n), size, replace) == (want_n, CAP, False)
        return row.astype(np.int64)


def _detector(model, F, **kw):
    from frustum_convnet_b200.frame_detect import SunrgbdFrameDetector
    kw.setdefault("seed", 11)
    return SunrgbdFrameDetector(model, frames=F, points=kw.pop("points", 100000), dets=kw.pop("dets", 8), **kw)


def _run(fd, frames, inp=None):
    if inp is None:
        inp = fd.inputs()
        fd.stage(inp, frames)
    call = int(fd.call.item())
    out = fd.detect(*inp)
    torch.cuda.synchronize()
    return out, inp, call


def _slot_counts(fd, frames):
    """Per slot the in-box count n > 2048 the offline extractor finds (0 for fewer, -1 for a slot without a candidate
    detection)."""
    from frustum_convnet_b200.sunrgbd_extract import SunrgbdFrustumExtractor
    from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES
    n = np.full(fd.B, -1, np.int64)
    wl = [c for i, c in enumerate(SUNRGBD_CLASSES) if (fd.class_mask >> i) & 1]
    for f, (cloud, cal, dets) in enumerate(frames):
        dets = [d for d in dets if d[0] in SUNRGBD_CLASSES][:fd.D]
        for j, (t, p, b) in enumerate(dets):
            if t not in wl:
                continue
            counts = []
            sx = SunrgbdFrustumExtractor(wl)
            sx._run({0: cloud[:fd.P]}, {0: cal}, [dict(frame=0, box=np.asarray(b, np.float64), type=t, prob=p,
                                                     skip=False)], False, False, _Counter(counts), None, None, 1)
            n[f * fd.D + j] = counts[0] if counts else 0         # only the capped counts are drawn from
    return n


class _Counter:
    """An rng that records each n it is asked to draw from and returns the first 2048 ranks."""

    def __init__(self, seen):
        self.seen = seen

    def choice(self, n, size, replace=True):
        self.seen.append(int(n))
        return np.arange(size)


def _offline(model, fd, frames, out, method):
    """The offline chain on `frames` with the frame path's cap rows and choice -> (frustums, builder, data, dict)."""
    from frustum_convnet_b200.detect import DetectionCollector
    from frustum_convnet_b200.sunrgbd_extract import SunrgbdFrustumExtractor
    from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES, TrainBatchBuilder
    wl = [c for i, c in enumerate(SUNRGBD_CLASSES) if (fd.class_mask >> i) & 1]
    ids, types, boxes, probs, slots = [], [], [], [], []
    for f, (_, _, dets) in enumerate(frames):
        j = 0
        for t, p, b in dets:
            if t not in SUNRGBD_CLASSES:
                continue
            ids.append(f), types.append(t), boxes.append(np.asarray(b, np.float64)), probs.append(p)
            slots.append(f * fd.D + j)
            j += 1
    n = _slot_counts(fd, frames)
    cap = out.cap_choice.cpu().numpy()
    rows = [(int(n[d]), cap[d]) for d, t in zip(slots, types) if t in wl and n[d] > CAP]
    sx = SunrgbdFrustumExtractor(wl)
    fr = sx.from_rgb_detections({f: x[0] for f, x in enumerate(frames)}, {f: x[1] for f, x in enumerate(frames)},
                                ids, types, boxes, probs, rng=_CapRng(rows))
    K = len(fr)
    fr.wait()
    tb = TrainBatchBuilder.from_frustums(fr, "sunrgbd", fd.strides, fd.N, labels=False, max_depth=fd.max_depth)
    table = tb.d_frustums
    tb._install_device(tb.T_of, fd.frustum_records[:K].clone(), tb.counts, tb.d_points, None)
    data = dict(tb.build(np.arange(K), {"choice": out.choice[:K].cpu().numpy()}))
    with torch.no_grad():
        res = model(data)
    col = DetectionCollector(fr.id_list, fr.type_list, fr.box2d_list, dataset="SUNRGBD", method=method)
    col.add(res, data, first=0)
    return fr, table, data, col.finalize()


def _same(a, b):
    assert list(a) == list(b)
    for i in a:
        assert list(a[i]) == list(b[i]), i
        for c in a[i]:
            assert a[i][c].shape == b[i][c].shape, (i, c)
            assert np.array_equal(a[i][c].view(np.int32), b[i][c].view(np.int32)), (i, c)


def _ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a.view(np.int64) - b.view(np.int64))


@pytest.mark.parametrize("method", ["top", "nms"])
@pytest.mark.parametrize("F", [1, 3])
def test_parity_with_the_offline_chain(method, F):
    from frustum_convnet_b200 import _lib
    model = _model()
    frames = _frames(40 + F, F)
    fd = _detector(model, F, method=method)
    out, _, _ = _run(fd, frames)
    assert out.status_bits() == 0
    fr, table, data, want = _offline(model, fd, frames, out, method)
    K = len(fr)
    assert K > 0 and int(out.valid.sum().item()) == K
    assert (np.asarray(fr.counts) == CAP).any() and (np.asarray(fr.counts) < CAP).any()
    # frustums: points, offsets and counts bit for bit
    M = int(fr.offsets[-1].item())
    assert torch.equal(fd.offsets[:K + 1].cpu(), fr.offsets.cpu())
    assert np.array_equal(fd.points[:M].cpu().numpy().view(np.int32), fr.points.cpu().numpy().view(np.int32))
    assert torch.equal(fd.points3[:M], fd.points[:M, :3])
    # records against frustum_table: the angle within 2 ulp (of the angle: rot = pi / 2 + angle is smaller, so one
    # ulp of the angle is several of rot), cos and sin within that and their own 2 ulp, the rest exact
    got = fd.frustum_records[:K].cpu().numpy().view(np.dtype(_lib.TrainFrustum)).reshape(K)
    ref = table.cpu().numpy().view(np.dtype(_lib.TrainFrustum)).reshape(K)
    ulp = np.spacing(np.abs(np.asarray(fr.frustum_angle_list, np.float64)))
    assert (np.abs(got["rot"] - ref["rot"]) <= 2 * ulp).all()
    for k in ("cs", "sn"):
        assert (np.abs(got[k] - ref[k]) <= 2 * ulp + 2 * np.spacing(np.abs(ref[k]))).all(), k
    print("bit-identical angle: %d of %d" % (int((got["rot"] == ref["rot"]).sum()), K))
    for k in ("cx", "cy", "K", "Rtilt", "rgb_prob", "cls_index", "T", "center", "heading", "size", "dist", "box2d",
              "P"):
        assert np.array_equal(got[k], ref[k]), k
    # the batch the frame path built equals the offline builder's on the same records and choice
    for k, v in data.items():
        mine = fd.batch[k][:K] if k in fd.batch else None
        if mine is None:
            continue
        assert np.array_equal(mine.reshape(v.shape).cpu().numpy().view(np.int32), v.cpu().numpy().view(np.int32)), k
    _same(out.to_dict(), want)


def test_cap_draw_and_resampling_equal_the_restatement():
    """Slots of n = 4, 5, 2047, 2048, 2049 and 300 000 in-box points: boxes sized on a sorted u grid."""
    model = _model()
    from oracle import sunrgbd_scene_synth as ss
    cloud, cal, _ = ss.large_frame(3, 530, 730, 0)
    from frustum_convnet_b200 import sunrgbd_extract as sx
    uv = sx.project_upright_depth_to_image(cloud.astype(np.float64), cal["Rtilt"], cal["K"])
    order = np.argsort(uv[:, 0], kind="stable")
    dets = []
    for n in (4, 5, 2047, 2048, 2049, 300000):
        u = uv[order, 0]
        hi = (u[n - 1] + u[n]) / 2 if u[n] > u[n - 1] else None
        assert hi is not None
        dets.append(("chair", 0.5, np.array([-1e9, -1e9, hi, 1e9])))
    fd = _detector(model, 1, points=len(cloud), dets=6, seed=(5 << 33) + 9)
    for rep in range(2):
        out, _, call = _run(fd, [(cloud, cal, dets)])
        assert out.status_bits() == 0
        cap = out.cap_choice.cpu().numpy()
        det = fd.det_index.cpu().numpy()
        off = fd.offsets.cpu().numpy()
        choice = out.choice.cpu().numpy()
        for j, n in enumerate((4, 5, 2047, 2048, 2049, 300000)):
            if n > CAP:
                assert np.array_equal(cap[j], choice_row(n, CAP, fd.seed, j, 2 ** 62 + call)), n
            else:
                assert not cap[j].any()
        assert list(det[:5]) == [1, 2, 3, 4, 5] and det[5] == -1
        for b in range(fd.B):
            n = int(off[b + 1] - off[b])
            slot = int(det[b]) if det[b] >= 0 else fd.B + b
            assert np.array_equal(choice[b], choice_row(n, fd.N, fd.seed, slot, call)), b
        assert list(np.diff(off)[:5]) == [5, 2047, 2048, 2048, 2048]
        # a capped frustum holds its drawn ranks' points, in draw order
        pts = fd.points.cpu().numpy()
        for j, b in ((4, 3), (5, 4)):
            inbox = np.flatnonzero(uv[:, 0] < dets[j][2][2])
            assert len(inbox) == (2049, 300000)[j - 4]
            want = sx.flip_axis_to_camera(cloud[inbox[cap[j]]])
            assert np.array_equal(pts[off[b]:off[b + 1]], want.astype(np.float32))


GUARD, PATTERN = 4096, 0xA5


def _guarded(shape, dtype):
    """A tensor of `shape` inside a buffer with GUARD bytes of PATTERN on each side (the inside holds PATTERN too)
    -> (buffer, tensor)."""
    n = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
    buf = torch.full((n + 2 * GUARD,), PATTERN, dtype=torch.uint8, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(dtype).view(shape)


def _entry(fd, inp, P_out, call):
    """fcn_sunrgbd_frame_extract on the host inputs `inp` (sunrgbd_frame_ref.stage's) in fd's capacities with
    frustum budget P_out, the cap's call counter `call` and every output inside a guarded buffer.  Asserts the guards
    and returns the outputs on the host."""
    import ctypes as C
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200._host import workspace
    clouds, cc, calibs, boxes, cls, prob, dc = inp
    F, D, B = fd.F, fd.D, fd.B
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    d_in = [dev(clouds), dev(cc), dev(np.array([np.concatenate([np.asarray(c["Rtilt"], np.float64).reshape(9),
                                                                 np.asarray(c["K"], np.float64).reshape(9)])
                                                 for c in calibs])),
            dev(boxes), dev(cls), dev(prob), dev(dc), torch.full((1,), call, dtype=torch.int64, device="cuda")]
    a = _lib.SunrgbdFrameExtractArgs.from_buffer_copy(fd._xa)
    a.out_capacity = P_out
    (a.clouds, a.cloud_counts, a.frames, a.boxes, a.det_class, a.det_prob, a.det_counts,
     a.call) = (t.data_ptr() for t in d_in)
    R = F * P_out + B
    outs = {"points": ((R, 6), torch.float32), "xyz": ((R, 3), torch.float32), "offsets": ((B + 1,), torch.int32),
            "det_index": ((B,), torch.int32), "valid": ((B,), torch.int32), "cls_index": ((B,), torch.int32),
            "seg": ((B,), torch.int32), "seg_class": ((F, 10), torch.int32), "rgb_prob": ((B,), torch.float32),
            "box2d": ((B, 4), torch.float32), "cap_choice": ((B, CAP), torch.int32),
            "records": ((B, C.sizeof(_lib.TrainFrustum)), torch.uint8), "status": ((1,), torch.int32)}
    held = {}
    for name, (shape, dt) in outs.items():
        held[name] = _guarded(shape, dt)
        setattr(a, name, held[name][1].data_ptr())
    held["status"][1].zero_()
    ws, a.workspace_bytes = workspace("fcn_sunrgbd_frame_extract_workspace_bytes", torch.device("cuda"), C.byref(a))
    a.workspace = ws.data_ptr()
    _lib.call("fcn_sunrgbd_frame_extract", C.byref(a), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for name, (buf, _) in held.items():
        assert (buf[:GUARD] == PATTERN).all() and (buf[-GUARD:] == PATTERN).all(), name
    return {name: t.cpu().numpy() for name, (_, t) in held.items()}


def _same_tables(got, want):
    """The device outputs of one call against sunrgbd_frame_ref.frame_tables over all B entries."""
    from frustum_convnet_b200 import _lib
    assert int(got["status"][0]) == want["status"]
    off = want["offsets"]
    M = int(off[-1])
    assert np.array_equal(got["offsets"], off)
    assert np.array_equal(got["points"][:M].view(np.int32), want["points"].view(np.int32))
    assert np.array_equal(got["xyz"][:M], want["points"][:, :3])
    for k in ("det_index", "valid", "cls_index", "seg", "seg_class", "rgb_prob", "box2d", "cap_choice"):
        assert np.array_equal(got[k], want[k]), k
    rec = got["records"].view(np.dtype(_lib.TrainFrustum)).reshape(-1)
    ref = want["records"]
    ulp = np.spacing(np.abs(want["angle"]))
    assert (np.abs(rec["rot"] - ref["rot"]) <= 2 * ulp).all()
    for k in ("cs", "sn"):
        assert (np.abs(rec[k] - ref[k]) <= 2 * ulp + 2 * np.spacing(np.abs(ref[k]))).all(), k
    for k in rec.dtype.names:
        if k not in ("rot", "cs", "sn"):
            assert np.array_equal(rec[k], ref[k]), k


def _ref_tables(fd, inp, P_out, call):
    import sunrgbd_frame_ref as sr
    return sr.frame_tables(*inp, P_out=P_out, class_mask=fd.class_mask, seed=fd.seed, call=call, strides=fd.strides,
                           max_depth=fd.max_depth)


def test_capacity_edges_against_the_restatement():
    """Cloud counts P + 1 / P / 0 / -1, detection counts D + 1 / D / 0 / -1, a bad class and non-finite boxes next
    to good ones: status bits, every output of all B entries (dummies included) against sunrgbd_frame_ref, and
    4 096-byte guards around every output buffer intact."""
    import sunrgbd_frame_ref as sr
    model = _model()
    P, D = 60000, 5
    fd = _detector(model, 6, points=P, dets=D)
    inp = sr.stage(sr.synth_frames(77, 6), P, D, cloud_counts=[P + 1, P, 0, -1, P, P],
                   det_counts=[D + 1, D, 3, 2, 0, -1])
    clouds, cc, calibs, boxes, cls, prob, dc = inp
    cls[1, 1] = 10
    boxes[1, 2, 0] = np.nan
    boxes[0, 3, 2] = np.inf
    call = 2 ** 62 + 7
    want = _ref_tables(fd, inp, fd.P_out, call)
    assert want["status"] == sr.SCAN_POINTS | sr.DETS | sr.BAD_DET
    assert 0 < int(want["valid"].sum()) < fd.B and (want["det_points"] > CAP).any()
    _same_tables(_entry(fd, inp, fd.P_out, call), want)


def test_frustum_budget_against_the_restatement():
    """P_out filled exactly by frame 0, one point over, and below its first frustum; frame 1's frustums of the same
    classes run under the same budget.  Every output against sunrgbd_frame_ref, guards intact."""
    import sunrgbd_frame_ref as sr
    model = _model()
    P, D = 100000, 6
    fd = _detector(model, 2, points=P, dets=D)
    frames = sr.synth_frames(91, 2)
    inp = sr.stage(frames, P, D)
    call = 2 ** 62 + 11
    full = _ref_tables(fd, inp, 1 << 20, call)
    k0 = full["kept"][:D]
    k0 = k0[k0 >= 0]
    assert len(k0) >= 3
    for P_out, n0 in ((int(k0.sum()), len(k0)), (int(k0.sum()) - 1, len(k0) - 1), (int(k0[0]) - 1, 0)):
        want = _ref_tables(fd, inp, P_out, call)
        assert sum(1 for d in want["det_index"] if 0 <= d < D) == n0, P_out
        if n0 < len(k0):
            assert want["status"] & sr.OUT_POINTS
        _same_tables(_entry(fd, inp, P_out, call), want)


@pytest.mark.parametrize("mask", [("chair",), ("bed", "table", "chair"), None])
def test_class_masks_and_classes_across_frames(mask):
    from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES
    model = _model()
    frames = _frames(5, 3)
    # the same classes in every frame, in a different order per frame
    kinds = ["chair", "bed", "table", "sofa"]
    frames = [(c, cal, [(kinds[(j + f) % 4], p, b) for j, (_, p, b) in enumerate(d)]) for f, (c, cal, d) in
              enumerate(frames)]
    fd = _detector(model, 3, type_whitelist=SUNRGBD_CLASSES if mask is None else mask)
    out, _, _ = _run(fd, frames)
    assert out.status_bits() == 0
    _, _, _, want = _offline(model, fd, frames, out, "top")
    got = out.to_dict()
    _same(got, want)
    seg_class = fd.seg_class.cpu().numpy()
    for f in range(3):
        names = [SUNRGBD_CLASSES[c] for c in seg_class[f] if c >= 0]
        assert names == list(got.get(f, {}))


def test_graph_replay_equals_eager_calls():
    model = _model()
    frames = _frames(9, 2)
    fd = _detector(model, 2)
    inp = fd.inputs()
    fd.stage(inp, frames)
    fd.detect(*inp)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fd.detect(*inp)
    fd.call.fill_(5)
    fd.cap_call.fill_(2 ** 62 + 5)
    g.replay()
    torch.cuda.synchronize()
    replay = (out.to_dict(), out.choice.clone(), out.cap_choice.clone())
    g.replay()
    torch.cuda.synchronize()
    assert not torch.equal(out.choice, replay[1]) and not torch.equal(out.cap_choice, replay[2])
    fd.call.fill_(5)
    fd.cap_call.fill_(2 ** 62 + 5)
    eager = fd.detect(*inp)
    torch.cuda.synchronize()
    assert torch.equal(eager.choice, replay[1]) and torch.equal(eager.cap_choice, replay[2])
    _same(eager.to_dict(), replay[0])


def test_collected_rows_score_like_the_dict():
    """Ground truth: the frame path's own kept rows, moved a little, so every class has matches and misses."""
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator, SunrgbdGroundTruth, det_corners
    model = _model()
    frames = _frames(21, 2)
    fd = _detector(model, 2, method="nms")
    out, _, _ = _run(fd, frames)
    d = out.to_dict()
    rng = np.random.default_rng(0)
    gt = {}
    for f, by_class in d.items():
        for c, rows in by_class.items():
            r = rows[::2]
            corners, ids = gt.setdefault(c, ([], []))
            corners.append(det_corners(r) + rng.uniform(-0.05, 0.05, (len(r), 1, 3)))
            ids += [f] * len(r)
    assert gt
    ev = SunrgbdEvaluator(SunrgbdGroundTruth({c: (np.concatenate(v[0]), np.array(v[1])) for c, v in gt.items()}))
    a = ev.evaluate_collected(out.collected())
    b = ev.evaluate(d)
    assert a.ap == b.ap
    for c in a.ap:
        assert np.array_equal(a.rec[c], b.rec[c]) and np.array_equal(a.prec[c], b.prec[c]), c
