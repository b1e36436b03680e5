"""GPU: FrameRefiner (frame_detect.py, C ABI section (22)) against the offline cascade on the same first-stage rows and
the same stage-2 resampling indices, its device draw, its capacity bits and guard regions, empty frames, graph replay
of both stages and FrameDetections.collected().

The offline chain is first.collected() -> RefineFrustumExtractor.from_collected -> TrainBatchBuilder.from_frustums(..,
"refine") -> build on the kept entries with the refiner's exported choice -> the center_ref* tensors edge-padded to
the refiner's W with np.pad(mode='edge') -> the refinement model -> DetectionCollector -> finalize().  As in
tests/test_gpu_frame_detect.py the forward runs on the K kept frustums alone: it works per frustum."""
import ctypes as C

import numpy as np
import pytest
import torch

from resample_ref import choice_row
from test_gpu_frame_detect import _frames, _model, _same

pytestmark = pytest.mark.gpu

TYPES = ("Car", "Pedestrian", "Cyclist")
GUARD = 4096


def _pair(F, method="nms", wl=("Car",), seed=1, frames=None, refine_wl=None, **kw):
    """A detector and its refiner (whitelist refine_wl, default wl); J defaults to 256 jobs a frame, room for every
    first-stage row of these frames."""
    from frustum_convnet_b200.frame_detect import FrameDetector, FrameRefiner
    kw.setdefault("jobs", 256)
    fd = FrameDetector(_model("car"), wl, method=method, seed=7, frames=F, points=120000, dets=8)
    fr = FrameRefiner(fd, _model("refine_car"), type_whitelist=refine_wl or wl, method=method, seed=seed, **kw)
    inp = fd.inputs()
    fd.stage(inp, frames if frames is not None else _frames(300 + F, F, types=wl))
    return fd, fr, inp


def _offline(fr, frames, first, out, wl, method):
    """The offline cascade from the first stage's device rows -> (finalize() dict, the refinement frustums)."""
    from frustum_convnet_b200.detect import DetectionCollector
    from frustum_convnet_b200.refine_extract import REFINE_STRIDES, RefineFrustumExtractor
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    F = len(frames)
    rf = RefineFrustumExtractor(wl).from_collected({f: x[0] for f, x in enumerate(frames)},
                                                   {f: x[1] for f, x in enumerate(frames)},
                                                   {f: x[2] for f, x in enumerate(frames)}, list(range(F)),
                                                   first.collected())
    K = len(rf)
    if K == 0:
        return {}, rf
    tb = TrainBatchBuilder.from_frustums(rf, "refine", strides=REFINE_STRIDES, npoints=fr.N)
    data = dict(tb.build(np.arange(K), {"choice": out.choice[:K].cpu().numpy()}))
    for s, w in enumerate(fr.T):
        c = data["center_ref%d" % (s + 1)].cpu().numpy()
        assert c.shape[2] <= w
        data["center_ref%d" % (s + 1)] = torch.from_numpy(
            np.pad(c, ((0, 0), (0, 0), (0, w - c.shape[2])), mode="edge")).cuda()
    with torch.no_grad():
        res = fr.model(data)
    col = DetectionCollector(rf.id_list, rf.type_list, rf.box2d_list, method=method)
    col.add(res, data, first=0)
    return col.finalize(), rf


def _cascade(fd, fr, inp):
    first = fd.detect(*inp)
    call = int(fr.call.item())
    out = fr.refine(inp, first)
    return first, out, call


@pytest.mark.parametrize("wl", [("Car",), TYPES])
@pytest.mark.parametrize("method", ["nms", "top"])
@pytest.mark.parametrize("F", [1, 4])
def test_parity_with_the_offline_cascade(F, method, wl):
    from frustum_convnet_b200 import refine_extract as rx
    frames = _frames(300 + F, F, types=wl)
    fd, fr, inp = _pair(F, method, wl, frames=frames)
    first, out, _ = _cascade(fd, fr, inp)
    assert out.status_bits() == first.status_bits() == 0
    want, rf = _offline(fr, frames, first, out, wl, method)
    K = len(rf)
    assert K > 0 and int(out.valid.sum().item()) == K
    _same(out.to_dict(), want)
    # the kept set, its order and points against the dict path
    d = rx.RefineFrustumExtractor(wl).from_detections({f: x[0] for f, x in enumerate(frames)},
                                                      {f: x[1] for f, x in enumerate(frames)},
                                                      {f: x[2] for f, x in enumerate(frames)}, list(range(F)),
                                                      first.to_dict())
    M = int(fr.offsets[K].item())
    assert np.array_equal(d.counts, np.diff(fr.offsets[:K + 1].cpu().numpy()))
    assert torch.equal(d.offsets, fr.offsets[:K + 1]) and torch.equal(d.points, fr.points4[:M])
    assert d.id_list == rf.id_list and d.type_list == rf.type_list
    ang = np.array(d.frustum_angle_list)
    got = rf.frustum_angle.cpu().numpy()
    assert (np.abs(ang - got) <= 4 * np.spacing(np.maximum(np.abs(ang), np.abs(got)))).all()
    # no extra padding: W equal to the kept batch's own widest T gives the same rows
    T = [int(t) for t in np.array(rf.record_words[:, :len(fr.T)].cpu().numpy()).max(0)]
    fd2, fr2, inp2 = _pair(F, method, wl, frames=frames, sections=T)
    first2, out2, _ = _cascade(fd2, fr2, inp2)
    want2, _ = _offline(fr2, frames, first2, out2, wl, method)
    _same(out2.to_dict(), want2)


def test_device_draw_and_stage_one_draws_differ():
    fd, fr, inp = _pair(4, wl=TYPES, seed=(5 << 40) + 3)
    for rep in range(2):
        first, out, call = _cascade(fd, fr, inp)
        choice, off, slot = out.choice.cpu().numpy(), fr.offsets.cpu().numpy(), fr.job_index.cpu().numpy()
        assert call == -2 ** 63 + rep
        for b in range(fr.B):
            n = int(off[b + 1] - off[b])
            s = int(slot[b]) if slot[b] >= 0 else fr.B + b
            want = choice_row(n, fr.N, fr.seed, s, call + 2 ** 64)
            assert np.array_equal(choice[b], want), b
            assert not np.array_equal(want, choice_row(n, fr.N, fr.seed, s, rep)) or n <= 1


def _guarded(t):
    """A copy of t's buffer inside 4096-byte guards -> (whole uint8 buffer, the inner view's address)."""
    nbytes = t.numel() * t.element_size()
    g = torch.full((nbytes + 2 * GUARD,), 0xA5, dtype=torch.uint8, device=t.device)
    return g, g.data_ptr() + GUARD, nbytes


def _extract_guarded(fr):
    """fcn_frame_refine_extract into guarded copies of every output; asserts the guards hold -> {name: bytes}."""
    from frustum_convnet_b200 import _lib
    a = _lib.FrameRefineArgs.from_buffer_copy(fr._xa)
    outs = {"points": fr.points4, "offsets": fr.offsets, "job_index": fr.job_index, "valid": fr.valid,
            "cls_index": fr.cls_index, "seg": fr.seg, "seg_class_out": fr.seg_class, "records": fr.frustum_records,
            "box2d": fr.box2d32}
    bufs = {}
    for name, t in outs.items():
        g, p, n = _guarded(t)
        setattr(a, name, p)
        bufs[name] = (g, n)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    a.status = status.data_ptr()
    _lib.call("fcn_frame_refine_extract", C.byref(a), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for name, (g, n) in bufs.items():
        h = g.cpu().numpy()
        assert (h[:GUARD] == 0xA5).all() and (h[GUARD + n:] == 0xA5).all(), name
    return int(status.item())


def _job_rows(first, wl):
    """{frame: [the first-stage row of job j]} in the frame path's job order: the whitelisted segments in class-rank
    order, then their kept rows."""
    meta = torch.cat([first.seg_offsets, first.keep_count, first.seg_class.reshape(-1)]).cpu().numpy()
    F = first.seg_class.shape[0]
    off, kc, cls = meta[:3 * F + 1], meta[3 * F + 1:6 * F + 1], meta[6 * F + 1:]
    return {f: [i for s in range(3 * f, 3 * f + 3) if cls[s] >= 0 and TYPES[cls[s]] in wl
                for i in range(int(off[s]), int(off[s] + kc[s]))] for f in range(F)}


def _without_rows(first, drop):
    """first with the rows `drop` taken out of their segments: what the offline chain is fed to refine the frustums
    the frame path kept (it has no capacities, and it raises on a bad row)."""
    from frustum_convnet_b200.frame_detect import FrameDetections
    rows, kc = first.rows.clone(), first.keep_count.clone()
    off, kch = first.seg_offsets.cpu().numpy(), first.keep_count.cpu().numpy()
    for s in range(len(kch)):
        keep = [i for i in range(int(off[s]), int(off[s] + kch[s])) if i not in drop]
        if len(keep) < kch[s]:
            if keep:
                rows[int(off[s]):int(off[s]) + len(keep)] = first.rows[keep]
            kc[s] = len(keep)
    return FrameDetections(rows, first.seg_offsets, kc, first.seg_class, first.status, first.choice, first.valid)


def test_capacity_bits_keep_the_frames_that_fit():
    """Each extraction capacity exceeded by some frames of a call: the bit is set, the guards hold, and the refined rows
    equal the offline chain's on the same first-stage rows without the jobs the capacity dropped."""
    from frustum_convnet_b200 import _lib
    F, wl = 4, ("Car",)
    frames = _frames(311, F)
    fd, fr, inp = _pair(F, frames=frames)
    first, out, _ = _cascade(fd, fr, inp)
    assert out.status_bits() == 0
    base = out.to_dict()
    rows = int(fr.counter.item())                  # candidate rows of a first call (the draws depend on the call)
    jobs = _job_rows(first, wl)
    K = int(fr.valid.sum().item())
    slot = fr.job_index[:K].cpu().numpy()
    pts = np.diff(fr.offsets[:K + 1].cpu().numpy())
    entry_row = [jobs[int(d) // fr.J][int(d) % fr.J] for d in slot]
    _, rf = _offline(fr, frames, first, out, wl, "nms")
    T = rf.record_words[:, :len(fr.T)].cpu().numpy()

    def check(bit, drop, **kw):
        assert drop and len(drop) < sum(len(v) for v in jobs.values())       # some frustums drop, some fit
        fdx, frx, inpx = _pair(F, frames=frames, **kw)
        firstx = fdx.detect(*inpx)
        got = frx.refine(inpx, firstx)
        assert got.status_bits() == bit, kw
        want, rfx = _offline(frx, frames, _without_rows(firstx, drop), got, wl, "nms")
        assert len(rfx) > 0 and int(frx.valid.sum().item()) == len(rfx), kw
        _same(got.to_dict(), want)
        assert _extract_guarded(frx) == bit, kw

    # J: one job less than the busiest frame's; the frames with at most J rows fit
    n = {f: len(v) for f, v in jobs.items()}
    J = max(n.values()) - 1
    assert min(n.values()) <= J
    check(_lib.FRAME_JOBS, {r for f in jobs for r in jobs[f][J:]}, jobs=J)
    # P2_out: one point less than the fullest frame's kept points; that frame loses a suffix of its frustums
    frame = slot // fr.J
    per_frame = np.bincount(frame, weights=pts, minlength=F).astype(np.int64)
    budget = int(per_frame.max()) - 1
    drop, run = set(), {}
    for k in range(K):
        run[frame[k]] = run.get(frame[k], 0) + int(pts[k])
        if run[frame[k]] > budget:
            drop.add(entry_row[k])
    check(_lib.FRAME_OUT_POINTS, drop, frustum_points=budget)
    fdp, frp, inpp = _pair(F, frames=frames, frustum_points=budget + 1)     # filled exactly: nothing drops
    got = frp.refine(inpp, fdp.detect(*inpp))
    assert got.status_bits() == 0
    _same(got.to_dict(), base)
    # W: the widest frustums one section over the first scale's width
    W = [int(T[:, 0].max()) - 1]
    for _ in range(1, len(fr.T)):
        W.append((W[-1] + 1) // 2)                 # the model's section pyramid
    assert W[0] >= 1
    check(_lib.FRAME_SECTIONS, {entry_row[k] for k in range(K) if (T[k] > np.array(W)).any()}, sections=W)
    # R2: rows - 1, rows, rows + 1 of the refinement's candidate rows
    for R, bit in ((rows - 1, _lib.FRAME_ROWS), (rows, 0), (rows + 1, 0)):
        fdr, frr, inpr = _pair(F, frames=frames, rows=R)
        got = frr.refine(inpr, fdr.detect(*inpr))
        assert got.status_bits() == bit, R
        if bit == 0:
            _same(got.to_dict(), base)


@pytest.mark.parametrize("what", ["nan", "inf", "-inf", "zero_l", "flat_2d"])
def test_bad_rows_next_to_good_rows(what):
    from frustum_convnet_b200 import _lib
    frames = _frames(321, 2)
    fd, fr, inp = _pair(2, frames=frames)
    first = fd.detect(*inp)
    k = int(first.seg_offsets[0].item())
    assert int(first.keep_count[0].item()) >= 2
    col, val = {"nan": (4, float("nan")), "inf": (6, float("inf")), "-inf": (10, -float("inf")),
                "zero_l": (9, 0.0), "flat_2d": (3, None)}[what]
    if val is None:
        first.rows[k, 3] = first.rows[k, 1] + 1.0                  # ymax - ymin < 5: dropped, no bit
    else:
        first.rows[k, col] = val
    out = fr.refine(inp, first)
    bit = 0 if what == "flat_2d" else _lib.FRAME_BAD_DET
    assert out.status_bits() & _lib.FRAME_BAD_DET == bit
    job = fr.job_index[:int(fr.valid.sum().item())].cpu().numpy()
    assert 0 not in job.tolist()                                    # slot 0 (the bad row) is not refined
    # the frames that fit keep their parity with the offline chain (which raises on the bad row: drop it there)
    want, rf = _offline(fr, frames, _without_rows(first, {k}), out, ("Car",), "nms")
    _same(out.to_dict(), want)


def test_frames_without_refinement_jobs():
    """Frames whose first-stage rows are all of classes the refiner does not take, and frames with no detection, in
    the same call as frames that refine; then a call where no frame refines."""
    from oracle import kitti_scan_synth as ks
    mixed = _frames(331, 2, types=TYPES)
    people = _frames(332, 1, types=("Pedestrian", "Cyclist"))
    rng = np.random.default_rng(3)
    empty = (ks.kitti_scan(rng, mixed[0][1], [], 20000), mixed[0][1], mixed[0][2], [])
    frames = [mixed[0], people[0], empty, mixed[1]]
    fd, fr, inp = _pair(4, frames=frames, wl=TYPES, refine_wl=("Car",))
    first, out, _ = _cascade(fd, fr, inp)
    assert 1 in first.to_dict() and "Car" not in first.to_dict()[1]       # stage 1 kept rows of frame 1
    got = out.to_dict()
    assert set(got) <= {0, 3} and got
    assert out.status_bits() == first.status_bits()
    want, _ = _offline(fr, frames, first, out, ("Car",), "nms")
    _same(got, want)
    # no frame with a job: zero rows and only the first stage's bits
    frames = [people[0], empty]
    fd, fr, inp = _pair(2, frames=frames, wl=TYPES, refine_wl=("Car",))
    first, out, _ = _cascade(fd, fr, inp)
    assert first.to_dict() and out.to_dict() == {} and int(out.seg_offsets[-1].item()) == 0
    assert out.status_bits() == first.status_bits()
    assert int(fr.valid.sum().item()) == 0


def test_graph_replay_of_both_stages():
    fd, fr, inp = _pair(2, wl=TYPES)
    _cascade(fd, fr, inp)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = fr.refine(inp, fd.detect(*inp))
    torch.cuda.current_stream().wait_stream(s)
    for rep in range(3):
        fd.stage(inp, _frames(340 + rep, 2, types=TYPES))
        c1, c2 = fd.call.clone(), fr.call.clone()
        g.replay()
        got = out.to_dict()
        st = out.status_bits()
        fd.call.copy_(c1)
        fr.call.copy_(c2)
        eager = fr.refine(inp, fd.detect(*inp))
        assert eager.status_bits() == st
        _same(got, eager.to_dict())
        assert got, rep


def test_collected_evaluates_like_the_dict():
    from det_feed_sets import kitti_set
    from test_gpu_det_eval_feed import compare_kitti_results, kitti_gt
    frames = _frames(351, 4, types=TYPES)
    fd, fr, inp = _pair(4, frames=frames, wl=TYPES)
    first, out, _ = _cascade(fd, fr, inp)
    gts, _ = kitti_set(4, seed=5)
    ev = kitti_gt(list(range(4)), gts)
    for res in (first, out):
        d = res.to_dict()
        assert d
        compare_kitti_results(ev.evaluate_collected(res.collected()), ev.evaluate(d))
