"""GPU: the single-frame detection stages of C ABI section (21), each called directly, against plain restatements at
their capacity and sampling edges.

  fcn_resample_choice        bit for bit against tests/resample_ref.py for N in {1, 7, 255, 256, 257, 1024, 2047,
                             2048} and n from 0 to 300 000 (n = N - 1, N, N + 1, 2N, ...) in one launch, a seed and a
                             call counter with their high words set, dummy entries (slot B + b);
  fcn_frame_extract          every table equal to tests/frame_ref.py (the angle within 2 ulp, everything else
                             bit for bit), the status bits exactly, the 4096-byte guards intact: counts past and below
                             the capacities, bad detections, every class mask, P_out filled exactly, one point over,
                             a large first frustum, classes dropped whole, F and F * D past one 1024-thread scan;
  fcn_det_candidates_valid,  against fcn_det_candidates + fcn_det_prepare + fcn_det_select on the valid entries alone:
  fcn_det_finalize_capacity  rows, offsets and keep counts bit for bit when R >= the row count, bit 8 and bounded
                             keep counts when R is one short;
  FrameDetector              frames over P_out equal the offline chain on the frustums they kept, and the inputs built
                             for the dummy entries equal oracle/input_builder within one float32 ulp."""
import ctypes as C

import numpy as np
import pytest
import torch

import frame_ref as fr
from resample_ref import choice_row
from test_gpu_frame_detect import TYPES, _frames, _guarded, _guards_hold, _model, _offline, _same

pytestmark = pytest.mark.gpu

PAT = 0xA5


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(x, dtype):
    return torch.from_numpy(np.ascontiguousarray(x)).to(device="cuda", dtype=dtype)


# ---------------------------------------------------------------------------------------------------- resampling
def _resample(ns, det_index, N, seed, call):
    from frustum_convnet_b200 import _lib
    B = len(ns)
    off = _dev(np.concatenate([[0], np.cumsum(ns)]), torch.int32)
    det = _dev(np.asarray(det_index), torch.int32)
    callt = torch.tensor([call], dtype=torch.int64, device="cuda")
    buf, choice = _guarded((B, N), torch.int32, PAT)
    r = _lib.ResampleArgs()
    r.B, r.N, r.seed = B, N, seed
    r.offsets, r.det_index, r.call, r.choice = off.data_ptr(), det.data_ptr(), callt.data_ptr(), choice.data_ptr()
    _lib.call("fcn_resample_choice", C.byref(r), _stream())
    torch.cuda.synchronize()
    assert _guards_hold(buf, PAT)
    return choice.cpu().numpy()


@pytest.mark.parametrize("N", [1, 7, 255, 256, 257, 1024, 2047, 2048])
def test_resample_choice_equals_the_restatement(N):
    seed, call = (0x9E3779B9 << 32) | 0x1234567, (0xC0FFEE << 32) | 41
    ns = [0, 1, N - 1, N, N + 1, 2 * N, 2049, 65536, 300000]
    det = [3 * b + 1 if b % 2 == 0 else -1 for b in range(len(ns))]
    B = len(ns)
    got = _resample(ns, det, N, seed, call)
    for b, n in enumerate(ns):
        slot = det[b] if det[b] >= 0 else B + b
        assert np.array_equal(got[b], choice_row(n, N, seed, slot, call)), (b, n)
        if n >= N:
            assert len(np.unique(got[b])) == N and got[b].min() >= 0 and got[b].max() < n, (b, n)
        if n == N:
            assert np.array_equal(np.sort(got[b]), np.arange(N)), b
        if 0 < n < N:
            assert got[b].min() >= 0 and got[b].max() < n, (b, n)
    assert not got[0].any()
    # the dummy slot B + b is not slot b: the same n under a real slot draws differently
    if N >= 7:
        assert not np.array_equal(got[5], choice_row(ns[5], N, seed, 5, call))


def test_resample_choice_refuses_n_outside_1_to_2048():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    x = torch.zeros(8, dtype=torch.int64, device="cuda")
    r = _lib.ResampleArgs()
    r.B, r.seed = 1, 1
    r.offsets = r.det_index = r.call = r.choice = x.data_ptr()
    for N in (0, 2049):
        r.N = N
        assert lib.fcn_resample_choice(C.byref(r), None) == -1
        assert b"bad sizes" in lib.fcn_last_error()
    torch.cuda.synchronize()
    assert not x.any()


# ---------------------------------------------------------------------------------------------------- extraction
def _frame_buffer(calibs, hw):
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200.frustum_extract import _frame_record
    recs = (_lib.FrustumFrame * len(calibs))(*[_frame_record(c, h) for c, h in zip(calibs, hw)])
    return torch.frombuffer(bytearray(bytes(recs)), dtype=torch.uint8).cuda()


def _frame_extract(inp, P_out, class_mask):
    """fcn_frame_extract on the staged inputs -> ({output name: host array}, status); every output guarded."""
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200._host import workspace
    scans, sc, calibs, hw, boxes, cls, prob, dc = inp
    F, P = scans.shape[:2]
    D = boxes.shape[1]
    B = F * D
    keep = [_dev(scans, torch.float32), _dev(sc, torch.int32), _frame_buffer(calibs, hw), _dev(boxes, torch.float64),
            _dev(cls, torch.int32), _dev(prob, torch.float32), _dev(dc, torch.int32)]
    a = _lib.FrameExtractArgs()
    a.num_frames, a.scan_capacity, a.det_capacity, a.out_capacity, a.class_mask = F, P, D, P_out, class_mask
    (a.scans, a.scan_counts, a.frames, a.boxes, a.det_class, a.det_prob, a.det_counts) = (t.data_ptr() for t in keep)
    outs = {"points": ((F * P_out + B, 4), torch.float32), "offsets": ((B + 1,), torch.int32),
            "frustum_angle": ((B,), torch.float64), "box2d": ((B, 4), torch.float64), "P": ((B, 12), torch.float64),
            "det_index": ((B,), torch.int32), "valid": ((B,), torch.int32), "cls_index": ((B,), torch.int32),
            "seg": ((B,), torch.int32), "seg_class": ((F, 3), torch.int32), "rgb_prob": ((B,), torch.float32),
            "status": ((1,), torch.int32)}
    held = {}
    for name, (shape, dt) in outs.items():
        buf, t = _guarded(shape, dt, PAT)
        if name == "status":
            t.zero_()
        held[name] = (buf, t)
        setattr(a, name, t.data_ptr())
    ws, a.workspace_bytes = workspace("fcn_frame_extract_workspace_bytes", "cuda", C.byref(a))
    a.workspace = ws.data_ptr()
    _lib.call("fcn_frame_extract", C.byref(a), _stream())
    torch.cuda.synchronize()
    for name, (buf, _) in held.items():
        assert _guards_hold(buf, PAT), name
    got = {name: t.cpu().numpy() for name, (_, t) in held.items()}
    return got, int(got.pop("status")[0])


def _check_tables(inp, P_out, class_mask=7):
    """Device tables == frame_ref's; -> the restatement's tables."""
    want = fr.frame_tables(*inp, P_out=P_out, class_mask=class_mask)
    got, status = _frame_extract(inp, P_out, class_mask)
    assert status == want["status"], (status, want["status"])
    for name in ("offsets", "det_index", "valid", "cls_index", "seg", "seg_class"):
        assert np.array_equal(got[name], want[name]), name
    M = int(want["offsets"][-1])
    for name, g in (("points", got["points"][:M]), ("box2d", got["box2d"]), ("P", got["P"]),
                    ("rgb_prob", got["rgb_prob"])):
        assert g.tobytes() == np.ascontiguousarray(want[name]).tobytes(), name
    ang, ref = got["frustum_angle"], want["frustum_angle"]
    assert np.all(np.abs(ang - ref) <= 2 * np.spacing(np.abs(ref))), np.max(np.abs(ang - ref))
    return want


def _classes(dp, cls, D):
    """Per frame: the classes of its count-pass survivors."""
    return [set(int(c) for c, p in zip(cls[f], dp[f * D:(f + 1) * D]) if p >= 0) for f in range(len(cls))]


@pytest.mark.parametrize("class_mask", range(8))
def test_frame_extract_counts_bad_detections_and_class_masks(class_mask):
    """Scan counts 0, 1, P, P + 1, -1 and P; detection counts D, D, D + 1, D, D and -1; a bad class, a NaN and
    +-inf boxes next to good detections of the same frames."""
    P, D = 1500, 4
    frames = fr.synth_frames(np.random.default_rng(20), 6, 1700, 5)
    scans, sc, calibs, hw, boxes, cls, prob, dc = fr.stage(frames, P, D, scan_counts=[0, 1, P, P + 1, -1, P],
                                                           det_counts=[D, D, D + 1, D, D, -1])
    cls[2, 1], cls[3, 0] = 3, -2
    boxes[2, 3, 0], boxes[3, 2, 2], boxes[5, 0, 1] = np.nan, np.inf, -np.inf    # slot (5, 0) is past det_counts
    inp = (scans, sc, calibs, hw, boxes, cls, prob, dc)
    want = _check_tables(inp, P, class_mask)
    assert want["status"] & (fr.SCAN_POINTS | fr.DETS | fr.BAD_DET) == fr.SCAN_POINTS | fr.DETS | fr.BAD_DET
    if class_mask == 7:
        kept = want["det_index"][want["valid"] == 1] // D
        assert set(kept.tolist()) >= {2, 3} and not set(kept.tolist()) & {0, 4, 5}


@pytest.mark.parametrize("F", [1, 3])
def test_frame_extract_budgets(F):
    """P_out filled exactly, one point over, a first frustum larger than P_out (every later one drops with it) and a
    budget that drops every frustum of a class: each against the restatement."""
    P, D = 6000, 4
    frames = fr.synth_frames(np.random.default_rng(30 + F), F, 6000, D)
    inp = fr.stage(frames, P, D)
    cls = inp[5]
    dp = fr.frame_tables(*inp, P_out=1 << 20)["det_points"].reshape(F, D)
    totals = [int(r[r >= 0].sum()) for r in dp]
    firsts = [int(r[r >= 0][0]) for r in dp]
    assert min(firsts) > 0 and all(len(set(c)) == 3 for c in cls.tolist())
    # filled exactly: the fullest frame's kept frustums take exactly P_out points
    want = _check_tables(inp, max(totals))
    assert want["status"] & fr.OUT_POINTS == 0 and int(want["valid"].sum()) == int((dp >= 0).sum())
    # one point over: that frame's last kept frustum drops
    want = _check_tables(inp, max(totals) - 1)
    assert want["status"] & fr.OUT_POINTS and int(want["valid"].sum()) == int((dp >= 0).sum()) - 1
    # a first frustum larger than P_out: its frame keeps nothing
    want = _check_tables(inp, max(firsts) - 1)
    f_big = int(np.argmax(firsts))
    assert want["status"] & fr.OUT_POINTS and not np.any(want["det_index"] // D == f_big)
    assert (want["seg_class"][f_big] == -1).all()
    # every frame keeps its first frustum alone when P_out fits it and not the next: the later classes get no segment
    budget = max(firsts)
    want = _check_tables(inp, budget)
    kept = want["det_index"][want["valid"] == 1]
    before = _classes(dp.reshape(-1), cls, D)
    after = [set(int(cls[f, d % D]) for d in kept if d // D == f) for f in range(F)]
    assert any(a < b for a, b in zip(after, before))
    for f in range(F):
        assert sorted(c for c in want["seg_class"][f] if c >= 0) == sorted(after[f])


@pytest.mark.parametrize("F,D,P,n_points", [(1100, 1, 64, 64), (130, 8, 2048, 3000), (4, 600, 8192, 8192)])
def test_frame_extract_past_one_block_scan(F, D, P, n_points):
    """F > 1024 (frame_setup's frame loop) and F * D past 1024 and 2048 (frame_slots' slot loop)."""
    frames = fr.synth_frames(np.random.default_rng(F + D), F, n_points, D)
    inp = fr.stage(frames, P, D)
    want = _check_tables(inp, P_out=P // 2)
    K = int(want["valid"].sum())
    assert 0 < K < F * D


# ---------------------------------------------------------------------------------------------------- detection rows
# frustum -> segment: segment s holds SEG_FRUSTUMS[s] frustums (shuffled over the batch); one foreground position per
# frustum except FG_SPECIAL (frustum index within its segment -> foreground positions), so under 'nms' the segments
# hold 0, 1, 31, 32, 33, 70, 1 (an all-background frustum's fallback row) and 100 rows, under 'top' one row a frustum
SEG_FRUSTUMS = [0, 1, 31, 32, 33, 70, 1, 5]
FG_SPECIAL = {6: [0], 7: [20] * 5}


def _det_batch(workload, seed):
    from frustum_convnet_b200 import synth
    model = _model(workload)
    rng = np.random.default_rng(seed)
    B = sum(SEG_FRUSTUMS)
    data = {k: torch.from_numpy(v).cuda() for k, v in synth.make_frustums(workload, B, seed=seed).items()}
    with torch.no_grad():
        out = model(data)
    cls_probs, center, heading, size, _, size_probs = out
    T2 = int(cls_probs.shape[1])
    f32 = lambda t: t.detach().float().contiguous()
    size, center, heading, size_probs = f32(size), f32(center), f32(heading).reshape(B, T2), f32(size_probs)
    seg = np.concatenate([[s] * n for s, n in enumerate(SEG_FRUSTUMS)]).astype(np.int32)
    seg = seg[rng.permutation(B)]
    sz = size.cpu().numpy()
    ok = ~((sz < np.float32(0.01)).any(axis=2))                      # det_size_ok
    p = np.stack([np.full((B, T2), 0.6, np.float32), (0.4 - 0.3 * rng.random((B, T2))).astype(np.float32)], 2)
    within = {}
    for b in range(B):
        k = within.setdefault(seg[b], 0)
        within[seg[b]] = k + 1
        n_fg = FG_SPECIAL[seg[b]][k] if seg[b] in FG_SPECIAL else 1
        cand = np.flatnonzero(ok[b])
        assert len(cand) >= max(n_fg, 1)
        pick = rng.choice(cand, max(n_fg, 1), replace=False)
        if n_fg == 0:
            p[b, pick[0], 1] = 0.45                                  # the argmax, still background
        else:
            p[b, pick, 0] = 0.3
            p[b, pick, 1] = (0.5 + 0.5 * rng.random(n_fg)).astype(np.float32)
    tens = {"cls_probs": _dev(p, torch.float32), "center": center, "heading": heading, "size": size,
            "size_probs": size_probs,
            "rot_angle": _dev(rng.uniform(-np.pi, np.pi, B), torch.float32),
            "rgb_prob": _dev(rng.random(B), torch.float32),
            "box2d": _dev(rng.uniform(0, 1000, (B, 4)), torch.float32),
            "seg": _dev(seg, torch.int32)}
    return tens, B, T2, int(size_probs.shape[-1])


def _cand_args(t, B, T2, NS, method, capacity, counter, records):
    from frustum_convnet_b200 import _lib
    a = _lib.DetCandidateArgs()
    a.B, a.T2, a.NS, a.dataset, a.method = B, T2, NS, 0, method
    a.first, a.num_frustums, a.capacity = 0, B, capacity
    a.cls_probs, a.center, a.heading, a.size, a.size_probs = (t[k].data_ptr() for k in
                                                              ("cls_probs", "center", "heading", "size", "size_probs"))
    a.rot_angle, a.rgb_prob, a.ref_center = t["rot_angle"].data_ptr(), t["rgb_prob"].data_ptr(), None
    a.seg_of_frustum, a.counter, a.records = t["seg"].data_ptr(), counter.data_ptr(), records.data_ptr()
    return a


def _fin_args(t, S, B, capacity, method, counter, records, ws, nbytes, info, off, kc, rows):
    from frustum_convnet_b200 import _lib
    fa = _lib.DetFinalizeArgs()
    fa.num_segments, fa.num_frustums, fa.capacity, fa.method, fa.dataset = S, B, capacity, method, 0
    fa.top_k, fa.thresh = 300, 0.1
    fa.counter, fa.records, fa.box2d = counter.data_ptr(), records.data_ptr(), t["box2d"].data_ptr()
    fa.workspace, fa.workspace_bytes, fa.info = ws.data_ptr(), nbytes, info.data_ptr()
    fa.seg_offsets, fa.keep_count, fa.rows = off.data_ptr(), kc.data_ptr(), rows.data_ptr()
    return fa


def _offline_rows(t, idx, T2, NS, S, method):
    """fcn_det_candidates + fcn_det_prepare + fcn_det_select on the entries idx alone -> (rows produced, seg_offsets,
    keep_count, rows)."""
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200._host import workspace
    K = len(idx)
    ix = torch.from_numpy(idx).long().cuda()
    sub = {k: (v.index_select(0, ix).contiguous() if K else v[:1].contiguous()) for k, v in t.items()}
    cap = max(K * T2, 1)
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    records = torch.empty((cap, 12), dtype=torch.int32, device="cuda")
    a = _cand_args(sub, K, T2, NS, method, cap, counter, records)
    _lib.call("fcn_det_candidates", C.byref(a), _stream())
    ws, nbytes = workspace("fcn_det_workspace_bytes", "cuda", cap, S)
    info = torch.zeros(4, dtype=torch.int64, device="cuda")
    off = torch.zeros(S + 1, dtype=torch.int32, device="cuda")
    kc = torch.zeros(S, dtype=torch.int32, device="cuda")
    rows = torch.zeros((cap, 12), dtype=torch.float32, device="cuda")
    fa = _fin_args(sub, S, max(K, 1), cap, method, counter, records, ws, nbytes, info, off, kc, rows)
    _lib.call("fcn_det_prepare", C.byref(fa), _stream())
    n, mask_words = (int(v) for v in info[:2].tolist())
    mask = torch.empty(max(mask_words, 1), dtype=torch.int32, device="cuda")
    fa.n_counted, fa.mask, fa.mask_words = n, mask.data_ptr(), mask_words
    _lib.call("fcn_det_select", C.byref(fa), _stream())
    return n, off.cpu().numpy(), kc.cpu().numpy(), rows.cpu().numpy()


def _capacity_rows(t, valid, B, T2, NS, S, method, R):
    """fcn_det_candidates_valid + fcn_det_finalize_capacity over all B entries with capacity R, every output guarded
    -> (seg_offsets, keep_count, rows, status)."""
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200._host import workspace
    counter = torch.zeros(1, dtype=torch.int32, device="cuda")
    m = min(R, T2 * max(SEG_FRUSTUMS))                 # the most rows one segment can hold
    shapes = {"records": ((R, 12), torch.int32), "info": ((4,), torch.int64), "off": ((S + 1,), torch.int32),
              "kc": ((S,), torch.int32), "rows": ((R, 12), torch.float32),
              "mask": ((R * ((m + 31) // 32),), torch.int32), "status": ((1,), torch.int32)}
    held = {k: _guarded(s, dt, PAT) for k, (s, dt) in shapes.items()}
    g = {k: v[1] for k, v in held.items()}
    g["status"].zero_()
    a = _cand_args(t, B, T2, NS, method, R, counter, g["records"])
    _lib.call("fcn_det_candidates_valid", C.byref(a), valid.data_ptr(), _stream())
    ws, nbytes = workspace("fcn_det_workspace_bytes", "cuda", R, S)
    fa = _fin_args(t, S, B, R, method, counter, g["records"], ws, nbytes, g["info"], g["off"], g["kc"], g["rows"])
    fa.mask, fa.mask_words = g["mask"].data_ptr(), g["mask"].numel()
    _lib.call("fcn_det_finalize_capacity", C.byref(fa), g["status"].data_ptr(), _stream())
    torch.cuda.synchronize()
    for k, (buf, _) in held.items():
        assert _guards_hold(buf, PAT), k
    return g["off"].cpu().numpy(), g["kc"].cpu().numpy(), g["rows"].cpu().numpy(), int(g["status"].item())


@pytest.mark.parametrize("workload", ["car", "people"])
@pytest.mark.parametrize("method", ["nms", "top"])
def test_capacity_candidates_and_finalize_equal_the_valid_entries_alone(workload, method):
    t, B, T2, NS = _det_batch(workload, 61 if workload == "car" else 62)
    S, mth = len(SEG_FRUSTUMS), 0 if method == "nms" else 1
    patterns = {"all": np.ones(B, np.int32), "none": np.zeros(B, np.int32),
                "alternating": (np.arange(B) % 2 == 0).astype(np.int32),
                "last": (np.arange(B) == B - 1).astype(np.int32)}
    for name, v in patterns.items():
        n, off, kc, rows = _offline_rows(t, np.flatnonzero(v), T2, NS, S, mth)
        sizes = np.diff(off)
        if name == "all":
            want = [0, 1, 31, 32, 33, 70, 1, 100] if method == "nms" else SEG_FRUSTUMS
            assert sizes.tolist() == want
            if method == "nms":
                assert (kc < sizes).any()                           # the NMS suppressed something
        valid = _dev(v, torch.int32)
        for R in sorted({max(n - 1, 1), max(n, 1), n + 1}):
            g_off, g_kc, g_rows, status = _capacity_rows(t, valid, B, T2, NS, S, mth, R)
            if R >= n:
                assert status == 0, (name, R)
                assert np.array_equal(g_off, off) and np.array_equal(g_kc, kc), (name, R)
                for s in range(S):
                    a, b = off[s], off[s] + kc[s]
                    assert g_rows[a:b].tobytes() == rows[a:b].tobytes(), (name, R, s)
            else:
                assert status == 8, (name, R)
                assert g_off[0] == 0 and g_off[-1] == R and (np.diff(g_off) >= 0).all(), (name, R)
                assert (g_kc >= 0).all() and (g_kc <= np.diff(g_off)).all(), (name, R)


# ---------------------------------------------------------------------------------------------------- FrameDetector
def _staged(frames, D):
    """_frames' frames in frame_ref's staging (class indices)."""
    return fr.stage([(s, c, hw, [(TYPES.index(t), p, b) for t, p, b in dets]) for s, c, hw, dets in frames],
                    max(len(x[0]) for x in frames), D)


@pytest.mark.parametrize("method", ["nms", "top"])
def test_over_budget_frames_equal_the_offline_chain_on_their_kept_frustums(method):
    """P_out keeps each frame's first frustum and drops some later ones, whole classes among them (bit 4): the rows
    equal the offline chain's on the kept frustums alone, fed the same choice rows, and a class whose frustums were
    all dropped has no entry."""
    from frustum_convnet_b200.frame_detect import FrameDetector
    model = _model("car")
    F, D = 3, 8
    frames = _frames(43, F)
    inp = _staged(frames, D)
    dp = fr.frame_tables(*inp, P_out=1 << 20)["det_points"].reshape(F, D)
    P_out = max(int(r[r >= 0][0]) for r in dp)
    want_t = fr.frame_tables(*inp, P_out=P_out)
    assert want_t["status"] == fr.OUT_POINTS
    fd = FrameDetector(model, TYPES, method=method, seed=11, frames=F, points=120000, dets=D, frustum_points=P_out)
    finp = fd.inputs()
    fd.stage(finp, frames)
    out = fd.detect(*finp)
    got = out.to_dict()
    assert out.status_bits() == fr.OUT_POINTS
    kept = fd.det_index.cpu().numpy()[:int(out.valid.sum().item())]
    assert np.array_equal(kept, want_t["det_index"][want_t["valid"] == 1])
    sub = [(s, c, hw, [d for j, d in enumerate(dets) if f * D + j in set(kept.tolist())])
           for f, (s, c, hw, dets) in enumerate(frames)]
    want, K = _offline(model, sub, TYPES, method, out.choice)
    assert K == len(kept)
    _same(got, want)
    before = _classes(dp.reshape(-1), inp[5], D)
    assert any(len(got.get(f, {})) < len(before[f]) for f in range(F))


def test_inputs_built_for_dummy_entries_equal_the_oracle():
    """fcn_build_inputs on a frame batch with dummy entries (one point at the origin, box (0, 0, 1, 1), a unit P)
    gives oracle/input_builder's values within one float32 ulp, all finite."""
    from frustum_convnet_b200.frame_detect import FrameDetector
    from oracle.input_builder import build_inputs
    model = _model("car")
    fd = FrameDetector(model, ("Car",), seed=2, frames=2, points=120000, dets=8)
    inp = fd.inputs()
    fd.stage(inp, _frames(44, 2))
    fd.detect(*inp)
    torch.cuda.synchronize()
    off = fd.offsets.cpu().numpy()
    K, B = int(fd.valid.sum().item()), fd.B
    assert 0 < K < B
    got = {k: v.cpu().numpy() for k, v in fd.fb.out.items()}
    ref = build_inputs(fd.points3.cpu().numpy()[:off[-1]], off, fd.choice.cpu().numpy(), fd.angle.cpu().numpy(),
                       fd.box2d.cpu().numpy(), fd.Pm.cpu().numpy().reshape(B, 3, 4), fd.fb.strides, fd.fb.max_depth,
                       cls_index=fd.cls_index.cpu().numpy())
    for k, r in ref.items():
        g = got[k]
        assert g.shape == r.shape and np.isfinite(g).all(), k
        x, y = g.astype(np.float64), r.astype(np.float64)
        assert np.all(np.abs(x - y) <= np.spacing(np.maximum(np.abs(g), np.abs(r))).astype(np.float64)), k
