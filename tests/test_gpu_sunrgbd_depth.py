"""GPU: fcn_sunrgbd_depth_cloud (C ABI section (24)) against the reference's own read_3d_points
(tests/golden/sunrgbd_depth.npz) and oracle/sunrgbd_depth.py, bit for bit with point order and counts, every output
inside guard bands; its overflow and crop bits; and the two paths it feeds: SunrgbdFrameDetector.detect_depth against
detect() on oracle-built clouds (eager and from a captured graph), and depth_clouds into the offline extractor."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden", "sunrgbd_depth.npz")
GUARD = 1024                       # elements of sentinel before and after every output
SENTINEL = np.int32(0x7FA5A5A5)    # a NaN pattern no conversion writes


def _golden_frames():
    z = np.load(GOLDEN)
    return [(z["depth_" + c], z["rgb_" + c], z["calib_" + c], z["ref_" + c]) for c in (str(c) for c in z["cases"])]


def _guarded(n, dtype):
    """A sentinel-filled device buffer with GUARD elements either side of n -> (whole buffer, the n-element view)."""
    whole = torch.full((n + 2 * GUARD,), int(SENTINEL), dtype=torch.int32, device="cuda")
    view = whole[GUARD:GUARD + n]
    return whole, view if dtype == torch.int32 else view.view(dtype)


def _convert(frames, H, W, P, rgb=True, hw=None):
    """One device call over frames [(depth, rgb, calib), ...] zero-padded to H x W -> (clouds (F, P, 6) as int32
    bits, counts, status, the guard bands intact)."""
    from frustum_convnet_b200.sunrgbd_depth import DepthCloudStage
    F = len(frames)
    h_depth, h_rgb = np.zeros((F, H, W), np.uint16), np.zeros((F, H, W, 3), np.uint8)
    h_hw = np.zeros((F, 2), np.int32)
    for f, (d, c, _) in enumerate(frames):
        h, w = min(d.shape[0], H), min(d.shape[1], W)
        h_depth[f, :h, :w], h_rgb[f, :h, :w], h_hw[f] = d[:h, :w], c[:h, :w], d.shape
    if hw is not None:
        h_hw[:] = hw
    dev = torch.device("cuda")
    st = DepthCloudStage(F, H, W, P, dev)
    depth = torch.from_numpy(h_depth.view(np.int16)).cuda().view(torch.uint16)
    rgbt = torch.from_numpy(h_rgb).cuda() if rgb else None
    cal = torch.from_numpy(np.stack([c for _, _, c in frames])).cuda()
    cw, clouds = _guarded(F * P * 6, torch.float32)
    nw, counts = _guarded(F, torch.int32)
    sw, status = _guarded(1, torch.int32)
    status.zero_()
    hwt = torch.from_numpy(h_hw).cuda()
    st.check("test", depth, rgbt, hwt, cal)
    st.run(depth, rgbt, hwt, cal, clouds.view(F, P, 6), counts, status, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for whole in (cw, nw, sw):
        g = whole.cpu().numpy()
        assert (g[:GUARD] == SENTINEL).all() and (g[-GUARD:] == SENTINEL).all()
    return clouds.view(torch.int32).view(F, P, 6).cpu().numpy(), counts.cpu().numpy(), int(status.item())


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def _oracle(frames, H, W, P, rgb=True, hw=None):
    from oracle import sunrgbd_depth as osd
    out = []
    for f, (d, c, cal) in enumerate(frames):
        size = d.shape if hw is None else hw[f]
        pad = np.zeros((H, W), np.uint16)
        padc = np.zeros((H, W, 3), np.uint8)
        h, w = min(d.shape[0], H), min(d.shape[1], W)
        pad[:h, :w], padc[:h, :w] = d[:h, :w], c[:h, :w]
        out.append(osd.frame_cloud(pad, padc if rgb else None, size, cal, H, W, P))
    return out


def _check(got, want, P):
    clouds, counts, status = got
    bits = 0
    for f, (cloud, n, b) in enumerate(want):
        k = min(n, P)
        assert counts[f] == k, f
        assert np.array_equal(clouds[f, :k], _bits(cloud)), f
        assert (clouds[f, k:] == SENTINEL).all(), f           # rows past the count are not written
        bits |= b
    assert status == bits


def test_golden_frames_of_different_sizes_in_one_call():
    gold = _golden_frames()
    frames = [(d, c, cal) for d, c, cal, _ in gold]
    H, W = max(d.shape[0] for d, *_ in gold), max(d.shape[1] for d, *_ in gold)
    got = _convert(frames, H, W, H * W)
    for f, (d, c, cal, ref) in enumerate(gold):
        n = len(ref)
        assert got[1][f] == n
        assert np.array_equal(got[0][f, :n], _bits(ref.astype(np.float32))), f
    _check(got, _oracle(frames, H, W, H * W), H * W)
    assert got[2] == 0


def test_rgb_null_gives_the_same_xyz_and_zero_colour():
    gold = _golden_frames()
    frames = [(d, c, cal) for d, c, cal, _ in gold]
    H, W = 23, 31
    a, b = _convert(frames, H, W, H * W), _convert(frames, H, W, H * W, rgb=False)
    assert np.array_equal(a[1], b[1])
    for f, n in enumerate(a[1]):
        assert np.array_equal(a[0][f, :n, :3], b[0][f, :n, :3])
        assert (b[0][f, :n, 3:] == 0).all()
    _check(b, _oracle(frames, H, W, H * W, rgb=False), H * W)


def _scene(seed, H, W, hole=0.1):
    """A synthetic depth frame: a tilted floor-to-wall ramp with boxes in front, `hole` of its pixels 0."""
    from oracle.make_golden_sunrgbd_depth import calibs, rot_left3
    rng = np.random.default_rng(seed)
    v, u = np.mgrid[0:H, 0:W]
    d = 2.0 + 4.0 * (1 - v / H) + 0.5 * np.sin(u / 37.0)
    boxes = []
    for _ in range(6):
        h, w = rng.integers(20, min(90, H // 2, W // 2), 2)
        y0, x0 = rng.integers(0, H - h), rng.integers(0, W - w)
        d[y0:y0 + h, x0:x0 + w] = rng.uniform(1.0, 3.0)
        boxes.append(np.array([x0, y0, x0 + w, y0 + h], np.float64))
    raw = rot_left3(np.clip(np.round(d * 1000), 1, 65535).astype(np.int64))
    raw[rng.random((H, W)) < hole] = 0
    rgb = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    R, K = calibs()[seed % 2]
    K = K.copy()
    K[0, 2], K[1, 2] = W / 2 + 0.375, H / 2 - 0.625
    return raw, rgb, np.concatenate([R.reshape(-1), K.reshape(-1)]), boxes


def test_full_size_frames_match_the_oracle():
    H, W = 530, 730
    frames = [_scene(s, H, W)[:3] for s in range(3)]
    frames[2] = (frames[2][0][:400, :600], frames[2][1][:400, :600], frames[2][2])
    got = _convert(frames, H, W, H * W)
    _check(got, _oracle(frames, H, W, H * W), H * W)


def test_overflow_and_crop_set_their_bits():
    H, W = 60, 80
    frames = [_scene(s, 64, 90)[:3] for s in range(4)]
    from oracle import sunrgbd_depth as osd
    n0 = len(osd.depth_cloud(frames[0][0][:H, :W], None, frames[0][2][:9].reshape(3, 3),
                             frames[0][2][9:].reshape(3, 3)))
    P = n0 - 37                                             # frame 0 (and the others) overflow P
    hw = np.array([[H, W], [64, 90], [H, W + 1], [-3, W]], np.int32)
    got = _convert(frames, H, W, P, hw=hw)
    want = _oracle(frames, H, W, P, hw=hw)
    assert want[0][2] == 1 and want[1][2] & 128 and want[2][2] & 128 and want[3][1:] == (0, 0)
    _check(got, want, P)
    got = _convert(frames[:1], H, W, n0, hw=hw[:1])           # exactly P: no bit
    assert got[1][0] == n0 and got[2] == 0


# ---------------------------------------------------------------------------------------------- the detector
NAMES = ("chair", "table", "bed", "sofa", "desk", "lamp", "toilet", "dresser")


def _depth_frames(seed, F, H, W):
    out = []
    rng = np.random.default_rng(seed)
    for f in range(F):
        raw, rgb, cal, boxes = _scene(seed * 10 + f, H, W)
        dets = [(NAMES[(f + j) % len(NAMES)], float(np.float32(rng.uniform(0.1, 1.0))), b)
                for j, b in enumerate(boxes)]
        c = (boxes[0][:2] + boxes[0][2:]) / 2                 # one frustum under the cap
        dets.append(("chair", 0.5, np.concatenate([c - 12, c + 12])))
        out.append((raw, rgb if f % 2 == 0 else None, cal, dets))
    return out


def _cloud_frames(frames):
    from oracle import sunrgbd_depth as osd
    return [(osd.depth_cloud(d, c, cal[:9].reshape(3, 3), cal[9:].reshape(3, 3)),
             {"Rtilt": cal[:9].reshape(3, 3), "K": cal[9:].reshape(3, 3)}, dets) for d, c, cal, dets in frames]


def _depth_stage(frames):
    return [(d, c, {"Rtilt": cal[:9].reshape(3, 3), "K": cal[9:].reshape(3, 3)}, dets) for d, c, cal, dets in frames]


def _snapshot(out):
    n = int(out.seg_offsets[-1].item())
    return {"rows": out.rows[:n].cpu(), "seg_offsets": out.seg_offsets.cpu(), "keep_count": out.keep_count.cpu(),
            "seg_class": out.seg_class.cpu(), "status": out.status.cpu(), "choice": out.choice.cpu(),
            "cap_choice": out.cap_choice.cpu(), "valid": out.valid.cpu()}


def _same(a, b):
    for k in a:
        assert torch.equal(a[k], b[k]), k


@pytest.fixture(scope="module")
def model():
    from frustum_convnet_b200 import config
    from train_ref import make_model
    config.load_workload("sunrgbd")
    return make_model("sunrgbd", 5).eval()


def _detector(model, F, H, W):
    from frustum_convnet_b200.frame_detect import SunrgbdFrameDetector
    return SunrgbdFrameDetector(model, frames=F, points=H * W, dets=8, seed=13)


@pytest.mark.parametrize("F", [1, 3])
def test_detect_depth_equals_detect_on_oracle_clouds(model, F):
    H, W = 240, 320
    frames = _depth_frames(F, F, H, W)
    fa, fb = _detector(model, F, H, W), _detector(model, F, H, W)
    inp = fa.inputs_depth(H, W)
    fa.stage_depth(inp, _depth_stage(frames))
    a = _snapshot(fa.detect_depth(*inp))
    cin = fb.inputs()
    fb.stage(cin, _cloud_frames(frames))
    b = _snapshot(fb.detect(*cin))
    _same(a, b)
    assert int(a["keep_count"].sum()) > 0 and (a["cap_choice"] != 0).any()     # rows kept and the cap drawn
    assert int(fa.call.item()) == int(fb.call.item()) == 1


def test_detect_depth_without_rgb_buffers_and_with_overflow(model):
    H, W = 120, 160
    frames = _depth_frames(7, 2, 130, 160)
    frames = [(d, None, cal, dets) for d, _, cal, dets in frames]
    from frustum_convnet_b200.frame_detect import SunrgbdFrameDetector
    fa = SunrgbdFrameDetector(model, frames=2, points=9000, dets=8, seed=13)
    fb = SunrgbdFrameDetector(model, frames=2, points=9000, dets=8, seed=13)
    inp = fa.inputs_depth(H, W, rgb=False)
    fa.stage_depth(inp, _depth_stage(frames))
    a = _snapshot(fa.detect_depth(*inp))
    crop = [(d[:H, :W], c, cal, dets) for d, c, cal, dets in frames]
    cin = fb.inputs()
    fb.stage(cin, _cloud_frames(crop))
    b = _snapshot(fb.detect(*cin))
    assert int(a["status"].item()) == int(b["status"].item()) | 128 and int(b["status"].item()) & 1
    a["status"] = b["status"]
    _same(a, b)


def test_captured_graph_replays_over_new_frames(model):
    F, H, W = 2, 240, 320
    sets = [_depth_frames(s, F, H, W) for s in (21, 22)]
    fg, fe = _detector(model, F, H, W), _detector(model, F, H, W)
    inp, ein = fg.inputs_depth(H, W), fe.inputs_depth(H, W)
    fg.stage_depth(inp, _depth_stage(sets[0]))
    fg.detect_depth(*inp)                                   # the eager call before capture
    fe.stage_depth(ein, _depth_stage(sets[0]))
    fe.detect_depth(*ein)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fg.detect_depth(*inp)
    for k in (1, 0):
        fg.stage_depth(inp, _depth_stage(sets[k]))
        g.replay()
        torch.cuda.synchronize()
        fe.stage_depth(ein, _depth_stage(sets[k]))
        _same(_snapshot(out), _snapshot(fe.detect_depth(*ein)))


def test_depth_clouds_feed_the_offline_extractor():
    from frustum_convnet_b200.sunrgbd_depth import depth_clouds
    from frustum_convnet_b200.sunrgbd_extract import SunrgbdFrustumExtractor
    frames = _depth_frames(31, 3, 200, 260)
    frames[1] = (frames[1][0][:150, :220], frames[1][1], frames[1][2], frames[1][3])   # sizes differ in a chunk
    ids = [5, 9, 2]
    calibs = {i: {"Rtilt": cal[:9].reshape(3, 3), "K": cal[9:].reshape(3, 3)} for i, (_, _, cal, _) in zip(ids, frames)}
    dev = depth_clouds([d for d, *_ in frames], [c for _, c, *_ in frames], [calibs[i] for i in ids], ids, chunk=2)
    ora = {i: c for i, (c, _, _) in zip(ids, _cloud_frames(frames))}
    for i in ids:
        assert dev[i].is_cuda and np.array_equal(_bits(dev[i].cpu().numpy()), _bits(ora[i]))
    det = [(i, t, b, p) for i, (_, _, _, dets) in zip(ids, frames) for t, p, b in dets]
    lists = [list(x) for x in zip(*det)]
    sx = SunrgbdFrustumExtractor()
    ra, rb = np.random.RandomState(4), np.random.RandomState(4)
    a = sx.from_rgb_detections(dev, calibs, *lists, rng=ra)
    b = sx.from_rgb_detections(ora, calibs, *lists, rng=rb)
    ia, ib = a.input_list(), b.input_list()
    assert len(ia) == len(ib) > 0
    assert all(np.array_equal(x, y) for x, y in zip(ia, ib))
    assert a.id_list == b.id_list and np.array_equal(a.frustum_angle_list, b.frustum_angle_list)
    assert ra.random() == rb.random()
