"""GPU: the frustum extractor on the device (csrc/frustum_extract.cu via frustum_convnet_b200/frustum_extract.py)
against the reference's pickle (tests/golden/frustum_extract.npz) and against oracle/frustum_extract.py on larger
random scenes; then the chains it feeds: FrustumBatchBuilder.set_frustums_device + build, and DetectionCollector's
segment table.  Everything is bit-identical except the frustum angle (CUDA's atan2 against glibc's: within 2 ulp) and
what the builder derives from it (within 1 float32 ulp)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(GOLDEN_DIR, "frustum_extract.npz")
ALL = ("Car", "Pedestrian", "Cyclist")


def _angles_close(mine, ref, ulps=2):
    mine, ref = np.asarray(mine, np.float64), np.asarray(ref, np.float64)
    assert mine.shape == ref.shape
    assert np.all(np.abs(mine - ref) <= ulps * np.spacing(np.abs(ref))), np.max(np.abs(mine - ref))


def _extract(scans, calibs, hw, lines, whitelist, stream=None):
    from frustum_convnet_b200.frustum_extract import FrustumExtractor, read_rgb_detections
    ids, types, probs, boxes = read_rgb_detections(lines)
    return FrustumExtractor(whitelist).extract(scans, calibs, hw, ids, types, probs, boxes, stream=stream)


def _check_against(fr, ids, types, probs, boxes, counts, points, angles, P2):
    """fr: the extractor's result; the rest: the reference's (or the oracle's) lists."""
    assert fr.id_list == list(ids) and fr.type_list == list(types)
    assert np.array(fr.prob_list, np.float64).tobytes() == np.asarray(probs, np.float64).tobytes()
    assert np.array(fr.box2d_list).reshape(-1, 4).tobytes() == np.asarray(boxes, np.float64).reshape(-1, 4).tobytes()
    assert fr.counts.tolist() == list(counts)
    assert fr.offsets.cpu().numpy().tolist() == [0] + np.cumsum(counts).tolist()
    assert fr.points.cpu().numpy().tobytes() == np.asarray(points, np.float32).reshape(-1, 4).tobytes()
    assert fr.box2d.cpu().numpy().tobytes() == np.asarray(boxes, np.float64).reshape(-1, 4).tobytes()
    assert fr.P.cpu().numpy().tobytes() == np.asarray(P2, np.float64).reshape(-1, 12).tobytes()
    _angles_close(fr.frustum_angle.cpu().numpy(), angles)


@pytest.mark.parametrize("part", ["exact", "real"])
def test_fixture_matches_the_reference_pickle(part):
    from oracle import kitti_scan_synth as ks
    z = np.load(GOLDEN)
    scans, calibs, hw, lines = ks.fixture_scenes(z, part)
    fr = _extract(scans, calibs, hw, lines, tuple(z[part + "_whitelist"]))
    _check_against(fr, z[part + "_ids"].tolist(), z[part + "_types"].tolist(), z[part + "_probs"],
                   z[part + "_boxes"], z[part + "_counts"].tolist(), z[part + "_points"], z[part + "_angles"],
                   z[part + "_P2"])


def _oracle_check(fr, scene, whitelist):
    from oracle import frustum_extract as ofx
    r_id, r_box, r_in, r_type, r_ang, r_prob, r_cal = ofx.extract(*scene, type_whitelist=whitelist)
    pts = np.concatenate(r_in) if r_in else np.zeros((0, 4), np.float32)
    _check_against(fr, r_id, r_type, r_prob, r_box, [len(p) for p in r_in], pts, r_ang, [c["P2"] for c in r_cal])
    return len(r_id)


def test_matches_the_oracle_on_large_scenes():
    from frustum_convnet_b200.frustum_extract import FrustumExtractor
    from oracle import kitti_scan_synth as ks
    scene = ks.large_scene(5, n_frames=16, n_points=120000, n_dets=30, empty_frame=3)
    scans = dict(scene[0])
    for k in list(scans)[::2]:                      # half of the scans already on the device
        scans[k] = torch.from_numpy(scans[k]).cuda()
    fr = FrustumExtractor(ALL).extract(scans, *scene[1:])
    K = _oracle_check(fr, scene, ALL)
    assert 100 < K < len(scene[3])                  # kept and dropped detections both occur
    empty_id = 100 + 7 * 3
    assert empty_id in scene[3] and empty_id not in fr.id_list
    fr2 = FrustumExtractor(("Car",)).extract(scene[0], *scene[1:])
    _oracle_check(fr2, scene, ("Car",))
    assert fr2.points.cpu().numpy().tobytes() != fr.points.cpu().numpy().tobytes()


def test_every_detection_dropped_gives_empty_tensors():
    from frustum_convnet_b200.frustum_extract import FrustumExtractor
    from oracle import kitti_scan_synth as ks
    scans, calibs, hw, ids, types, probs, boxes = ks.large_scene(6, n_frames=3, n_points=20000, n_dets=8)
    tiny = [np.array([b[0], b[1], b[0] + 0.5, b[1] + 20]) for b in boxes]      # under 1 px wide
    fr = FrustumExtractor(ALL).extract(scans, calibs, hw, ids, types, probs, tiny)
    assert len(fr) == 0 and fr.points.shape == (0, 4) and fr.offsets.cpu().tolist() == [0]
    assert fr.frustum_angle.shape == (0,) and fr.box2d.shape == (0, 4) and fr.P.shape == (0, 12)
    fr = FrustumExtractor(("Van",)).extract(scans, calibs, hw, ids, types, probs, boxes)     # nothing whitelisted
    assert len(fr) == 0 and fr.points.shape == (0, 4) and fr.offsets.cpu().tolist() == [0]


def test_builder_chain_equals_set_frustums_on_the_pickle():
    from frustum_convnet_b200.input_builder import FrustumBatchBuilder
    from oracle import kitti_scan_synth as ks
    z = np.load(GOLDEN)
    scans, calibs, hw, lines = ks.fixture_scenes(z, "real")
    fr = _extract(scans, calibs, hw, lines, ALL)
    counts = z["real_counts"]
    off = np.concatenate([[0], np.cumsum(counts)])
    pts = [z["real_points"][off[k]:off[k + 1]] for k in range(len(counts))]
    cls = np.array([ALL.index(t) for t in z["real_types"].tolist()], dtype=np.int32)
    rng = np.random.default_rng(0)
    N = 1024
    choice = np.stack([rng.choice(n, N, n < N) for n in counts]).astype(np.int32)
    a = FrustumBatchBuilder((0.25, 0.5, 1.0, 2.0), 70.0, N)
    a.set_frustums_device(fr.points, fr.offsets, fr.frustum_angle, fr.box2d, fr.P, cls)
    out_a = {k: v.cpu().numpy() for k, v in a.build(choice).items()}
    b = FrustumBatchBuilder((0.25, 0.5, 1.0, 2.0), 70.0, N)
    b.set_frustums(pts, z["real_angles"], z["real_boxes"], z["real_P2"], cls)
    out_b = {k: v.cpu().numpy() for k, v in b.build(choice).items()}
    assert sorted(out_a) == sorted(out_b)
    for k in out_b:
        x, y = out_a[k], out_b[k]
        assert x.shape == y.shape and x.dtype == y.dtype, k
        assert np.all(np.abs(x - y) <= np.spacing(np.maximum(np.abs(x), np.abs(y)))), k
    assert np.array_equal(out_a["one_hot"], out_b["one_hot"])


def test_collector_segments_equal_the_pickle_lists():
    from frustum_convnet_b200.detect import DetectionCollector
    from oracle import kitti_scan_synth as ks
    z = np.load(GOLDEN)
    for part in ("exact", "real"):
        scans, calibs, hw, lines = ks.fixture_scenes(z, part)
        fr = _extract(scans, calibs, hw, lines, tuple(z[part + "_whitelist"]))
        mine = DetectionCollector(fr.id_list, fr.type_list, fr.box2d_list)
        ref = DetectionCollector(z[part + "_ids"].tolist(), z[part + "_types"].tolist(), list(z[part + "_boxes"]))
        assert mine.segments == ref.segments
        assert np.array_equal(mine._seg_host, ref._seg_host)
        assert torch.equal(mine.box2d, ref.box2d)


def test_runs_on_the_current_stream():
    from oracle import kitti_scan_synth as ks
    z = np.load(GOLDEN)
    scans, calibs, hw, lines = ks.fixture_scenes(z, "real")
    base = _extract(scans, calibs, hw, lines, ALL)
    side = torch.cuda.Stream()
    dev_scans = {k: torch.from_numpy(v).cuda() for k, v in scans.items()}
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        fr = _extract(dev_scans, calibs, hw, lines, ALL)
        got = [t.cpu().numpy() for t in (fr.points, fr.offsets, fr.frustum_angle, fr.box2d, fr.P)]
    want = [t.cpu().numpy() for t in (base.points, base.offsets, base.frustum_angle, base.box2d, base.P)]
    assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want))
    fr = _extract(dev_scans, calibs, hw, lines, ALL, stream=side)
    side.synchronize()
    assert fr.points.cpu().numpy().tobytes() == want[0].tobytes()
