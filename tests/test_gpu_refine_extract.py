"""GPU: the refinement extractor on the device (csrc/refine_extract.cu via frustum_convnet_b200/refine_extract.py)
against the reference's pickles (tests/golden/refine_extract.npz) and against oracle/refine_extract.py on KITTI-sized
scenes, the empty cases, the caller's stream, TrainBatchBuilder.from_frustums against set_dataset, and the two-stage
chain from the first stage's collector through the refinement forward to the evaluator."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(GOLDEN_DIR, "refine_extract.npz")


def _lists(fr):
    L = {n: getattr(fr, n) for n in ("id_list", "box2d_list", "type_list", "frustum_angle_list", "prob_list",
                                     "calib_list", "box3d_list", "heading_list", "size_list", "pred_box3d_list",
                                     "pred_box3d_size_list", "pred_box3d_angle_list")}
    L["input_list"] = fr.input_list()
    if fr.has_labels:
        L["label_list"] = fr.label_list()
    return L


def _run(part, scans, calibs, hws, ids, labels, results, rng=None, stream=None):
    from frustum_convnet_b200 import refine_extract as rx
    from oracle import kitti_refine_synth as krs
    from oracle import make_golden_refine_extract as mg
    kw = mg.MODES[part]
    x = rx.RefineFrustumExtractor(mg.WHITELIST)
    if kw["mode"] == "gt":
        return x.from_ground_truth(scans, calibs, hws, ids, krs.objects(labels), kw.get("perturb", False),
                                   kw.get("augment", 1), rng, kw.get("remove_diff", False), stream=stream)
    if kw["mode"] == "matched":
        return x.from_matched_detections(scans, calibs, hws, ids, krs.objects(results), krs.objects(labels),
                                         remove_diff=True, stream=stream)
    return x.from_detections(scans, calibs, hws, ids, krs.objects(results), stream=stream)


@pytest.mark.parametrize("part", ["gt_train", "gt_val", "matched", "det"])
def test_fixture_matches_the_reference_pickle(part):
    from oracle import kitti_refine_synth as krs
    from test_refine_extract_cpu import check_lists
    z = np.load(GOLDEN)
    scans, calibs, hws, labels, results = krs.fixture_scenes(z)
    fr = _run(part, scans, calibs, hws, z["frame_ids"].tolist(), labels, results,
              np.random.RandomState(int(z["train_seed"])))
    check_lists(z, part, _lists(fr))
    assert fr.offsets.cpu().numpy().tolist() == [0] + np.cumsum(z[part + "_counts"]).tolist()
    assert (fr.label is None) == (part == "det")


@pytest.mark.parametrize("part", ["gt_train", "matched", "det"])
def test_large_scenes_match_the_oracle(part):
    from oracle import kitti_refine_synth as krs
    from oracle import make_golden_refine_extract as mg
    from oracle import refine_extract as orx
    scans, calibs, hws, labels, results = krs.large_scene(11, n_frames=6)
    ids = sorted(scans)
    fr = _run(part, scans, calibs, hws, ids, labels, results, np.random.RandomState(5))
    kw = mg.MODES[part]
    ref = orx.extract(kw["mode"], scans, calibs, hws, ids, krs.objects(results), krs.objects(labels), mg.WHITELIST,
                      kw.get("remove_diff", False), kw.get("perturb", False), kw.get("augment", 1),
                      np.random.RandomState(5))
    mine = _lists(fr)
    assert len(mine["id_list"]) > 0 and mine["id_list"] == ref["id_list"]
    for n in ("input_list", "label_list"):
        if n in ref:
            assert all(a.tobytes() == np.asarray(b, a.dtype).tobytes() for a, b in zip(mine[n], ref[n])), n
    for n in ("frustum_angle_list", "pred_box3d_list", "box3d_list", "heading_list", "prob_list"):
        if n in ref:
            assert np.array(mine[n]).tobytes() == np.array(ref[n]).tobytes(), n


def test_empty_cases():
    from frustum_convnet_b200 import refine_extract as rx
    from oracle import kitti_refine_synth as krs
    scans, calibs, hws, labels, results = krs.large_scene(12, n_frames=2, n_points=5000)
    ids = sorted(scans)
    x = rx.RefineFrustumExtractor(("Car",))

    def empty(fr, labelled):
        assert len(fr) == 0 and fr.points.shape == (0, 4) and fr.offsets.cpu().tolist() == [0]
        assert (fr.label is not None) == labelled and fr.points.is_cuda

    empty(x.from_detections(scans, calibs, hws, [], {}), False)                       # no frames
    empty(x.from_detections(scans, calibs, hws, ids, {}), False)                      # no detections
    far = {i: [rx.KittiObject.parse("Car -1 -1 0 10 10 60 60 1.5 1.6 3.9 0 1.6 -30 0 0.5")] for i in ids}
    empty(x.from_detections(scans, calibs, hws, ids, far), False)                     # every box dropped (no point)
    no_gt = {i: [] for i in ids}
    empty(x.from_matched_detections(scans, calibs, hws, ids, krs.objects(results), no_gt), True)   # frames without GT
    blank = {i: np.zeros((0, 4), np.float32) for i in ids}                                       # no in-image point
    empty(x.from_ground_truth(blank, calibs, hws, ids, krs.objects(labels)), True)
    with pytest.raises(RuntimeError):
        rx.RefineFrustumExtractor(device="cpu")
    with pytest.raises(RuntimeError):
        x.from_detections({i: torch.zeros((3, 4)) for i in ids}, calibs, hws, ids, krs.objects(results))


def test_runs_on_the_callers_stream():
    from oracle import kitti_refine_synth as krs
    scans, calibs, hws, labels, results = krs.large_scene(13, n_frames=3, n_points=40000)
    ids = sorted(scans)
    base = _run("det", scans, calibs, hws, ids, labels, results)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fr = _run("det", scans, calibs, hws, ids, labels, results)
        assert torch.cuda.current_stream().cuda_stream == s.cuda_stream
    fr2 = _run("det", {k: torch.from_numpy(v).cuda() for k, v in scans.items()}, calibs, hws, ids, labels, results,
               stream=s)
    s.synchronize()
    for f in (fr, fr2):
        assert torch.equal(f.points, base.points) and torch.equal(f.offsets, base.offsets)


@pytest.mark.parametrize("part", ["gt_train", "det"])
def test_from_frustums_builds_what_set_dataset_builds(part):
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    from oracle import kitti_refine_synth as krs
    scans, calibs, hws, labels, results = krs.large_scene(14, n_frames=4, n_points=40000)
    fr = _run(part, scans, calibs, hws, sorted(scans), labels, results, np.random.RandomState(2))
    labelled = part != "det"
    strides, npoints = [0.25, 0.5, 1.0, 2.0], 280
    a = TrainBatchBuilder.from_frustums(fr, "refine", strides=strides, npoints=npoints, labels=labelled)
    b = TrainBatchBuilder("refine", strides, npoints, labels=labelled)
    L = _lists(fr)
    b.set_dataset(L["input_list"], L["type_list"], box3d_list=L["box3d_list"], heading_list=L["heading_list"],
                  size_list=L["size_list"], prob_list=L["prob_list"], pred_box3d_list=L["pred_box3d_list"],
                  pred_box3d_size_list=L["pred_box3d_size_list"], pred_box3d_angle_list=L["pred_box3d_angle_list"])
    idx = np.arange(min(len(fr), 16))
    draws = a.draw(idx, np.random.RandomState(9))
    oa = {k: v.clone() for k, v in a.build(idx, draws).items()}
    ob = b.build(idx, draws)
    assert oa.keys() == ob.keys()
    for k in oa:
        assert torch.equal(oa[k], ob[k]), k


def _write_results(result_dir, dets, ids):
    """The text write_detection_results (train/test_net_det.py:88-123) writes for the collector's dict, one file per
    image of `ids` (an image without detections gets an empty file, as fill_files makes it)."""
    from frustum_convnet_b200.kitti_eval import compute_alpha
    os.makedirs(result_dir, exist_ok=True)
    for i in ids:
        per_class = dets.get(i, {})
        out = []
        for c, rows in per_class.items():
            for r in rows:
                s = c + " -1 -1 " + "%.4f " % compute_alpha(r[4], r[6], r[10]) + "%.4f %.4f %.4f %.4f " % tuple(r[:4])
                s += "%.4f %.4f %.4f %.4f %.4f %.4f %.4f %f" % (r[7], r[8], r[9], r[4], r[5], r[6], r[10], r[11])
                out.append(s + "\n")
        with open(os.path.join(result_dir, "%06d.txt" % i), "w") as f:
            f.write("".join(out))


def _same_frustums(a, b):
    assert torch.equal(a.points, b.points) and torch.equal(a.offsets, b.offsets)
    assert a.id_list == b.id_list and a.prob_list == b.prob_list and a.type_list == b.type_list
    assert np.array(a.box2d_list).tobytes() == np.array(b.box2d_list).tobytes()
    for n in ("pred_box3d_list", "pred_box3d_size_list", "pred_box3d_angle_list", "frustum_angle_list"):
        assert np.array(getattr(a, n)).tobytes() == np.array(getattr(b, n)).tobytes(), n


def test_collector_detections_equal_their_result_files(tmp_path):
    """Collector-shaped detections give the same refinement frustums as the result files written for them."""
    from frustum_convnet_b200 import refine_extract as rx
    from oracle import kitti_refine_synth as krs
    scans, calibs, hws, labels, results = krs.large_scene(15, n_frames=3, n_points=30000)
    ids = sorted(scans)
    dets = {}
    for i in ids:
        rows = {}
        for o in krs.objects(results)[i]:
            rows.setdefault(o.type, []).append(list(o.box2d) + list(o.t) + [o.h, o.w, o.l, o.ry, o.score])
        dets[i] = {c: np.array(r, np.float32) for c, r in rows.items()}
    _write_results(str(tmp_path), dets, ids)
    x = rx.RefineFrustumExtractor(("Car", "Pedestrian"))
    fr = x.from_detections(scans, calibs, hws, ids, dets)
    assert len(fr) > 0
    _same_frustums(fr, x.from_detections(scans, calibs, hws, ids, rx.read_result_dir(str(tmp_path), ids)))


def test_two_stage_chain(tmp_path):
    """scene -> FrustumExtractor -> first-stage forward (synthetic weights) -> DetectionCollector.finalize() ->
    from_detections -> TrainBatchBuilder.from_frustums("refine", labels=False) -> refinement forward -> collector ->
    KittiEvaluator; the refinement frustums of finalize()'s dict equal those of the same detections written as result
    files and read back with read_result_dir."""
    from train_ref import make_model
    from frustum_convnet_b200 import config
    from frustum_convnet_b200 import refine_extract as rx
    from frustum_convnet_b200.detect import DetectionCollector
    from frustum_convnet_b200.frustum_extract import FrustumExtractor
    from frustum_convnet_b200.input_builder import FrustumBatchBuilder
    from frustum_convnet_b200.kitti_eval import KittiEvaluator, KittiGroundTruth, detection_records
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    from oracle import kitti_refine_synth as krs
    classes = ("Car", "Pedestrian", "Cyclist")
    scans, calibs, hws, labels, results = krs.large_scene(16, n_frames=4, n_points=40000)
    ids = sorted(scans)
    label_dir = tmp_path / "label_2"
    label_dir.mkdir()
    for i in ids:
        (label_dir / ("%06d.txt" % i)).write_text("".join(ln + "\n" for ln in labels[i]))
    # first stage: 2-D boxes of the whitelisted ground truth as the 2-D detector's output
    gt = krs.objects(labels)
    lines = [(i, o.type, 0.9, o.box2d) for i in ids for o in gt[i] if o.type in classes]
    fr1 = FrustumExtractor(classes).extract(scans, calibs, hws, *map(list, zip(*lines)))
    assert len(fr1) > 0
    m1 = make_model("car", 3).eval()
    cfg, _ = config.load_workload("car")
    N = int(cfg.DATA.NUM_SAMPLES)
    fb = FrustumBatchBuilder(list(cfg.DATA.STRIDE), float(cfg.DATA.MAX_DEPTH), N)
    fb.set_frustums_device(fr1.points, fr1.offsets, fr1.frustum_angle, fr1.box2d, fr1.P,
                           np.array([classes.index(t) for t in fr1.type_list], np.int32))
    rng = np.random.RandomState(1)
    data = dict(fb.build(np.stack([rng.choice(n, N, n < N) for n in fr1.counts]).astype(np.int32)),
                rgb_prob=torch.tensor(fr1.prob_list, dtype=torch.float32, device="cuda"))
    with torch.no_grad():
        out = m1(data)
    col = DetectionCollector(fr1.id_list, fr1.type_list, fr1.box2d_list)
    col.add(out, data, first=0)
    dets = col.finalize()
    assert sum(len(r) for d in dets.values() for r in d.values()) > 0
    # a synthetic-weight model may decode non-positive sizes; the reference's Qhull rejects those boxes, so does this
    good = {i: {c: r[(detection_records(r, c)[:, 6:9] > 0).all(1)] for c, r in d.items()} for i, d in dets.items()}
    x = rx.RefineFrustumExtractor(classes)
    if any(len(good[i][c]) < len(dets[i][c]) for i in dets for c in dets[i]):
        with pytest.raises(ValueError, match="positive l, w, h"):
            x.from_detections(scans, calibs, hws, ids, dets)
    fr = x.from_detections(scans, calibs, hws, ids, good)
    assert len(fr) > 0
    _write_results(str(tmp_path / "data"), good, ids)
    _same_frustums(fr, x.from_detections(scans, calibs, hws, ids, rx.read_result_dir(str(tmp_path / "data"), ids)))
    # refinement stage on the extractor's device tensors
    m2 = make_model("refine_car", 5).eval()
    cfg, _ = config.load_workload("refine_car")
    tb = TrainBatchBuilder.from_frustums(fr, "refine", strides=list(cfg.DATA.STRIDE),
                                         npoints=int(cfg.DATA.NUM_SAMPLES), labels=False)
    idx = np.arange(len(fr))
    data2 = tb.build(idx, tb.draw(idx, np.random.RandomState(2)))
    with torch.no_grad():
        out2 = m2(data2)
    col2 = DetectionCollector(fr.id_list, fr.type_list, fr.box2d_list)
    col2.add(out2, data2, first=0)
    refined = col2.finalize()
    assert sum(len(r) for d in refined.values() for r in d.values()) > 0
    res = KittiEvaluator(KittiGroundTruth.from_label_dir(str(label_dir), ids)).evaluate(refined)
    assert len(res.lines()) > 0


def test_matched_mode_checks_extents_only_once_matched():
    """A whitelisted detection with a zero extent matches nothing (its IoU is 0): the reference skips it before any
    Delaunay call, and so does the extractor."""
    from frustum_convnet_b200 import refine_extract as rx
    from oracle import kitti_refine_synth as krs
    scans, calibs, hws, labels, results = krs.large_scene(17, n_frames=2, n_points=20000)
    ids = sorted(scans)
    dets = krs.objects(results)
    flat = rx.KittiObject.parse("Car -1 -1 0 10 10 60 60 1.5 0 3.9 1 1.6 20 0 0.5", "flat:1")
    dets[ids[0]] = dets[ids[0]] + [flat]
    x = rx.RefineFrustumExtractor(("Car",))
    a = x.from_matched_detections(scans, calibs, hws, ids, dets, krs.objects(labels))
    b = x.from_matched_detections(scans, calibs, hws, ids, krs.objects(results), krs.objects(labels))
    assert torch.equal(a.points, b.points) and a.id_list == b.id_list
    with pytest.raises(ValueError, match="flat:1"):
        x.from_detections(scans, calibs, hws, ids, dets)


def test_lists_wait_for_the_extraction_stream():
    from oracle import kitti_refine_synth as krs
    scans, calibs, hws, labels, results = krs.large_scene(18, n_frames=3, n_points=40000)
    ids = sorted(scans)
    base = _run("gt_val", scans, calibs, hws, ids, labels, results)
    want = [p.tobytes() for p in base.input_list()]
    side = torch.cuda.Stream()
    dev_scans = {k: torch.from_numpy(v).cuda() for k, v in scans.items()}
    torch.cuda.synchronize()
    fr = _run("gt_val", dev_scans, calibs, hws, ids, labels, results, stream=side)
    assert fr.stream is side
    assert [p.tobytes() for p in fr.input_list()] == want          # no synchronize: input_list waits for `side`
