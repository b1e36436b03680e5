"""GPU: the first-stage ground-truth extractor on the device (csrc/gt_extract.cu via frustum_convnet_b200/gt_extract.py)
against the reference's pickles (tests/golden/gt_extract.npz) and against oracle/gt_extract.py on KITTI-sized scenes,
the empty cases, the caller's stream, the workspace check, TrainBatchBuilder.from_frustums("det") against set_dataset,
the chain into one training step and the validation pass, and the pickle round trip."""
import ctypes
import math
import pickle

import numpy as np
import pytest
import torch

from test_gt_extract_cpu import PARTS, check_lists, part_args, scenes

pytestmark = pytest.mark.gpu


def _lists(fr):
    from frustum_convnet_b200 import gt_extract as gx
    L = {n: getattr(fr, n) for n in gx.NAMES if n not in ("input_list", "label_list")}
    L["input_list"], L["label_list"] = fr.input_list(), fr.label_list()
    return L


def _run(part, scans, calibs, hws, ids, labels, dets, rng=None, stream=None):
    from frustum_convnet_b200 import gt_extract as gx
    from frustum_convnet_b200.frustum_extract import read_rgb_detections
    from oracle import kitti_refine_synth as krs
    wl, mode, perturb, augment = part_args(part)
    x = gx.GtFrustumExtractor(wl)
    if mode == "gt":
        return x.from_ground_truth(scans, calibs, hws, ids, krs.objects(labels), perturb, augment, rng, stream=stream)
    return x.from_matched_detections(scans, calibs, hws, ids, *read_rgb_detections(dets), krs.objects(labels),
                                     perturb, augment, rng, stream=stream)


def _large(seed, **kw):
    from oracle import kitti_refine_synth as krs
    from oracle import make_golden_gt_extract as mg
    scans, calibs, hws, labels, results = krs.large_scene(seed, **kw)
    return scans, calibs, hws, labels, mg.det_lines(results)


@pytest.mark.parametrize("part", PARTS)
def test_fixture_matches_the_reference_pickle(part):
    z, scans, calibs, hws, labels, dets = scenes()
    fr = _run(part, scans, calibs, hws, z["frame_ids"].tolist(), labels, dets,
              np.random.RandomState(int(z["train_seed"])))
    check_lists(z, part, _lists(fr))
    assert fr.offsets.cpu().numpy().tolist() == [0] + np.cumsum(z[part + "_counts"]).tolist()
    assert fr.label.dtype == torch.uint8 and fr.points.dtype == torch.float32


@pytest.mark.parametrize("part", ["car_train", "car_val", "car_matched", "people_matched"])
def test_large_scenes_match_the_oracle(part):
    from frustum_convnet_b200.frustum_extract import read_rgb_detections
    from oracle import gt_extract as ogx
    from oracle import kitti_refine_synth as krs
    scans, calibs, hws, labels, dets = _large(21, n_frames=6)
    ids = sorted(scans)
    fr = _run(part, scans, calibs, hws, ids, labels, dets, np.random.RandomState(5))
    wl, mode, perturb, augment = part_args(part)
    ref = ogx.extract(mode, scans, calibs, hws, ids, krs.objects(labels), wl, perturb, augment,
                      np.random.RandomState(5), read_rgb_detections(dets))
    mine = _lists(fr)
    assert len(mine["id_list"]) > 0 and mine["id_list"] == ref["id_list"]
    for n in ("input_list", "label_list"):
        assert all(a.tobytes() == b.tobytes() for a, b in zip(mine[n], ref[n])), n
    for n in ("box2d_list", "box3d_list", "heading_list", "size_list", "frustum_angle_list", "gt_box2d_list"):
        assert np.array(mine[n]).tobytes() == np.array(ref[n]).tobytes(), n


def test_empty_cases():
    from frustum_convnet_b200 import gt_extract as gx
    scans, calibs, hws, labels, dets = _large(22, n_frames=2, n_points=5000)
    ids = sorted(scans)
    from oracle import kitti_refine_synth as krs
    gt = krs.objects(labels)
    x = gx.GtFrustumExtractor(("Car",))

    def empty(fr):
        assert len(fr) == 0 and fr.points.shape == (0, 4) and fr.offsets.cpu().tolist() == [0]
        assert fr.label.shape == (0,) and fr.points.is_cuda and fr.input_list() == []

    empty(x.from_ground_truth(scans, calibs, hws, [], gt))                                  # no frames
    empty(gx.GtFrustumExtractor(("Tram",)).from_ground_truth(scans, calibs, hws, ids, gt))  # no whitelisted object
    blank = {i: np.zeros((0, 4), np.float32) for i in ids}                                 # every job dropped
    empty(x.from_ground_truth(blank, calibs, hws, ids, gt))
    empty(x.from_matched_detections(scans, calibs, hws, ids, [], [], [], [], gt))           # no detection
    with pytest.raises(RuntimeError):
        x.from_ground_truth({i: torch.zeros((3, 4)) for i in ids}, calibs, hws, ids, gt)   # CPU tensors


def test_runs_on_the_callers_stream():
    scans, calibs, hws, labels, dets = _large(23, n_frames=3, n_points=40000)
    ids = sorted(scans)
    base = _run("car_val", scans, calibs, hws, ids, labels, dets)
    want = [p.tobytes() for p in base.input_list()]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fr = _run("car_val", scans, calibs, hws, ids, labels, dets)
        assert torch.cuda.current_stream().cuda_stream == s.cuda_stream
    dev_scans = {k: torch.from_numpy(v).cuda() for k, v in scans.items()}
    torch.cuda.synchronize()
    s2 = torch.cuda.Stream()
    fr2 = _run("car_val", dev_scans, calibs, hws, ids, labels, dets, stream=s2)
    assert fr2.stream is s2
    assert [p.tobytes() for p in fr2.input_list()] == want         # no synchronize: input_list waits for s2
    s.synchronize()
    for f in (fr, fr2):
        assert torch.equal(f.points, base.points) and torch.equal(f.offsets, base.offsets)
        assert torch.equal(f.label, base.label)


def test_workspace_one_byte_short_is_refused_and_the_queried_size_runs(monkeypatch):
    from frustum_convnet_b200 import _lib
    lib, real_call, seen = _lib.load(), _lib.call, []

    def call(name, *args):
        if name in ("fcn_gt_extract_count", "fcn_gt_extract_write"):
            a = args[0]._obj
            n = lib.fcn_gt_extract_workspace_bytes(ctypes.byref(a))
            assert n > 0 and a.workspace_bytes == n, (name, n, a.workspace_bytes)
            a.workspace_bytes = n - 1
            assert getattr(lib, name)(*args) == -1, name
            assert b"workspace smaller than fcn_gt_extract_workspace_bytes()" in lib.fcn_last_error()
            a.workspace_bytes = n
            if name == "fcn_gt_extract_count":             # bad scan offsets are refused too
                so = np.ctypeslib.as_array(ctypes.cast(a.host_scan_offsets, ctypes.POINTER(ctypes.c_int32)),
                                           (a.num_frames + 1,))
                keep = so[1]
                so[1] = so[-1] + 1
                assert getattr(lib, name)(*args) == -1
                assert b"scan offsets must start at 0" in lib.fcn_last_error()
                so[1] = keep
            seen.append(name)
        real_call(name, *args)

    monkeypatch.setattr(_lib, "call", call)
    z, scans, calibs, hws, labels, dets = scenes()
    assert len(_run("car_matched", scans, calibs, hws, z["frame_ids"].tolist(), labels, dets,
                    np.random.RandomState(1)))
    assert seen == ["fcn_gt_extract_count", "fcn_gt_extract_write"]


def _set_dataset_builder(fr, strides, npoints, **kw):
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    L = _lists(fr)
    b = TrainBatchBuilder("det", strides, npoints, **kw)
    b.set_dataset(L["input_list"], L["type_list"], **{n: L[n] for n in (
        "label_list", "box3d_list", "heading_list", "size_list", "frustum_angle_list", "box2d_list", "calib_list")})
    return b


@pytest.mark.parametrize("part", ["car_train", "people_matched"])
def test_from_frustums_builds_what_set_dataset_builds(part):
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    scans, calibs, hws, labels, dets = _large(24, n_frames=4, n_points=40000)
    fr = _run(part, scans, calibs, hws, sorted(scans), labels, dets, np.random.RandomState(2))
    strides, npoints = [0.25, 0.5, 1.0, 2.0], 280
    a = TrainBatchBuilder.from_frustums(fr, "det", strides=strides, npoints=npoints)
    b = _set_dataset_builder(fr, strides, npoints)
    assert a.d_seg.dtype == torch.int32 and torch.equal(a.d_seg, b.d_seg)
    idx = np.arange(min(len(fr), 16))
    draws = a.draw(idx, np.random.RandomState(9))
    oa = {k: v.clone() for k, v in a.build(idx, draws).items()}
    ob = b.build(idx, draws)
    assert oa.keys() == ob.keys() and "seg_label" in oa
    for k in oa:
        assert torch.equal(oa[k], ob[k]), k
    with pytest.raises(ValueError):
        TrainBatchBuilder.from_frustums(fr, "refine", strides=strides, npoints=npoints)


def test_refine_frustums_still_refuse_det():
    from frustum_convnet_b200 import refine_extract as rx
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    from oracle import kitti_refine_synth as krs
    scans, calibs, hws, labels, results = krs.large_scene(25, n_frames=2, n_points=20000)
    fr = rx.RefineFrustumExtractor(("Car",)).from_ground_truth(scans, calibs, hws, sorted(scans),
                                                               krs.objects(labels))
    with pytest.raises(ValueError, match="kind='refine'"):
        TrainBatchBuilder.from_frustums(fr, "det", strides=[0.25, 0.5, 1.0, 2.0], npoints=280)


def test_chain_into_a_training_step_and_the_validation_pass():
    """train extraction -> from_frustums("det") -> one TrainStep.forward_backward on the car workload (synthetic
    weights), losses equal to the same step on the set_dataset batch; the val extraction through the Validator."""
    from train_ref import make_model
    from frustum_convnet_b200 import config
    from frustum_convnet_b200.train_engine import TrainStep
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    from frustum_convnet_b200.validate import Validator
    cfg, _ = config.load_workload("car")
    strides, N = list(cfg.DATA.STRIDE), int(cfg.DATA.NUM_SAMPLES)
    scans, calibs, hws, labels, dets = _large(26, n_frames=6, n_points=60000)
    ids = sorted(scans)
    train = _run("car_train", scans, calibs, hws, ids, labels, dets, np.random.RandomState(3))
    assert len(train) >= 8
    a = TrainBatchBuilder.from_frustums(train, "det", strides=strides, npoints=N)
    b = _set_dataset_builder(train, strides, N)
    idx = np.arange(8)
    draws = a.draw(idx, np.random.RandomState(4))
    losses = []
    for tb in (a, b):
        data = tb.build(idx, draws)
        lo, _ = TrainStep(make_model("car", 13)).forward_backward(data)
        torch.cuda.synchronize()
        losses.append({k: float(v) for k, v in lo.items()})
    assert losses[0].keys() == losses[1].keys() and len(losses[0]) > 0
    for k, ref_v in losses[1].items():         # the batches are torch.equal; the tolerance is the step's own
        assert abs(losses[0][k] - ref_v) <= 1e-5 * max(1e-6, abs(ref_v)), (k, losses[0][k], ref_v)
        assert math.isfinite(losses[0][k]), k
    val = _run("car_val", scans, calibs, hws, ids, labels, dets)
    tv = TrainBatchBuilder.from_frustums(val, "det", strides=strides, npoints=N, random_flip=False,
                                         random_shift=False)
    v = Validator(make_model("car", 14).eval())
    for start in range(0, len(val), 8):
        i = np.arange(start, min(start + 8, len(val)))
        v.add(tv.build(i, tv.draw(i, np.random.RandomState(start))))
    meters = v.finalize()
    assert len(meters) > 0 and all(math.isfinite(x) for x in meters.values()), meters


def test_to_pickle_round_trip(tmp_path):
    from frustum_convnet_b200 import gt_extract as gx
    z, scans, calibs, hws, labels, dets = scenes()
    for part in ("car_train", "car_matched"):
        fr = _run(part, scans, calibs, hws, z["frame_ids"].tolist(), labels, dets,
                  np.random.RandomState(int(z["train_seed"])))
        p = tmp_path / (part + ".pickle")
        fr.to_pickle(str(p))
        with open(p, "rb") as f:
            back = {n: pickle.load(f) for n in gx.NAMES}
        assert list(back) == list(gx.NAMES)
        check_lists(z, part, back)
