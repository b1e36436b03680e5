"""GPU: the SUN-RGBD frustum extractor on the device (csrc/sunrgbd_extract.cu via
frustum_convnet_b200/sunrgbd_extract.py) against the reference's pickles (tests/golden/sunrgbd_extract.npz) and
against oracle/sunrgbd_extract.py on seeded sets at SUN-RGBD scale, the round window, the caller's stream, the empty
and malformed cases, TrainBatchBuilder.from_frustums("sunrgbd") against set_dataset and the pickle round trip."""
import pickle

import numpy as np
import pytest
import torch

from test_sunrgbd_extract_cpu import PARTS, check_dict, scenes

pytestmark = pytest.mark.gpu


def as_dict(fr):
    from frustum_convnet_b200 import sunrgbd_extract as sx
    keys = sx.GT_KEYS if fr.has_labels else sx.DET_KEYS
    out = {}
    for k, n in keys:
        out[k] = fr.input_list() if k == "input" else fr.label_list() if k == "label" else getattr(fr, n)
    return out


def run(part, z, points, calibs, labels, dets, rng, **kw):
    from frustum_convnet_b200 import sunrgbd_extract as sx
    x = sx.SunrgbdFrustumExtractor()
    ids = z["frame_ids"].tolist() if z is not None else sorted(points)
    if part == "train":
        return x.from_ground_truth(points, calibs, ids, labels, perturb=True, augment=5, rng=rng, **kw)
    if part == "val":
        return x.from_ground_truth(points, calibs, ids, labels, rng=rng, **kw)
    valid = (z["valid"].tolist() if z is not None else ids[::2]) if part == "det_valid" else None
    return x.from_rgb_detections(points, calibs, *dets, valid_ids=valid, rng=rng, **kw)


@pytest.mark.parametrize("part", PARTS)
def test_fixture_matches_the_reference_pickle(part):
    z, *sc = scenes()
    rng = np.random.RandomState(int(z["seed"]))
    fr = run(part, z, *sc, rng)
    check_dict(z, part, as_dict(fr))
    assert rng.random() == float(z[part + "_next_random"])
    assert fr.offsets.cpu().numpy().tolist() == [0] + np.cumsum(z[part + "_counts"]).tolist()
    assert fr.points.dtype == torch.float32 and fr.points.shape[1] == 6
    assert (fr.label is None) == part.startswith("det")


_LARGE = {}


def large():
    if not _LARGE:
        from oracle import sunrgbd_scene_synth as sss
        _LARGE["set"] = sss.large_set(5, n_frames=16)
    return _LARGE["set"]


def _oracle(part, points, calibs, labels, dets, rng):
    from oracle import sunrgbd_extract as osx
    ids = sorted(points)
    if part == "train":
        return osx.from_ground_truth(points, calibs, ids, labels, perturb=True, augment=5, rng=rng)[0]
    if part == "val":
        return osx.from_ground_truth(points, calibs, ids, labels, rng=rng)[0]
    return osx.from_rgb_detections(points, calibs, *dets, valid_ids=ids[::2] if part == "det_valid" else None,
                                   rng=rng)[0]


def same_dict(a, b):
    assert list(a) == list(b)
    for k in a:
        assert len(a[k]) == len(b[k]), k
        for x, y in zip(a[k], b[k]):
            x, y = np.asarray(x), np.asarray(y)
            assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), k


@pytest.mark.parametrize("part", PARTS)
def test_sunrgbd_scale_sets_match_the_oracle(part):
    """16 frames of a 530 x 730 depth grid, 8 objects each (10 classes and a lamp), augment 5."""
    points, calibs, labels, dets = large()
    rng = np.random.RandomState(17)
    fr = run(part, None, points, calibs, labels, dets, rng)
    seq = np.random.RandomState(17)
    ref = _oracle(part, points, calibs, labels, dets, seq)
    assert len(ref["id"]) > 20
    same_dict(as_dict(fr), ref)
    assert rng.random() == seq.random()
    if part == "train":
        assert fr.rounds > 1


def test_windows_one_and_whole_set_agree():
    points, calibs, labels, dets = large()
    sub = {k: points[k] for k in sorted(points)[:4]}
    outs = []
    for window in (1, 10 ** 6):
        rng = np.random.RandomState(3)
        fr = run("train", None, sub, calibs, labels, dets, rng, window=window)
        outs.append((as_dict(fr), rng.random()))
    same_dict(outs[0][0], outs[1][0])
    assert outs[0][1] == outs[1][1]


def test_runs_on_the_callers_stream_and_concurrently():
    points, calibs, labels, dets = large()
    sub = {k: points[k] for k in sorted(points)[:4]}
    base = run("train", None, sub, calibs, labels, dets, np.random.RandomState(4))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fr = run("train", None, sub, calibs, labels, dets, np.random.RandomState(4))
    dev = {k: torch.from_numpy(v).cuda() for k, v in sub.items()}
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = run("train", None, dev, calibs, labels, dets, np.random.RandomState(4), stream=s1)
    b = run("val", None, dev, calibs, labels, dets, np.random.RandomState(4), stream=s2)
    assert a.stream is s1 and b.stream is s2
    vb = run("val", None, sub, calibs, labels, dets, np.random.RandomState(4))
    s.synchronize()
    for f in (fr, a):
        same_dict(as_dict(f), as_dict(base))
    same_dict(as_dict(b), as_dict(vb))


def test_empty_and_malformed_inputs():
    from frustum_convnet_b200 import sunrgbd_extract as sx
    z, points, calibs, labels, dets = scenes()
    ids = z["frame_ids"].tolist()
    x = sx.SunrgbdFrustumExtractor()

    def empty(fr):
        assert len(fr) == 0 and fr.points.shape == (0, 6) and fr.offsets.cpu().tolist() == [0]
        assert fr.input_list() == []

    empty(x.from_ground_truth(points, calibs, [], labels))
    empty(sx.SunrgbdFrustumExtractor(("lamp_post",)).from_ground_truth(points, calibs, ids, labels))
    empty(x.from_rgb_detections(points, calibs, [], [], [], []))
    blank = {i: np.zeros((0, 6), np.float32) for i in ids}
    empty(x.from_ground_truth(blank, calibs, ids, labels, perturb=True, augment=2, rng=np.random.RandomState(0)))
    with pytest.raises(ValueError, match=r"\(n, 6\) float32"):
        x.from_ground_truth({i: p[:, :4] for i, p in points.items()}, calibs, ids, labels)
    with pytest.raises(ValueError, match=r"\(n, 6\) float32"):
        x.from_ground_truth({i: p.astype(np.float64) for i, p in points.items()}, calibs, ids, labels)
    with pytest.raises(ValueError, match="3 x 3"):
        x.from_ground_truth(points, {i: {"Rtilt": c["Rtilt"], "K": c["K"][:2]} for i, c in calibs.items()}, ids,
                            labels)
    with pytest.raises(ValueError, match="frame"):
        x.from_ground_truth({ids[0]: points[ids[0]]}, calibs, ids, labels)
    bad = sx.SUNObject3d("bed 1 2 nan 4 0 1 2 0.5 0.5 0.5 0 0 0 0 1 0", "bad:1")
    with pytest.raises(ValueError, match="bad:1"):
        x.from_ground_truth(points, calibs, ids[:1], {ids[0]: [bad]})
    with pytest.raises(ValueError, match="detection line 0"):
        x.from_rgb_detections(points, calibs, [ids[0]], ["bed"], [np.array([0.0, 0.0, np.inf, 4.0])], [0.5])
    with pytest.raises(RuntimeError):
        x.from_ground_truth({i: torch.from_numpy(p) for i, p in points.items()}, calibs, ids, labels)


def _set_dataset(fr_or_dict, labelled, strides, npoints):
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    d = fr_or_dict if isinstance(fr_or_dict, dict) else as_dict(fr_or_dict)
    b = TrainBatchBuilder("sunrgbd", strides, npoints, labels=labelled)
    kw = dict(frustum_angle_list=d["frustum_angle"], box2d_list=d["box2d"], calib_K_list=d["calib_K"],
              calib_R_list=d["calib_R"])
    if labelled:
        kw.update(label_list=d["label"], box3d_list=d["box3d"], heading_list=d["box3d_heading"],
                  size_list=d["box3d_size"])
    else:
        kw["prob_list"] = d["box2d_prob"]
    b.set_dataset(d["input"], d["type"], **kw)
    return b


@pytest.mark.parametrize("part", ["train", "det"])
def test_from_frustums_builds_what_set_dataset_builds(part):
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    z, *sc = scenes()
    fr = run(part, z, *sc, np.random.RandomState(int(z["seed"])))
    labelled = part == "train"
    strides, npoints = [0.25, 0.5, 1.0, 2.0, 4.0], 1024
    a = TrainBatchBuilder.from_frustums(fr, "sunrgbd", strides=strides, npoints=npoints)
    assert a.labels == labelled
    b = _set_dataset(fr, labelled, strides, npoints)
    ref_dict, _ = __import__("test_sunrgbd_extract_cpu").oracle_part(part, z, *sc,
                                                                      np.random.RandomState(int(z["seed"])))
    c = _set_dataset(ref_dict, labelled, strides, npoints)
    if labelled:
        assert a.d_seg.dtype == torch.int32 and torch.equal(a.d_seg, b.d_seg) and torch.equal(a.d_seg, c.d_seg)
    idx = np.arange(min(len(fr), 16))
    draws = a.draw(idx, np.random.RandomState(9))
    oa = {k: v.clone() for k, v in a.build(idx, draws).items()}
    ob = {k: v.clone() for k, v in b.build(idx, draws).items()}
    oc = c.build(idx, draws)
    assert oa.keys() == ob.keys() == oc.keys()
    for k in oa:
        assert torch.equal(oa[k], ob[k]) and torch.equal(oa[k], oc[k]), k
    with pytest.raises(ValueError, match="kind='sunrgbd'"):
        TrainBatchBuilder.from_frustums(fr, "det", strides=strides[:4], npoints=npoints)


def test_to_pickle_round_trip(tmp_path):
    z, *sc = scenes()
    for part in ("train", "det_valid"):
        fr = run(part, z, *sc, np.random.RandomState(int(z["seed"])))
        p = tmp_path / (part + ".pickle")
        fr.to_pickle(str(p))
        with open(p, "rb") as f:
            back = pickle.load(f)
        check_dict(z, part, back)
