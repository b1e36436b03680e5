"""GPU: the SUN-RGBD kind of the training-batch builder (C ABI section 11, FCN_TRAIN_SUNRGBD) against the batches the
reference's own provider_sample_sunrgbd + default_collate produced (tests/golden/train_inputs_sunrgbd.npz) and against
the numpy restatement (oracle/train_inputs_sunrgbd.py) on a 2 000-frustum random dataset.  Float outputs must be
within one float32 ulp and >= 99.9 % bit-identical (np.dot goes through BLAS in the reference); int outputs exact;
cls_label exact except for refs within 1e-9 m of a box face.  Then what the batches feed: CUDA-graph replay, one
training step, the validation pass and the detection collector, each on the built batch against the reference batch."""
import numpy as np
import pytest
import torch

from test_train_inputs_sunrgbd_cpu import SUN, compare, fixture_batches, fixture_lists, load_fixture, oracle_batch

pytestmark = pytest.mark.gpu


def _builder(mode, L, N=2048, strides=SUN):
    from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES, TrainBatchBuilder
    aug, labels = mode == "train", mode != "rgb"
    tb = TrainBatchBuilder("sunrgbd", strides, N, random_flip=aug, random_shift=aug, labels=labels)
    tb.set_dataset(L["input_list"], L["type_list"], SUNRGBD_CLASSES,
                   **{k: v for k, v in L.items() if k not in ("input_list", "type_list")})
    return tb


def _host(out):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def _cuda(batch):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in batch.items() if not k.startswith("_")}


def test_builder_matches_the_reference_fixture():
    g = load_fixture()
    total = same = 0
    for mode, index, draws, ref in fixture_batches(g):
        tb = _builder(mode, fixture_lists(g, mode != "rgb"))
        out = _host(tb.build(index, draws))
        assert set(out) == set(ref), set(out) ^ set(ref)
        margins = oracle_batch(g, mode, index, draws).get("_margins")
        t, s = compare(out, ref, margins, exact=False)
        total, same = total + t, same + s
    assert same >= 0.999 * total, (same, total)
    print("sunrgbd: %d / %d float values bit-identical to the reference provider" % (same, total))


def random_sun_lists(F, rng, labels=True):
    """F random SUN-RGBD frustums in the prepared pickles' dtypes: float32 points with 6 columns, float32 box2d, bool
    seg labels, tilted Rtilt, f_u != f_v, all 10 classes."""
    from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES, compute_box_3d
    from oracle.train_inputs_sunrgbd import project_image_to_upright_camera
    n = rng.integers(1, 3000, F)
    L = {k: [] for k in ("input_list", "type_list", "box2d_list", "frustum_angle_list", "calib_K_list",
                         "calib_R_list", "prob_list", "label_list", "box3d_list", "heading_list", "size_list")}
    for i in range(F):
        K = np.array([[529.5 + rng.normal(0, 5), 0, 365 + rng.normal(0, 5)],
                      [0, 529.5 + rng.normal(0, 5), 262 + rng.normal(0, 5)], [0, 0, 1]])
        ax, az = rng.uniform(-0.15, 0.15), rng.uniform(-0.05, 0.05)
        R = np.array([[np.cos(az), -np.sin(az), 0], [np.sin(az), np.cos(az), 0], [0, 0, 1]]) @ \
            np.array([[1, 0, 0], [0, np.cos(ax), -np.sin(ax)], [0, np.sin(ax), np.cos(ax)]])
        u, v = rng.uniform(100, 630), rng.uniform(80, 450)
        box2d = np.array([u - rng.uniform(10, 90), v - rng.uniform(10, 90), u + rng.uniform(10, 90),
                          v + rng.uniform(10, 90)], dtype=np.float32)
        uvd = np.array([[(box2d[0] + box2d[2]) / 2.0, (box2d[1] + box2d[3]) / 2.0, 20.0]])
        ray = project_image_to_upright_camera(uvd, K, R)[0] / 20.0
        angle = -np.arctan2(ray[2], ray[0])
        C = ray * rng.uniform(0.5, 7.5) + rng.normal(0, 0.2, 3)
        size = rng.uniform(0.4, 2.2, 3)
        L["input_list"].append(np.concatenate([C + rng.normal(0, 0.5, (n[i], 3)), rng.uniform(0, 1, (n[i], 3))],
                                              1).astype(np.float32))
        L["type_list"].append(SUNRGBD_CLASSES[rng.integers(0, 10)])
        L["box2d_list"].append(box2d)
        L["frustum_angle_list"].append(angle)
        L["calib_K_list"].append(K)
        L["calib_R_list"].append(R)
        L["prob_list"].append(float(rng.uniform(0.1, 1.0)))
        heading = rng.uniform(-np.pi, np.pi)
        L["label_list"].append(rng.uniform(0, 1, n[i]) < 0.3)
        L["box3d_list"].append(compute_box_3d(C, size, heading))
        L["heading_list"].append(float(heading))
        L["size_list"].append(size)
    if not labels:
        for k in ("label_list", "box3d_list", "heading_list", "size_list"):
            del L[k]
    return L


@pytest.mark.parametrize("labels", [True, False])
def test_random_dataset_shuffled_batches_match_the_oracle(labels):
    from oracle import train_inputs_sunrgbd as ots
    rng = np.random.default_rng(31 + labels)
    F, B = 2000, 32
    L = random_sun_lists(F, rng, labels)
    tb = _builder("train" if labels else "rgb", L)
    order = rng.permutation(F)
    total = same = 0
    for k in range(4):
        index = order[k * B: (k + 1) * B]
        index[-1] = index[0]                                             # a repeated index
        np.random.seed(200 + k)
        draws = tb.draw(index)
        assert ("height_u" in draws) and (draws["height_u"] != 0).all() == labels
        out = _host(tb.build(index, draws))
        ref = ots.build("sunrgbd", L, index, draws, SUN, 8.0, random_flip=labels, random_shift=labels,
                        labels=labels)
        margins = ref.pop("_margins", None)
        assert set(out) == set(ref)
        t, s = compare(out, ref, margins, exact=False)
        total, same = total + t, same + s
    assert same >= 0.999 * total, (same, total)
    print("sunrgbd random (labels=%s): %d / %d float values bit-identical to the oracle" % (labels, same, total))


def test_graph_replay_equals_eager():
    rng = np.random.default_rng(6)
    L = random_sun_lists(300, rng)
    tb = _builder("train", L)
    index = [rng.permutation(300)[:16] for _ in range(4)]
    draws = []
    for k in range(4):
        np.random.seed(k)
        draws.append(tb.draw(index[k]))
    eager = [_host(tb.build(index[k], draws[k])) for k in range(4)]
    tb.upload(index[0], draws[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        tb.launch()                                                      # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        tb.launch()
    for k in (1, 2, 3):
        tb.upload(index[k], draws[k])
        graph.replay()
        got = _host(tb.outputs())
        for key in eager[k]:
            assert np.array_equal(got[key], eager[k][key]), (k, key)


def test_training_step_on_the_built_batch_equals_the_reference_batch():
    from train_ref import make_model
    from frustum_convnet_b200.train_engine import TrainStep
    g = load_fixture()
    for mode, index, draws, ref in fixture_batches(g):
        if mode != "train":
            continue
        built = _builder(mode, fixture_lists(g)).build(index, draws)
        losses = []
        for data in (built, _cuda(ref)):
            lo, _ = TrainStep(make_model("sunrgbd", 13)).forward_backward(data)
            torch.cuda.synchronize()
            losses.append({k: float(v) for k, v in lo.items()})
        for k, ref_v in losses[1].items():
            assert abs(losses[0][k] - ref_v) <= 1e-5 * max(1e-6, abs(ref_v)), (k, losses[0][k], ref_v)


def test_validator_on_built_val_batches_equals_the_reference_batches():
    from train_ref import make_model
    from frustum_convnet_b200.validate import Validator
    g = load_fixture()
    m = make_model("sunrgbd", 17).eval()
    v_dev, v_ref = Validator(m), Validator(m)
    n = 0
    for mode, index, draws, ref in fixture_batches(g):
        if mode == "rgb":
            continue
        # the train batches' draws too, built without augmentation: a val split over other items
        val_draws = dict(draws, flip_u=np.zeros_like(draws["flip_u"]), shift_n=np.zeros_like(draws["shift_n"]),
                         height_u=np.zeros_like(draws["height_u"]))
        v_dev.add(_builder("val", fixture_lists(g)).build(index, val_draws))
        want = ref if mode == "val" else oracle_batch(g, "val", index, val_draws)
        v_ref.add(_cuda(want))
        n += 1
    assert n == 3
    a, b = v_dev.finalize(), v_ref.finalize()
    assert list(a) == list(b)
    for k in a:
        assert abs(a[k] - b[k]) <= 1e-5 * max(1e-6, abs(b[k])), (k, a[k], b[k])


def test_rgb_detection_batch_through_the_model_and_the_collector():
    from train_ref import make_model
    from frustum_convnet_b200.detect import DetectionCollector
    g = load_fixture()
    (mode, index, draws, ref), = [b for b in fixture_batches(g) if b[0] == "rgb"]
    L = fixture_lists(g, labels=False)
    built = _builder(mode, L).build(index, draws)
    bit_identical = all(np.array_equal(built[k].cpu().numpy(), v) for k, v in ref.items())
    m = make_model("sunrgbd", 19).eval()
    B = len(index)
    ids = [100 + int(i) // 3 for i in index]                           # several frustums per image
    types = [L["type_list"][i] for i in index]
    box2d = np.stack([L["box2d_list"][i] for i in index])
    results, outs = [], []
    for data in (built, _cuda(ref)):
        with torch.no_grad():
            o = m(data)
        col = DetectionCollector(ids, types, box2d, dataset="SUNRGBD", method="nms", thresh=0.1)
        col.add(o, data, first=0)
        results.append(col.finalize())
        outs.append([t.float().cpu().numpy() for t in o])
    for j, (got, want) in enumerate(zip(*outs)):
        assert got.shape == want.shape, j
        assert np.abs(got - want).max() <= 2.5e-3 * max(1.0, np.abs(want).max()), j
    assert list(results[0]) == list(results[1])
    if bit_identical:
        for i in results[1]:
            assert list(results[0][i]) == list(results[1][i])
            for c in results[1][i]:
                assert np.array_equal(results[0][i][c], results[1][i][c]), (i, c)
    print("rgb batch bit-identical to the reference: %s; detections %d" %
          (bit_identical, sum(len(r) for d in results[1].values() for r in d.values())))
