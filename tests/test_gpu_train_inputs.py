"""GPU: the training-batch builder (C ABI section 11, frustum_convnet_b200/train_inputs.py) against the batches the
reference's own providers + collates produced (tests/golden/train_inputs_{det,refine}.npz) and against the numpy
restatement (oracle/train_inputs.py) on a 2 000-frustum random dataset.  Float outputs must be within one float32 ulp
and >= 99.9 % bit-identical (np.dot goes through BLAS in the reference); int outputs exact; cls_label exact except
for refs within 1e-9 m of a box face.  Also: CUDA-graph replay, two builders on two streams, and one training step on
the built batch against the same step on the reference batch."""
import numpy as np
import pytest
import torch

from test_train_inputs_cpu import compare, fixture_batches, fixture_lists, load_fixture, oracle_batch

pytestmark = pytest.mark.gpu

CAR, PEOPLE, REFINE = (0.25, 0.5, 1.0, 2.0), (0.1, 0.2, 0.4, 0.8), (0.1, 0.2, 0.4, 0.8)


def _builder(kind, strides, N, L, labels=True, max_depth=70.0, classes=("Car", "Pedestrian", "Cyclist")):
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    tb = TrainBatchBuilder(kind, strides, N, max_depth=max_depth, labels=labels)
    tb.set_dataset(L["input_list"], L["type_list"], classes,
                   **{k: v for k, v in L.items() if k not in ("input_list", "type_list")
                      and (kind == "det" or k != "label_list")})
    return tb


def _host(out):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


@pytest.mark.parametrize("name", ["det", "refine"])
def test_builder_matches_the_reference_fixture(name):
    g = load_fixture(name)
    N = int(g["npoints"])
    total = same = 0
    for kind, prefix, strides, index, draws, ref in fixture_batches(g):
        L = fixture_lists(g, prefix)
        tb = _builder(kind, strides, N, L, labels=prefix != "rgb_", max_depth=float(g.get("max_depth", 70.0)))
        out = _host(tb.build(index, draws))
        assert set(out) == set(ref), set(out) ^ set(ref)
        margins = oracle_batch(g, kind, prefix, strides, index, draws).get("_margins")
        t, s = compare(out, ref, margins, exact=False)
        total, same = total + t, same + s
    assert same >= 0.999 * total, (same, total)
    print("%s: %d / %d float values bit-identical to the reference provider" % (name, same, total))


def random_lists(kind, F, rng, labels=True):
    """F random frustums in the reference's dtypes (det points float32, refine train float64, rgb float32)."""
    from frustum_convnet_b200.train_inputs import compute_box_3d
    Pm = np.array([[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791], [0.0, 0.0, 1.0, 0.002745884]])
    L = {}
    n = rng.integers(1, 3000, F)
    size = np.array([3.9, 1.6, 1.5]) * rng.uniform(0.8, 1.2, (F, 3))
    C = np.stack([rng.uniform(-15, 15, F), rng.uniform(0.5, 2.0, F), rng.uniform(1, 69, F)], 1)
    heading = rng.uniform(-np.pi, np.pi, F)
    dtype = np.float64 if kind == "refine" and labels else np.float32
    L["input_list"] = [(C[i] + rng.normal(0, 1.5, (n[i], 3))).astype(dtype) for i in range(F)]
    L["type_list"] = ["Car"] * F
    L["box3d_list"] = [compute_box_3d(C[i], size[i], heading[i]) for i in range(F)]
    L["heading_list"] = [float(h) for h in heading]
    L["size_list"] = list(size)
    if kind == "det":
        L["label_list"] = [(rng.uniform(0, 1, k) < 0.3).astype(np.float64) for k in n]
        L["frustum_angle_list"] = [float(-np.arctan2(c[2], c[0]) + rng.normal(0, 0.02)) for c in C]
        P = [Pm + rng.normal(0, 0.5, (3, 4)) * (Pm != 0) for _ in range(F)]
        L["calib_list"] = [{"P2": p.reshape(-1)} for p in P]
        uv = [(p[0, 0] * c[0] + p[0, 2] * c[2] + p[0, 3]) / c[2] for p, c in zip(P, C)]
        vv = [(p[1, 1] * c[1] + p[1, 2] * c[2] + p[1, 3]) / c[2] for p, c in zip(P, C)]
        L["box2d_list"] = [np.array([u - 40, v - 30, u + 40, v + 30]) for u, v in zip(uv, vv)]
    else:
        pa = heading + rng.normal(0, 0.2, F)
        psize = size * rng.uniform(0.8, 1.2, (F, 3))
        psize[:, 1] = rng.uniform(0.3, 2.5, F)
        L["pred_box3d_list"] = [compute_box_3d(C[i] + rng.normal(0, 0.3, 3), psize[i], pa[i]) for i in range(F)]
        L["pred_box3d_size_list"] = list(psize)
        L["pred_box3d_angle_list"] = [float(a) for a in pa]
        L["prob_list"] = [float(p) for p in rng.uniform(0.1, 1.0, F)]
        if not labels:
            for k in ("box3d_list", "heading_list", "size_list"):
                del L[k]
    return L


@pytest.mark.parametrize("kind,labels", [("det", True), ("refine", True), ("refine", False)])
def test_random_dataset_shuffled_batches_match_the_oracle(kind, labels):
    from oracle import train_inputs as oti
    rng = np.random.default_rng(11 + labels)
    F, B = 2000, 32
    L = random_lists(kind, F, rng, labels)
    strides, N = (CAR, 1024) if kind == "det" else (REFINE, 512)
    tb = _builder(kind, strides, N, L, labels=labels)
    order = rng.permutation(F)
    total = same = 0
    for k in range(4):
        index = order[k * B: (k + 1) * B]
        index[-1] = index[0]                                             # a repeated index
        np.random.seed(100 + k)
        draws = tb.draw(index)
        out = _host(tb.build(index, draws))
        ref = oti.build(kind, L, index, draws, strides, 70.0, labels=labels)
        margins = ref.pop("_margins", None)
        assert set(out) == set(ref)
        t, s = compare(out, ref, margins, exact=False)
        total, same = total + t, same + s
    assert same >= 0.999 * total, (same, total)


def test_graph_replay_and_two_streams_equal_eager():
    rng = np.random.default_rng(5)
    L = random_lists("refine", 300, rng)
    index = [rng.permutation(300)[:16] for _ in range(4)]
    tb = _builder("refine", REFINE, 512, L)
    draws = []
    for k in range(4):
        np.random.seed(k)
        draws.append(tb.draw(index[k]))
    eager = [_host(tb.build(index[k], draws[k])) for k in range(4)]
    # graph: capture the launch with batch 0 staged, replay with batches 1..3 uploaded
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
    # two builders on two streams, interleaved
    tb2 = _builder("det", CAR, 1024, random_lists("det", 200, rng))
    idx2 = [rng.permutation(200)[:24] for _ in range(2)]
    d2 = [tb2.draw(i) for i in idx2]
    eager2 = [_host(tb2.build(idx2[k], d2[k])) for k in range(2)]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for k in range(2):
        with torch.cuda.stream(s1):
            o1 = tb.build(index[k], draws[k])
        with torch.cuda.stream(s2):
            o2 = tb2.build(idx2[k], d2[k])
        torch.cuda.synchronize()
        for key in eager[k]:
            assert np.array_equal(o1[key].cpu().numpy(), eager[k][key]), (k, key)
        for key in eager2[k]:
            assert np.array_equal(o2[key].cpu().numpy(), eager2[k][key]), (k, key)


def test_training_step_on_the_built_batch_equals_the_reference_batch():
    from frustum_convnet_b200 import config, synth
    from frustum_convnet_b200.det_base import PointNetDet
    from frustum_convnet_b200.train_engine import TrainStep
    g = load_fixture("refine")
    kind, prefix, strides, index, draws, ref = fixture_batches(g)[0]
    tb = _builder(kind, strides, int(g["npoints"]), fixture_lists(g, prefix))
    built = tb.build(index, draws)
    cfg, w = config.load_workload("refine_car")
    sd = synth.make_state_dict(w["arch"], 3, "KITTI", seed=11)
    losses = []
    for data in (built, {k: torch.from_numpy(v).cuda() for k, v in ref.items()}):
        m = PointNetDet(3, num_vec=3)
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
        m = m.cuda().train()
        lo, _ = TrainStep(m).forward_backward(data)
        torch.cuda.synchronize()
        losses.append({k: float(v) for k, v in lo.items()})
    for k, ref_v in losses[1].items():
        assert abs(losses[0][k] - ref_v) <= 1e-5 * max(1e-6, abs(ref_v)), (k, losses[0][k], ref_v)


def test_rejects_bad_inputs():
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    g = load_fixture("det")
    L = fixture_lists(g)
    tb = _builder("det", CAR, int(g["npoints"]), L)
    F = len(L["input_list"])
    d = tb.draw([0, 1])
    with pytest.raises(IndexError):
        tb.build([0, F], d)
    with pytest.raises(IndexError):
        tb.build([-1, 0], d)
    bad = dict(d, choice=d["choice"] + 5000)
    with pytest.raises(IndexError):
        tb.build([0, 1], bad)
    with pytest.raises(TypeError):
        tb.build(torch.tensor([0, 1], device="cuda"), d)
    with pytest.raises(RuntimeError):
        TrainBatchBuilder("det", CAR, 1024, device="cpu")
    with pytest.raises(ValueError):
        tb.set_dataset([np.zeros((0, 3), np.float32)], ["Car"], label_list=[np.zeros(0)], box3d_list=[np.zeros((8, 3))],
                       heading_list=[0.0], size_list=[np.ones(3)], frustum_angle_list=[0.0], box2d_list=[np.zeros(4)],
                       calib_list=[{"P2": np.ones(12)}])
