"""GPU: the per-image detection step on the device (csrc/detect.cu via frustum_convnet_b200/detect.py) against the
fixtures captured from the reference's ``test()`` and against oracle/detect.py on random inputs.

Bit-exact: foreground positions and the argmax fallback (row counts and order), dropped rows, score, ry, h/w/l and
the box2d columns.  tx, ty, tz: within 1e-5 * max(1, |ref|) (cosf/sinf against numpy).  Keep lists and their order
are exact wherever no pair of the list is within 1e-4 of the IoU threshold or of the bounding-cube test."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu

def _cuda_batches(batches):
    out = []
    for first, outs, rot, rgb, ref in batches:
        d = {"rot_angle": torch.from_numpy(np.asarray(rot).reshape(-1, 1).copy()).cuda()}
        if rgb is not None:
            d["rgb_prob"] = torch.from_numpy(np.asarray(rgb).reshape(-1, 1).copy()).cuda()
        if ref is not None:
            d["ref_center"] = torch.from_numpy(np.asarray(ref).copy()).cuda()
        out.append((first, tuple(torch.from_numpy(np.ascontiguousarray(o)).cuda() for o in outs), d))
    return out


def _device(batches, ids, types, box2d, dataset, method, thresh, **kw):
    from frustum_convnet_b200.detect import DetectionCollector
    col = DetectionCollector(ids, types, box2d, dataset=dataset, method=method, thresh=thresh, **kw)
    for first, outs, d in _cuda_batches(batches):
        col.add(outs, d, first=first)
    return col, col.finalize()


def _flat(res):
    return {(i, c): res[i][c] for i in res for c in res[i]}


def _compare(got, want, pre, dataset, thresh, method):
    """got/want: {(idx, cls): (n, 12)} in dict order; pre: the oracle's lists before NMS.  Returns the keys of the
    lists compared."""
    from oracle import detect as od
    assert list(got) == list(want)
    compared = []
    for k in want:
        w, g = want[k].reshape(-1, 12), got[k]
        if method == "nms" and len(pre[k]) > 1:
            m, edge = od.sparse_pair_margin(od.nms_boxes(np.asarray(pre[k], np.float32).reshape(-1, 12), dataset),
                                            thresh)
            if m < 1e-4 or edge < 1e-4:
                continue
        assert g.shape == w.shape, (k, g.shape, w.shape)
        exact = [0, 1, 2, 3, 7, 8, 9, 10, 11]
        assert np.array_equal(g[:, exact], w[:, exact]), k
        tol = 1e-5 * np.maximum(1.0, np.abs(w[:, 4:7]))
        assert (np.abs(g[:, 4:7] - w[:, 4:7]) <= tol).all(), k
        compared.append(k)
    return compared


@pytest.mark.parametrize("name,dataset", [("kitti", "KITTI"), ("sunrgbd", "SUNRGBD")])
def test_fixtures(name, dataset):
    from oracle import detect as od
    from oracle.make_golden_detect import batches
    from test_detect_cpu import fixture_runs
    g = dict(np.load(os.path.join(GOLDEN_DIR, "detect_%s.npz" % name)))
    ids, types = [int(i) for i in g["id_list"]], [str(t) for t in g["type_list"]]
    thr = float(g["thresh"])
    for method, use_ref, use_rgb, want in fixture_runs(g):
        bt = batches(g, use_ref, use_rgb)
        pre = od.collect(bt, ids, types, list(g["box2d"]), dataset, method)
        pre = {(i, c): pre[i][c] for i in pre for c in pre[i]}
        _, got = _device(bt, ids, types, g["box2d"], dataset, method, thr)
        n = len(_compare(_flat(got), want, pre, dataset, thr, method))
        assert n == len(want), (method, n, len(want))       # the fixtures hold no ambiguous pair


def _random_case(seed, dataset="KITTI"):
    """Lists of 1, 513 and >= 1500 rows plus small clustered ones; T2 = 140."""
    rng = np.random.default_rng(seed)
    T2, NS = 140, 8
    plan = [(1, "Car")] + [(2, "Car")] * 4 + [(3, "Car")] * 12 + [(4, "Pedestrian")] * 3 + [(2, "Cyclist")] * 2
    F = len(plan)
    p1 = rng.uniform(0, 1, (F, T2)).astype(np.float32)
    ctr = rng.normal([0, 1, 20], [3, 0.2, 3], (F, T2, 3))
    size = rng.uniform([3, 1.4, 1.3], [4.5, 1.9, 1.8], (F, T2, 3))
    rot = rng.uniform(-0.5, 0.5, F).astype(np.float32)
    ref = rng.normal([0, 1, 20], [4, 0.3, 6], (F, 3)).astype(np.float32)
    p1[0] = 0.1
    p1[0, 33] = 0.9                                                      # image 1: one row
    p1[1:5] = 0.9                                                        # image 2: 3 * 140 + 93 = 513 rows
    p1[4, 93:] = 0.1
    p1[5:17] = 0.9                                                       # image 3: 12 * 140 = 1680 rows
    head = rng.uniform(-np.pi, np.pi, (F, T2))
    # images 2 and 3: boxes on a 7 m grid (no two cubes overlap), every 5th a copy of its neighbour shifted by
    # 0.4 m (IoU far above the threshold): the oracle stays tractable and the keep lists are unambiguous
    for group in (range(1, 5), range(5, 17)):
        for j, f in enumerate(group):
            rot[f], ref[f] = rot[group[0]], ref[group[0]]
            k = j * T2 + np.arange(T2)
            cell = np.where(k % 5 == 4, k - 1, k)
            ctr[f, :, 0] = -140 + 7.0 * (cell % 40)
            ctr[f, :, 2] = 7.0 * (cell // 40)
            ctr[f, :, 1] = 1.0
            ctr[f, k % 5 == 4, 2] += 0.4
            dup = np.nonzero(k % 5 == 4)[0]
            head[f, dup], size[f, dup] = head[f, dup - 1], size[f, dup - 1]
    cls = np.stack([1 - p1, p1], -1).astype(np.float32)
    outs = [cls, ctr.astype(np.float32), head.astype(np.float32),
            size.astype(np.float32), np.zeros((F, T2, 12), np.float32),
            rng.dirichlet(np.ones(NS), (F, T2)).astype(np.float32)]
    B = 5
    bt = [(s, tuple(o[s:s + B] for o in outs), rot[s:s + B], None, ref[s:s + B]) for s in range(0, F, B)]
    ids = [p[0] for p in plan]
    types = [p[1] for p in plan]
    box2d = rng.uniform(0, 1000, (F, 4)).astype(np.float32)
    return bt, ids, types, box2d


def test_random_lists_of_1_513_and_1680_rows_with_top_k():
    from oracle import detect as od
    bt, ids, types, box2d = _random_case(5)
    thr = 0.25
    det = od.collect(bt, ids, types, list(box2d), "KITTI", "nms")
    pre = {(i, c): det[i][c] for i in det for c in det[i]}
    assert sorted(len(v) for v in pre.values())[:1] == [1] and {513, 1680} <= {len(v) for v in pre.values()}
    want, keeps = od.nms_results(det, thr, "KITTI", "nms")
    assert max(len(k) for k in keeps.values()) == 300                    # truncated at top_k
    _, got = _device(bt, ids, types, box2d, "KITTI", "nms", thr)
    done = _compare(_flat(got), _flat(want), pre, "KITTI", thr, "nms")
    assert {(1, "Car"), (2, "Car"), (3, "Car")} <= set(done), done


def test_two_streams_and_out_of_order_adds_match_one_stream():
    from frustum_convnet_b200.detect import DetectionCollector
    bt, ids, types, box2d = _random_case(6)
    _, ref = _device(bt, ids, types, box2d, "KITTI", "nms", 0.25)
    col = DetectionCollector(ids, types, box2d, dataset="KITTI", method="nms", thresh=0.25)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    cb = _cuda_batches(bt)
    torch.cuda.synchronize()
    for j, (first, outs, d) in enumerate(reversed(cb)):                  # one image is spread over several adds
        with torch.cuda.stream(streams[j % 2]):
            col.add(outs, d, first=first)
    got = col.finalize()
    assert list(_flat(got)) == list(_flat(ref))
    for k, v in _flat(ref).items():
        assert np.array_equal(_flat(got)[k], v), k


def test_graph_captured_add_equals_eager_and_does_not_sync():
    from frustum_convnet_b200.detect import DetectionCollector
    bt, ids, types, box2d = _random_case(7)
    cb = _cuda_batches(bt)
    eager = DetectionCollector(ids, types, box2d, dataset="KITTI", method="nms", thresh=0.25)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for first, outs, d in cb:
            eager.add(outs, d, first=first)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    want = eager.finalize()
    graphed = DetectionCollector(ids, types, box2d, dataset="KITTI", method="nms", thresh=0.25)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            for first, outs, d in cb:
                graphed.add(outs, d, first=first)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graphed.counter.zero_()                                              # capture does not run the kernels
    graph.replay()
    got = graphed.finalize()
    assert list(_flat(got)) == list(_flat(want))
    for k, v in _flat(want).items():
        assert np.array_equal(_flat(got)[k], v), k


def test_overflow_raises_with_the_capacity_needed():
    from oracle import detect as od
    bt, ids, types, box2d = _random_case(8)
    n = sum(len(r) for d in od.collect(bt, ids, types, list(box2d), "KITTI", "nms").values() for r in d.values())
    from frustum_convnet_b200.detect import DetectionCollector
    col = DetectionCollector(ids, types, box2d, dataset="KITTI", method="nms", thresh=0.25, capacity=100)
    for first, outs, d in _cuda_batches(bt):
        col.add(outs, d, first=first)
    with pytest.raises(RuntimeError, match="capacity >= %d" % n):
        col.finalize()


def test_cpu_tensors_raise():
    from frustum_convnet_b200.detect import DetectionCollector
    bt, ids, types, box2d = _random_case(9)
    col = DetectionCollector(ids, types, box2d)
    first, outs, rot, rgb, ref = bt[0]
    with pytest.raises(RuntimeError):
        col.add(tuple(torch.from_numpy(o) for o in outs), {"rot_angle": torch.from_numpy(rot)}, first=first)


def test_end_to_end_model_outputs_to_collector(golden_loader):
    """PointNetDet (eval, hand-written kernels) on a golden car case -> collector, against the oracle fed the same
    outputs."""
    from frustum_convnet_b200.det_base import PointNetDet
    from oracle import detect as od
    g, data, sd, w, cfg = golden_loader("car_small_b3")
    m = PointNetDet(3, num_vec=3)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    m = m.cuda().eval()
    dd = {k: torch.from_numpy(v).cuda() for k, v in data.items()}
    B = dd["point_cloud"].shape[0]
    rot = torch.linspace(-0.3, 0.4, B, device="cuda").reshape(B, 1)
    dd["rot_angle"] = rot
    with torch.no_grad():
        outs = m(dd)
    ids, types, box2d = [11] * B, ["Car"] * B, np.arange(4 * B, dtype=np.float32).reshape(B, 4)
    from frustum_convnet_b200.detect import DetectionCollector
    col = DetectionCollector(ids, types, box2d, dataset="KITTI", method="nms", thresh=0.1)
    col.add(outs, dd, first=0)
    got = col.finalize()
    host = [o.detach().cpu().numpy() for o in outs]
    bt = [(0, tuple(host), rot.cpu().numpy(), None, None)]
    det = od.collect(bt, ids, types, list(box2d), "KITTI", "nms")
    want, _ = od.nms_results(det, 0.1, "KITTI", "nms")
    pre = {(i, c): det[i][c] for i in det for c in det[i]}
    assert len(_compare(_flat(got), _flat(want), pre, "KITTI", 0.1, "nms")) == 1
