"""ORACLE (test infrastructure) - fixtures of the per-image detection step (csrc/detect.cu, frustum_convnet_b200/detect.py).

Runs the UNMODIFIED reference ``test()`` of train/test_net_det.py (KITTI) and train/test_net_det_sunrgbd.py
(SUN-RGBD) on stored model outputs and captures the dict it hands to ``write_detection_results``.  Around it:
  * oracle/ref_import.py shims, plus a stub ``ops.pybind11.rbbox_iou`` whose ``rotate_nms_3d_cc`` (= ``cube_nms``) is
    oracle/nms.py (the pybind11 extension needs Boost, which is absent here);
  * a stand-in model returning the stored six-tuples, a list-backed loader and dataset;
  * ``Tensor.cuda`` and ``torch.cuda.synchronize`` are no-ops (the outputs are CPU tensors);
  * ``write_detection_results`` is replaced by a capture; the evaluators (evaluate_*_wrapper, eval_det,
    get_gt_all) by no-ops, so they never run; SUN-RGBD's ``save_file_name`` points into a temp dir.

    python -m oracle.make_golden_detect          # authoring container only (needs /root/reference)

Each fixture holds the inputs of GEN() and, per run (method x optional inputs), the captured dict flattened as
keys (image, class) in dict order, rows per key and the (n, 12) rows."""
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402
from oracle import nms as onms  # noqa: E402

RUNS = [("nms", True, True), ("nms", False, False), ("top", True, False), ("top", False, True)]
THRESH = 0.25


def gen(dataset, seed):
    """Frustum outputs covering the fixture cases (see tests/test_detect_cpu.py)."""
    rng = np.random.default_rng(seed)
    T2, NH, NS, B = 140, 12, (8 if dataset == "KITTI" else 10), 4
    classes = ("Car", "Pedestrian", "Cyclist") if dataset == "KITTI" else ("bed", "table", "chair")
    # frustum -> (image id, class): image 7 spans batches 0 and 2 (frustums 0, 1, 9); image 40 is the long list
    # (frustums 12-16, > 512 rows, > 300 kept); image 5 has one frustum whose rows are all dropped
    plan = [(7, 0), (7, 0), (3, 1), (3, 2), (12, 0), (12, 1), (12, 2), (5, 0), (20, 1), (7, 0), (20, 1), (21, 2),
            (40, 0), (40, 0), (40, 0), (40, 0), (40, 0), (9, 0), (9, 1), (9, 0), (33, 2), (33, 2), (2, 0), (2, 1)]
    F = len(plan)
    ids = np.array([p[0] for p in plan], dtype=np.int64)
    types_ = np.array([classes[p[1]] for p in plan])
    box2d = np.round(rng.uniform(0, 1200, (F, 4)), 2)
    p1 = rng.uniform(0, 1, (F, T2)).astype(np.float32)
    p1[rng.random((F, T2)) < 0.05] = 0.5                                    # exact p0 == p1 ties
    cls = np.stack([1 - p1, p1], -1).astype(np.float32)
    rot = rng.uniform(-0.8, 0.8, F).astype(np.float32)
    rgb = rng.uniform(0.3, 1.0, F).astype(np.float32)
    ref = rng.normal([0, 1, 20], [4, 0.3, 6], (F, 3)).astype(np.float32)
    # boxes in triples: positions 3c, 3c+1, 3c+2 are one box shifted by 0, 0.4 and 0.8 m along z (NMS suppresses
    # and cascades), the triples on a 7 m grid (no other cubes overlap), every frustum at its own height (lists
    # mixing frustums of one image do not collide by chance): no pair is near the IoU threshold or the cube test
    t = np.arange(T2)
    ctr = np.zeros((F, T2, 3))
    ctr[:, :, 0] = -35 + 7.0 * ((t // 3) % 10)
    ctr[:, :, 2] = 5 + 7.0 * (t // 30) + 0.4 * (t % 3)
    ctr[:, :, 1] = 5.0 * np.arange(F)[:, None]
    size = rng.uniform([3, 1.4, 1.3], [4.5, 1.9, 1.8], (F, T2, 3))
    head = rng.uniform(-np.pi, np.pi, (F, T2))
    size, head = size[:, t - t % 3], head[:, t - t % 3]
    # all-background frustums: 3 (argmax tie at two positions -> the first) and 19
    for f in (3, 19):
        cls[f, :, 1] = rng.uniform(0, 0.45, T2)
        cls[f, :, 0] = 1 - cls[f, :, 1]
    cls[3, [17, 90], 1] = 0.49
    cls[3, [17, 90], 0] = 0.51
    # tiny boxes (h, w or l < 0.01) here and there; frustum 7 (image 5) drops everything; one h == float32(0.01)
    tiny = rng.random((F, T2)) < 0.04
    size[tiny, rng.integers(0, 3, tiny.sum())] = 0.005
    size[7, :, 2] = 0.009
    size[0, :, 2] = np.where(np.arange(T2) == 5, np.float32(0.01), size[0, :, 2])
    cls[0, 5] = [0.2, 0.8]
    # the long list: frustums 12-16 all foreground, same rotation and reference centre, boxes on a 7 m grid
    # (no two cubes overlap) except every 7th, a copy of its neighbour shifted by 0.3 m
    for j, f in enumerate(range(12, 17)):
        cls[f, :, 1] = rng.uniform(0.55, 1.0, T2)
        cls[f, :, 0] = 1 - cls[f, :, 1]
        rot[f], rgb[f], ref[f] = rot[12], rgb[12], ref[12]
        k = j * T2 + np.arange(T2)
        cell = np.where(k % 7 == 6, k - 1, k)
        ctr[f, :, 0] = -70 + 7.0 * (cell % 20)
        ctr[f, :, 2] = 7.0 * (cell // 20)
        ctr[f, :, 1] = 1.0
        ctr[f, k % 7 == 6, 0] += 0.3
        size[f] = rng.uniform([3, 1.4, 1.3], [4.5, 1.9, 1.8], (T2, 3))
        dup = np.nonzero(k % 7 == 6)[0]
        size[f, dup], head[f, dup] = size[f, dup - 1], head[f, dup - 1]
    hp = np.zeros((F, T2, NH), dtype=np.float32)
    sp = rng.dirichlet(np.ones(NS), (F, T2)).astype(np.float32)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(cls_probs=f32(cls), center=f32(ctr), heading=f32(head), size=f32(size), heading_probs=hp,
                size_probs=sp, rot_angle=rot, rgb_prob=rgb, ref_center=ref, id_list=ids, type_list=types_,
                box2d=box2d, batch_size=np.int64(B))


def batches(g, use_ref, use_rgb):
    """(first, outputs, rot, rgb or None, ref or None) per batch, in loader order."""
    F, B = len(g["id_list"]), int(g["batch_size"])
    out = []
    for first in range(0, F, B):
        sl = slice(first, min(F, first + B))
        outs = tuple(g[k][sl] for k in ("cls_probs", "center", "heading", "size", "heading_probs", "size_probs"))
        out.append((first, outs, g["rot_angle"][sl], g["rgb_prob"][sl] if use_rgb else None,
                    g["ref_center"][sl] if use_ref else None))
    return out


def flatten(res):
    keys_i, keys_c, counts, rows = [], [], [], []
    for idx in res:
        for ct in res[idx]:
            d = np.asarray(res[idx][ct], dtype=np.float32).reshape(-1, 12)
            keys_i.append(int(idx))
            keys_c.append(str(ct))
            counts.append(len(d))
            rows.append(d)
    return (np.array(keys_i, dtype=np.int64), np.array(keys_c), np.array(counts, dtype=np.int64),
            np.concatenate(rows) if rows else np.zeros((0, 12), np.float32))


def _stub_modules():
    ref_import._install_shims()
    m = types.ModuleType("ops.pybind11.rbbox_iou")
    m.rotate_nms_3d_cc = lambda dets, thresh, top_k=300: onms.rotate_nms_3d_cc(np.asarray(dets), thresh, top_k)

    def _unused(*a, **k):
        raise AssertionError("not part of the captured path")
    m.cube_nms_np = m.bev_nms_np = m.rotate_nms_bev_cc = _unused
    sys.modules[m.__name__] = m
    for name in ("train.sunrgbd_eval.compare_matlab_python_eval", "train.sunrgbd_eval.eval_det"):
        mod = types.ModuleType(name)
        mod.get_gt_all = lambda *a, **k: None
        mod.eval_det = lambda *a, **k: None
        sys.modules[name] = mod


class _Model:
    def __init__(self, outs):
        self.outs, self.i = outs, 0

    def eval(self):
        return self

    def __call__(self, data):
        o = self.outs[self.i]
        self.i += 1
        return tuple(torch.from_numpy(np.ascontiguousarray(x)) for x in o)


class _Loader:
    def __init__(self, items, batch_size):
        self.items, self.batch_size = items, batch_size

    def __len__(self):
        return len(self.items)

    def __iter__(self):
        return iter(self.items)


class _Dataset:
    def __init__(self, g):
        self.id_list = [int(i) for i in g["id_list"]]
        self.type_list = [str(t) for t in g["type_list"]]
        self.box2d_list = [np.asarray(b) for b in g["box2d"]]


def run_reference(dataset, g, method, use_ref, use_rgb):
    import importlib
    modname = "train.test_net_det" if dataset == "KITTI" else "train.test_net_det_sunrgbd"
    drv = importlib.import_module(modname)
    drv.cfg.TEST.METHOD = method
    drv.cfg.TEST.THRESH = THRESH
    captured = []
    drv.write_detection_results = lambda out_dir, det: captured.append(det)
    if dataset == "KITTI":
        drv.evaluate_py_wrapper = drv.evaluate_cuda_wrapper = lambda *a, **k: None
    drv.get_gt_all = lambda *a, **k: None
    drv.eval_det = lambda *a, **k: None
    tmp = tempfile.mkdtemp()
    drv.save_file_name = os.path.join(tmp, "detection.pkl")
    items, outs = [], []
    for first, o, rot, rgb, ref in batches(g, use_ref, use_rgb):
        B = len(rot)
        d = {"point_cloud": torch.zeros((B, 3, 4)), "rot_angle": torch.from_numpy(rot.reshape(B, 1).copy())}
        if rgb is not None:
            d["rgb_prob"] = torch.from_numpy(rgb.reshape(B, 1).copy())
        if ref is not None:
            d["ref_center"] = torch.from_numpy(ref.copy())
        items.append(d)
        outs.append(o)
    drv.test(_Model(outs), _Dataset(g), _Loader(items, int(g["batch_size"])), drv.save_file_name, tmp)
    assert len(captured) == 1
    return captured[0]


def main():
    assert ref_import.reference_available(), "needs /root/reference (authoring container only)"
    _stub_modules()
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.cuda.synchronize = lambda *a, **k: None
    for dataset, name, seed in (("KITTI", "kitti", 61), ("SUNRGBD", "sunrgbd", 62)):
        g = gen(dataset, seed)
        store = dict(g)
        store["thresh"] = np.float64(THRESH)
        store["runs"] = np.array(["%s,%d,%d" % r for r in RUNS])
        for r, (method, use_ref, use_rgb) in enumerate(RUNS):
            res = run_reference(dataset, g, method, use_ref, use_rgb)
            ki, kc, cnt, rows = flatten(res)
            store.update({"run%d_key_idx" % r: ki, "run%d_key_cls" % r: kc, "run%d_counts" % r: cnt,
                          "run%d_rows" % r: rows})
            print(name, method, use_ref, use_rgb, "lists", len(ki), "rows", int(cnt.sum()), "max", int(cnt.max()))
        path = os.path.join(ROOT, "tests", "golden", "detect_%s.npz" % name)
        np.savez_compressed(path, **store)
        print(path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
