"""TEST INFRASTRUCTURE - generates tests/golden/train_inputs_{det,refine}.npz by running the REFERENCE'S OWN
``datasets.provider_sample.ProviderDataset.__getitem__`` + default_collate and
``datasets.provider_sample_refine.ProviderDataset.__getitem__`` + ``collate_fn`` on synthetic lists.  The instances are
created without their pickle-loading constructors and fed the lists they would have read, in the dtypes the
reference's prepare scripts write (detection points float32, refine train points float64, refine rgb-detection points
float32, boxes / sizes / seg labels float64).  np.random is seeded per batch; the draws the reference makes are
recorded and must equal what ``frustum_convnet_b200.train_inputs.draw_items`` replays from the same seed.  Seeds are
searched so that the batches hit the augmentation clips the tests rely on.
Run in the authoring container only (needs the reference tree):  python -m oracle.make_golden_train_inputs"""
import os
import sys

import numpy as np

from . import ref_import
from frustum_convnet_b200.train_inputs import compute_box_3d, draw_items, rotate_pc_along_y

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLASSES = ["Car", "Pedestrian", "Cyclist"]
CAR_SIZE = np.array([3.9, 1.6, 1.5])
EPS = 1e-7                      # refs placed this far inside / outside a face


def _reference(yaml_name):
    ref_import._install_shims()
    for k in [k for k in sys.modules if k.startswith(("configs", "models", "datasets"))]:
        del sys.modules[k]
    from configs.config import cfg, merge_cfg_from_file  # type: ignore
    merge_cfg_from_file(os.path.join(ref_import.REF, "cfgs", yaml_name))
    return cfg


class _Recorder:
    """Wraps np.random.choice / random / randn while the reference draws, keeping the values in call order."""

    def __init__(self):
        self.calls = []

    def __enter__(self):
        self.saved = (np.random.choice, np.random.random, np.random.randn)
        ch, rd, rn = self.saved

        def choice(*a, **k):
            v = ch(*a, **k)
            self.calls.append(("choice", v))
            return v

        def random(*a, **k):
            v = rd(*a, **k)
            self.calls.append(("random", v))
            return v

        def randn(*a, **k):
            v = rn(*a, **k)
            self.calls.append(("randn", v))
            return v

        np.random.choice, np.random.random, np.random.randn = choice, random, randn
        return self

    def __exit__(self, *exc):
        np.random.choice, np.random.random, np.random.randn = self.saved

    def draws(self, B, N):
        out = {"choice": np.zeros((B, N), np.int64), "flip_u": np.zeros(B), "shift_n": np.zeros(B)}
        b = -1
        for name, v in self.calls:
            if name == "choice":
                b += 1
                out["choice"][b] = v
            else:
                out["flip_u" if name == "random" else "shift_n"][b] = v
        assert b == B - 1
        return out


def _points(rng, n, center, dtype):
    p = center + rng.normal(0, 1.2, (n, 3)) * np.array([1.0, 0.4, 1.0])
    return p.astype(dtype)


def det_dataset(rng):
    """10 detection frustums: n = 1, n < N, n > N, n = N; GT near depth 0 and 70; refs 1e-7 m inside / outside the
    half and the full box's y faces; a GT off the frustum ray (argmin fallback)."""
    Pm = np.array([[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791], [0.0, 0.0, 1.0, 0.002745884]])
    Pf = Pm.copy()
    Pf[0, 2], Pf[1, 2] = 609.5, 172.75            # exact box-2D centre for the face cases
    L = {k: [] for k in ("input_list", "label_list", "box3d_list", "heading_list", "size_list", "frustum_angle_list",
                         "box2d_list", "calib_list", "type_list")}
    counts = [1, 300, 2000, 1024, 600, 650, 500, 550, 700, 400]
    for i, n in enumerate(counts):
        size = CAR_SIZE * rng.uniform(0.9, 1.1, 3)
        if i in (4, 5, 6, 7):
            P = Pf
            b_x, b_y = P[0, 3] / (-P[0, 0]), P[1, 3] / (-P[1, 1])
            fac = 0.5 if i in (4, 5) else 1.0
            e = -EPS if i in (4, 6) else EPS
            C = np.array([b_x, b_y - (size[2] * fac / 2 + e), 20.1 + 0.37 * i])
            angle = -np.pi / 2
            heading = np.pi / 2 + (np.pi / 2.0 + angle)    # length along the ray in the centre view
            box2d = np.array([P[0, 2] - 50, P[1, 2] - 40, P[0, 2] + 50, P[1, 2] + 40])
        else:
            P = Pm + rng.normal(0, 0.5, (3, 4)) * (Pm != 0)
            z = {2: 0.3, 3: 69.8}.get(i, rng.uniform(8, 50))
            C = np.array([0.05 if i in (2, 3) else rng.uniform(-8, 8), rng.uniform(0.8, 1.8), z])
            angle = -np.arctan2(C[2], C[0])
            heading = rng.uniform(-np.pi, np.pi)
            u = (P[0, 0] * C[0] + P[0, 2] * C[2] + P[0, 3]) / (C[2] + P[2, 3])
            v = (P[1, 1] * C[1] + P[1, 2] * C[2] + P[1, 3]) / (C[2] + P[2, 3])
            box2d = np.array([u - 40, v - 30, u + 40, v + 30])
            if i == 8:                                     # GT 2.5 m off the ray: no ref inside either box
                rot = np.pi / 2 + angle
                off = rotate_pc_along_y(np.array([[2.5, 0.0, 0.0]]), -rot)[0]
                C = C + off
        L["input_list"].append(_points(rng, n, C, np.float32))
        L["label_list"].append((rng.uniform(0, 1, n) < 0.4).astype(np.float64))
        L["box3d_list"].append(compute_box_3d(C, size, heading))
        L["heading_list"].append(float(heading))
        L["size_list"].append(size)
        L["frustum_angle_list"].append(float(angle))
        L["box2d_list"].append(box2d)
        L["calib_list"].append({"P2": P.reshape(-1)})
        L["type_list"].append("Car")
    return L


def refine_dataset(rng, labels):
    """Refinement frustums: predicted-box widths giving a different T at every scale (0.8 is an exact multiple of every
    stride), refs 1e-7 m inside / outside the 0.3x and 0.6x boxes' y faces, a GT off the predicted box's line."""
    widths = [1.55, 0.8, 1.6, 2.0, 1.3, 0.45, 1.75, 1.2]
    counts = [1, 200, 512, 900, 350, 60, 700, 480]
    L = {k: [] for k in ("input_list", "box3d_list", "heading_list", "size_list", "type_list", "pred_box3d_list",
                         "pred_box3d_size_list", "pred_box3d_angle_list", "prob_list", "label_list")}
    for i, (w, n) in enumerate(zip(widths, counts)):
        pc = np.array([rng.uniform(-8, 8), rng.uniform(0.8, 1.8), rng.uniform(6, 50)])
        pa = rng.uniform(-np.pi, np.pi)
        psize = np.array([rng.uniform(3.4, 4.4), w, rng.uniform(1.3, 1.7)])
        pred = compute_box_3d(pc, psize, pa)
        pc_exact = (pred[0, :] + pred[6, :]) / 2
        size = CAR_SIZE * rng.uniform(0.9, 1.1, 3)
        if labels and i in (2, 3, 4, 6):
            fac = 0.3 if i in (2, 3) else 0.6
            e = -EPS if i in (2, 4) else EPS
            C = pc_exact + np.array([0.0, -(size[2] * fac / 2 + e), 0.0])
            heading = pa + np.pi / 2
        else:
            off = np.array([1.0, 0.0, 0.0]) if i == 5 else rng.normal(0, 0.15, 3)
            C = pc_exact + rotate_pc_along_y(off[None, :], -pa)[0]
            heading = pa + rng.normal(0, 0.2)
        L["input_list"].append(_points(rng, n, pc, np.float64 if labels else np.float32))
        L["box3d_list"].append(compute_box_3d(C, size, heading))
        L["heading_list"].append(float(heading))
        L["size_list"].append(size)
        L["type_list"].append("Car")
        L["pred_box3d_list"].append(pred)
        L["pred_box3d_size_list"].append(psize)
        L["pred_box3d_angle_list"].append(float(pa))
        L["prob_list"].append(float(rng.uniform(0.2, 1.0)))
        L["label_list"].append(np.zeros(n))
    return L


def _search_seed(start, counts, index, N, flip, shift, pred):
    for seed in range(start, start + 200000):
        np.random.seed(seed)
        d = draw_items(counts, index, N, flip, shift)
        if pred(d):
            return seed
    raise RuntimeError("no seed found")


def _run(ds, index, seed, N, collate):
    np.random.seed(seed)
    with _Recorder() as rec:
        items = [ds[int(i)] for i in index]
    batch = collate(items)
    d = rec.draws(len(index), N)
    counts = [len(p) for p in ds.input_list]
    np.random.seed(seed)
    replay = draw_items(counts, index, N, ds.random_flip and not ds.from_rgb_detection,
                        ds.random_shift and not ds.from_rgb_detection)
    for k in d:
        assert np.array_equal(d[k], replay[k]), k
    return {k: (v.numpy() if hasattr(v, "numpy") else np.asarray(v)) for k, v in batch.items()}, d


def _store_lists(g, prefix, L, names):
    counts = np.array([len(p) for p in L["input_list"]])
    g[prefix + "counts"] = counts
    g[prefix + "points"] = np.concatenate(L["input_list"])
    for n in names:
        if n == "calib_list":
            g[prefix + n] = np.stack([c["P2"] for c in L[n]])
        elif n == "label_list":
            g[prefix + n] = np.concatenate(L[n])
        elif n == "type_list":
            g[prefix + n] = np.array(L[n])
        else:
            g[prefix + n] = np.asarray(L[n], dtype=np.float64)


def make_det(path):
    from torch.utils.data.dataloader import default_collate
    cfg = _reference("det_sample.yaml")
    from datasets import provider_sample as ps  # type: ignore
    from datasets.dataset_info import DATASET_INFO  # type: ignore
    rng = np.random.default_rng(2025)
    L = det_dataset(rng)
    ds = object.__new__(ps.ProviderDataset)
    ds.npoints, ds.one_hot, ds.from_rgb_detection = cfg.DATA.NUM_SAMPLES, True, False
    ds.random_flip, ds.random_shift = True, True
    ds.category_info = DATASET_INFO[cfg.DATA.DATASET_NAME]
    for k, v in L.items():
        setattr(ds, k, v)
    N = cfg.DATA.NUM_SAMPLES
    counts = [len(p) for p in L["input_list"]]
    g = {"classes": np.array(CLASSES), "numpy_version": np.array(np.__version__), "npoints": np.int64(N)}
    _store_lists(g, "", L, [k for k in L if k != "input_list"])
    car, people = tuple(cfg.DATA.STRIDE), (0.1, 0.2, 0.4, 0.8)
    batches = [  # (strides, index, predicate on the draws)
        (car, [3, 1, 3, 0, 5, 2, 4, 9], lambda d: (d["shift_n"] > 2.6).any() and d["shift_n"][5] < -0.5
         and max(d["shift_n"][0], d["shift_n"][2]) > 0.5 and (d["flip_u"] > 0.5).any() and (d["flip_u"] <= 0.5).any()),
        (car, [6, 7, 8, 2, 3, 0, 4, 5], lambda d: (d["shift_n"] < -2.6).any()
         and (d["flip_u"] > 0.5).any() and (d["flip_u"] <= 0.5).any()),
        (people, [7, 4, 6, 5, 8, 1, 2, 3], lambda d: (d["flip_u"] > 0.5).any() and (d["flip_u"] <= 0.5).any()),
    ]
    for k, (strides, index, pred) in enumerate(batches):
        cfg.DATA.STRIDE = strides
        seed = _search_seed(1000 * (k + 1), counts, index, N, True, True, pred)
        out, d = _run(ds, index, seed, N, default_collate)
        g["b%d_strides" % k], g["b%d_index" % k], g["b%d_seed" % k] = np.array(strides), np.array(index), seed
        for name, v in d.items():
            g["b%d_%s" % (k, name)] = v.astype(np.int32) if name == "choice" else v
        for name, v in out.items():
            g["b%d_ref_%s" % (k, name)] = v
    g["max_depth"] = np.float64(cfg.DATA.MAX_DEPTH)
    g["n_batches"] = np.int64(len(batches))
    np.savez_compressed(path, **g)


def make_refine(path):
    cfg = _reference("refine_car.yaml")
    from datasets import provider_sample_refine as pr  # type: ignore
    from datasets.dataset_info import DATASET_INFO  # type: ignore
    rng = np.random.default_rng(2026)
    N = cfg.DATA.NUM_SAMPLES
    g = {"classes": np.array(CLASSES), "numpy_version": np.array(np.__version__), "npoints": np.int64(N),
         "strides": np.array(cfg.DATA.STRIDE, dtype=np.float64)}
    k = 0
    for labels, prefix in ((True, "train_"), (False, "rgb_")):
        L = refine_dataset(rng, labels)
        ds = object.__new__(pr.ProviderDataset)
        ds.npoints, ds.one_hot, ds.from_rgb_detection = N, True, not labels
        ds.random_flip, ds.random_shift = True, True
        ds.category_info = DATASET_INFO[cfg.DATA.DATASET_NAME]
        for name, v in L.items():
            setattr(ds, name, v)
        _store_lists(g, prefix, L, [n for n in L if n not in ("input_list", "label_list")])
        counts = [len(p) for p in L["input_list"]]
        s1 = cfg.DATA.STRIDE[0]
        dist = [np.sqrt(np.sum(s[0] ** 2 + s[1] ** 2)) for s in L["size_list"]]
        if labels:
            batches = [[2, 5, 2, 0, 7, 3], [1, 4, 6, 0, 3, 5]]
            preds = [lambda d, ix: any(n * dist[i] * 0.1 > 2 * s1 for n, i in zip(d["shift_n"], ix))
                     and any(n * dist[i] * 0.1 < -2 * s1 for n, i in zip(d["shift_n"], ix))
                     and (d["flip_u"] > 0.5).any() and (d["flip_u"] <= 0.5).any()] * 2
        else:
            batches, preds = [[4, 0, 2, 5, 1, 3, 4]], [lambda d, ix: True]
        for index, pred in zip(batches, preds):
            seed = _search_seed(5000 + 1000 * k, counts, index, N, labels, labels, lambda d, ix=index: pred(d, ix))
            out, d = _run(ds, index, seed, N, pr.collate_fn)
            g["b%d_kind" % k] = np.array(prefix[:-1])
            g["b%d_index" % k], g["b%d_seed" % k] = np.array(index), seed
            for name, v in d.items():
                g["b%d_%s" % (k, name)] = v.astype(np.int32) if name == "choice" else v
            for name, v in out.items():
                g["b%d_ref_%s" % (k, name)] = v
            k += 1
    g["n_batches"] = np.int64(k)
    np.savez_compressed(path, **g)


def main():
    for name, fn in (("det", make_det), ("refine", make_refine)):
        path = os.path.join(ROOT, "tests", "golden", "train_inputs_%s.npz" % name)
        fn(path)
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
