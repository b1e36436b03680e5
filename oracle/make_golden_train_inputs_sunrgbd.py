"""TEST INFRASTRUCTURE - generates tests/golden/train_inputs_sunrgbd.npz by running the REFERENCE'S OWN
``datasets.provider_sample_sunrgbd.ProviderDataset.__getitem__`` + ``collate_fn`` (default_collate) with
cfgs/det_sample_sunrgbd.yaml on synthetic lists.  As in oracle/make_golden_train_inputs.py, the instance is created
without its pickle-loading constructor and fed the lists it would have read, in the dtypes sunrgbd/prepare_data.py
writes: points float32 with 6 columns (xyz + rgb), box2d float32, seg labels bool, boxes / sizes / K / Rtilt float64.
np.random is seeded per batch; the draws the reference makes (choice, flip random(), shift randn(), height random())
are recorded and must equal what ``frustum_convnet_b200.train_inputs.draw_items(..., height=True)`` replays from the
same seed.  Seeds are searched so that the batches hit the augmentation clips the tests rely on.
Batches: two augmented train batches, a val-style batch (random_flip = random_shift = False) holding the refs placed
1e-7 m inside / outside the half and full boxes' faces, and a from_rgb_detection batch.
Run in the authoring container only (needs the reference tree):  python -m oracle.make_golden_train_inputs_sunrgbd"""
import os

import numpy as np

from .make_golden_train_inputs import ROOT, _Recorder, _reference
from .train_inputs_sunrgbd import project_image_to_upright_camera
from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES, compute_box_3d, draw_items, rotate_pc_along_y

EPS = 1e-7                      # refs placed this far inside / outside a face
MAX_DEPTH = 8.0
K_CAM = np.array([[529.5, 0.0, 365.0], [0.0, 531.25, 262.5], [0.0, 0.0, 1.0]])      # f_u != f_v


def _rtilt(ax, az):
    """A camera tilt: rotation about the depth frame's x (pitch) then z axes (upright depth <- depth)."""
    cx, sx, cz, sz = np.cos(ax), np.sin(ax), np.cos(az), np.sin(az)
    return np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])


class _Recorder4(_Recorder):
    """_Recorder with the SUN-RGBD provider's fourth draw: the random() after randn() is the height shift."""

    def draws(self, B, N):
        out = {"choice": np.zeros((B, N), np.int64), "flip_u": np.zeros(B), "shift_n": np.zeros(B),
               "height_u": np.zeros(B)}
        b, after_randn = -1, False
        for name, v in self.calls:
            if name == "choice":
                b, after_randn = b + 1, False
                out["choice"][b] = v
            elif name == "randn":
                out["shift_n"][b], after_randn = v, True
            else:
                out["height_u" if after_randn else "flip_u"][b] = v
        assert b == B - 1
        return out


def _search_seed(start, counts, index, N, aug, pred):
    for seed in range(start, start + 200000):
        np.random.seed(seed)
        if pred(draw_items(counts, index, N, aug, aug, height=True)):
            return seed
    raise RuntimeError("no seed found")


def _box2d_f32(rng, u, v):
    """float32 box around (u, v) whose centre (box[0] + box[2]) / 2. rounds differently in float32 than in float64."""
    while True:
        b = np.array([u - rng.uniform(20, 60), v - rng.uniform(15, 45), u + rng.uniform(20, 60),
                      v + rng.uniform(15, 45)]).astype(np.float32)
        if (b[0] + b[2]) / 2. != (np.float64(b[0]) + np.float64(b[2])) / 2.:
            return b


def _frustum_angle(box2d, K, R):
    """sunrgbd/prepare_data.py: the angle of the box-2D centre's ray at depth 20 in the upright camera."""
    uvd = np.zeros((1, 3))
    uvd[0, :2] = [(box2d[0] + box2d[2]) / 2.0, (box2d[1] + box2d[3]) / 2.0]
    uvd[0, 2] = 20
    c = project_image_to_upright_camera(uvd, K, R)
    return -1 * np.arctan2(c[0, 2], c[0, 0])


def _image_of(C, K, R):
    """Pixel (u, v) of an upright-camera point: the inverse of project_image_to_upright_camera."""
    up = np.array([C[0], C[2], -C[1]])                  # upright camera (X, Y, Z) -> upright depth (X, Z, -Y)
    d = R.T @ up                                        # -> depth
    cam = np.array([d[0], -d[2], d[1]])                 # depth (x, z, -y) -> camera (x, y, z)
    return K[0, 0] * cam[0] / cam[2] + K[0, 2], K[1, 1] * cam[1] / cam[2] + K[1, 2]


def sunrgbd_dataset(rng):
    """12 frustums over several classes: n = 1, n < N, n = N, n > N; GT near depth 0 and 8; a GT off the ray
    (argmin fallback, i = 9); refs 1e-7 m inside / outside the half and the full box's y faces (i = 4..7); every
    Rtilt tilted, every box2d centre different in float32 and float64."""
    counts = [1, 300, 2048, 2300, 420, 380, 450, 400, 350, 500, 260, 330]
    classes = ["chair", "bed", "table", "sofa", "chair", "desk", "night_stand", "dresser", "toilet", "chair",
               "bookshelf", "bathtub"]
    L = {k: [] for k in ("input_list", "label_list", "box3d_list", "heading_list", "size_list", "frustum_angle_list",
                         "box2d_list", "calib_K_list", "calib_R_list", "type_list", "prob_list")}
    for i, n in enumerate(counts):
        K = K_CAM + np.diag([rng.normal(0, 3), rng.normal(0, 3), 0.0])
        R = _rtilt(rng.uniform(0.03, 0.12), rng.uniform(-0.04, 0.04))
        size = np.array([rng.uniform(0.5, 2.0), rng.uniform(0.5, 2.0), rng.uniform(0.5, 1.5)])
        z = {2: 0.35, 3: 7.75}.get(i, rng.uniform(1.5, 6.5))
        C0 = np.array([0.05 if i in (2, 3) else rng.uniform(-1.5, 1.5), rng.uniform(-0.3, 1.0), z])
        box2d = _box2d_f32(rng, *_image_of(C0, K, R))
        angle = _frustum_angle(box2d, K, R)
        rot = np.pi / 2.0 + angle
        heading = rng.uniform(-np.pi, np.pi)                       # centre-view heading
        if i in (4, 5, 6, 7, 9):
            # the centre-view ref2 of this frustum (float64, as the provider computes it), GT placed against it
            s2 = 0.2
            zz = np.arange(0, MAX_DEPTH, s2) + s2 / 2.
            xyz = np.zeros((len(zz), 3))
            xyz[:, 0], xyz[:, 1], xyz[:, 2] = (box2d[0] + box2d[2]) / 2., (box2d[1] + box2d[3]) / 2., zz
            ref2 = rotate_pc_along_y(project_image_to_upright_camera(xyz, K, R), rot)
            p = ref2[int(np.argmin(np.abs(zz - 3.3)))]
            if i == 9:
                Cv = p + np.array([1.6, 0.0, 0.0])                 # 1.6 m off the ray: no ref inside either box
                size = np.array([0.6, 0.55, 0.8])
            else:
                fac = 0.5 if i in (4, 5) else 1.0
                e = -EPS if i in (4, 6) else EPS
                Cv = p - np.array([0.0, size[2] * fac / 2 + e, 0.0])
        else:
            Cv = rotate_pc_along_y(C0[None, :], rot)[0]
        C = rotate_pc_along_y(Cv[None, :], -rot)[0]
        pts = np.concatenate([C + rng.normal(0, 0.5, (n, 3)) * np.array([1.0, 0.5, 1.0]),
                              rng.integers(0, 256, (n, 3)) / 255.0], 1)
        L["input_list"].append(pts.astype(np.float32))
        L["label_list"].append(rng.uniform(0, 1, n) < 0.4)
        L["box3d_list"].append(compute_box_3d(C, size, heading + rot))
        L["heading_list"].append(float(heading + rot))
        L["size_list"].append(size)
        L["frustum_angle_list"].append(angle)
        L["box2d_list"].append(box2d)
        L["calib_K_list"].append(K)
        L["calib_R_list"].append(R)
        L["type_list"].append(classes[i])
        L["prob_list"].append(float(rng.uniform(0.2, 1.0)))
    return L


def _store_lists(g, L):
    counts = np.array([len(p) for p in L["input_list"]])
    g["counts"], g["points"] = counts, np.concatenate(L["input_list"])
    g["label_list"] = np.concatenate(L["label_list"])
    g["type_list"] = np.array(L["type_list"])
    g["box2d_list"] = np.stack(L["box2d_list"])                                  # float32, as prepare_data.py writes
    for n in ("box3d_list", "heading_list", "size_list", "frustum_angle_list", "calib_K_list", "calib_R_list",
              "prob_list"):
        g[n] = np.asarray(L[n], dtype=np.float64)


def make_sunrgbd(path):
    cfg = _reference("det_sample_sunrgbd.yaml")
    from datasets import provider_sample_sunrgbd as ps  # type: ignore
    rng = np.random.default_rng(2027)
    L = sunrgbd_dataset(rng)
    N, strides = cfg.DATA.NUM_SAMPLES, tuple(cfg.DATA.STRIDE)
    counts = [len(p) for p in L["input_list"]]
    dist = [np.sqrt(np.sum(s[0] ** 2 + s[1] ** 2)) for s in L["size_list"]]
    g = {"classes": np.array(SUNRGBD_CLASSES), "numpy_version": np.array(np.__version__), "npoints": np.int64(N),
         "strides": np.array(strides, dtype=np.float64), "max_depth": np.float64(cfg.DATA.MAX_DEPTH)}
    _store_lists(g, L)

    def flips(d):
        return (d["flip_u"] > 0.5).any() and (d["flip_u"] <= 0.5).any()

    def heights(d):
        return (d["height_u"] > 0.5).any() and (d["height_u"] < 0.5).any()

    batches = [  # (mode, index, predicate on the draws)
        # frustum 2 sits 0.35 m deep, frustum 3 0.25 m short of max_depth: their shifts clip at 0 / max_depth
        ("train", [2, 1, 9, 0, 2, 10], lambda d: flips(d) and heights(d) and d["shift_n"][0] * dist[2] * 0.2 < -0.6
         and any(n * 0.2 > 0.5 for n in d["shift_n"])),
        ("train", [3, 8, 11, 1, 3], lambda d: flips(d) and heights(d) and d["shift_n"][0] * dist[3] * 0.2 > 0.4
         and any(n * 0.2 < -0.5 for n in d["shift_n"])),
        ("val", [4, 5, 6, 7, 9, 2], lambda d: True),
        ("rgb", [8, 0, 3, 11, 6], lambda d: True),
    ]
    for k, (mode, index, pred) in enumerate(batches):
        ds = object.__new__(ps.ProviderDataset)
        ds.npoints, ds.one_hot, ds.from_rgb_detection = N, True, mode == "rgb"
        ds.random_flip = ds.random_shift = mode == "train"
        for name, v in L.items():
            if mode != "rgb" or name not in ("label_list", "box3d_list", "heading_list", "size_list"):
                setattr(ds, name, v)
        seed = _search_seed(7000 + 1000 * k, counts, index, N, mode == "train", pred)
        np.random.seed(seed)
        with _Recorder4() as rec:
            items = [ds[int(i)] for i in index]
        batch = ps.collate_fn(items)
        d = rec.draws(len(index), N)
        np.random.seed(seed)
        replay = draw_items(counts, index, N, mode == "train", mode == "train", height=True)
        for name in d:
            assert np.array_equal(d[name], replay[name]), name
        g["b%d_mode" % k], g["b%d_index" % k], g["b%d_seed" % k] = np.array(mode), np.array(index), seed
        for name, v in d.items():
            g["b%d_%s" % (k, name)] = v.astype(np.int32) if name == "choice" else v
        for name, v in batch.items():
            g["b%d_ref_%s" % (k, name)] = v.numpy()
    g["n_batches"] = np.int64(len(batches))
    np.savez_compressed(path, **g)


def main():
    path = os.path.join(ROOT, "tests", "golden", "train_inputs_sunrgbd.npz")
    make_sunrgbd(path)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
