"""Seeded synthetic KITTI scenes for the refinement extractor (frustum_convnet_b200/refine_extract.py): 3-D ground-truth
objects with points inside them and in the shell just outside (where the x1.2 enlarged and perturbed boxes cut; the
first object of a frame is a Car with only 3 points near its faces),
label_2 lines, and result lines of jittered detections and false positives.  The calibration and the background of
the scans are oracle/kitti_scan_synth's; everything is a pure function of its seed (numpy's PCG64), so tests
regenerate the scans and compare a checksum instead of storing them."""
from __future__ import annotations

import numpy as np

from oracle import kitti_scan_synth as ks

TYPES = ("Car", "Car", "Car", "Car", "Pedestrian", "car", "Van", "DontCare")


def rect_to_velo(calib, pts):
    """(n, 3) rect camera points -> (n, 3) Velodyne points (inverse of R0_rect and Tr_velo_to_cam)."""
    V = np.asarray(calib["Tr_velo_to_cam"]).reshape(3, 4)
    R0 = np.asarray(calib["R0_rect"]).reshape(3, 3)
    ref = np.linalg.solve(R0, pts.T).T
    return (ref - V[:, 3]) @ V[:, :3]


def _box2d(calib, a, hw):
    """The 2-D box of box array a's corners projected with P2, clipped to the image."""
    from frustum_convnet_b200.refine_extract import compute_box_3d_obj_array
    P = np.asarray(calib["P2"]).reshape(3, 4)
    c = compute_box_3d_obj_array(a)
    img = np.concatenate([c, np.ones((8, 1))], 1) @ P.T
    u, v = img[:, 0] / img[:, 2], img[:, 1] / img[:, 2]
    return [float(np.clip(u.min(), 0, hw[1] - 1)), float(np.clip(v.min(), 0, hw[0] - 1)),
            float(np.clip(u.max(), 0, hw[1] - 1)), float(np.clip(v.max(), 0, hw[0] - 1))]


def _points_in(rng, a, n, lo, hi):
    """n points of box array a = [cx, cy, cz, l, w, h, ry] at relative extents in [lo, hi) of the box (by rejection)."""
    out = []
    while sum(len(o) for o in out) < n:
        q = rng.uniform(-hi / 2, hi / 2, (4 * n, 3))
        r = np.max(np.abs(q), 1) * 2
        q = q[r >= lo][: n]
        lx, ly, lz = q[:, 0] * a[3], q[:, 1] * a[5], q[:, 2] * a[4]
        c, s = np.cos(a[6]), np.sin(a[6])
        out.append(np.stack([c * lx + s * lz + a[0], ly + a[1], -s * lx + c * lz + a[2]], 1))
    return np.concatenate(out)[:n] if out else np.zeros((0, 3))


def _line(typ, trunc, occ, box2d, h, w, l, t, ry, score=None):
    s = "%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
        (typ, trunc, occ, -10.0) + tuple(box2d) + (h, w, l) + tuple(t) + (ry,))
    return s if score is None else s + " %.6f" % score


def scene(seed, n_objects=6, n_points=20000):
    """One frame: (scan, calib, (H, W), label lines, result lines)."""
    rng = np.random.default_rng(seed)
    calib = ks.kitti_calib(rng)
    hw = (int(rng.integers(370, 376)), int(rng.integers(1224, 1243)))
    labels, results, parts = [], [], []
    for k in range(n_objects):
        typ = "Car" if k == 0 else TYPES[int(rng.integers(0, len(TYPES)))]
        l, w, h = rng.uniform(3.2, 4.6), rng.uniform(1.5, 1.9), rng.uniform(1.4, 1.7)
        if typ == "Pedestrian":
            l, w, h = rng.uniform(0.5, 1.0), rng.uniform(0.5, 0.8), rng.uniform(1.5, 1.9)
        t = np.array([rng.uniform(-12, 12), 1.65 + rng.normal(0, 0.05), rng.uniform(7, 45)]).round(2)
        l, w, h, ry = round(l, 2), round(w, 2), round(h, 2), round(rng.uniform(-np.pi, np.pi), 2)
        a = np.array([t[0], t[1] - h / 2, t[2], l, w, h, ry])
        box2d = _box2d(calib, a, hw)
        trunc, occ = float(rng.choice([0.0, 0.0, 0.3, 0.6])), int(rng.choice([0, 0, 1, 2, 3]))
        labels.append(_line(typ, trunc, occ, box2d, h, w, l, t, ry))
        if k == 0:           # a sparse object: 3 points near its faces, which a perturbed box can lose altogether
            parts.append(_points_in(rng, a, 3, 0.85, 1.0))
        else:
            parts += [_points_in(rng, a, int(rng.integers(0, 200)), 0.0, 1.0),
                      _points_in(rng, a, int(rng.integers(0, 120)), 1.0, 1.4)]
        if typ != "DontCare" and rng.uniform() < 0.85:           # a detection of this object
            j = lambda x, s: round(float(x) + rng.normal(0, s), 2)
            dt = [j(t[0], 0.3), j(t[1], 0.1), j(t[2], 0.4)]
            b2 = [round(b + rng.normal(0, 2), 2) for b in box2d]
            hj, wj, lj = (max(j(v, sd), 0.1) for v, sd in ((h, 0.1), (w, 0.1), (l, 0.3)))     # positive sizes
            results.append(_line(typ, -1, -1, b2, hj, wj, lj, dt, j(ry, 0.2), rng.uniform()))
    for _ in range(3):                                             # false positives, one with a 2-D box < 5 px tall
        t = [round(rng.uniform(-15, 15), 2), 1.6, round(rng.uniform(6, 50), 2)]
        a = np.array([t[0], 1.6 - 0.75, t[2], 3.9, 1.6, 1.5, 0.3])
        b = _box2d(calib, a, hw)
        if rng.uniform() < 0.3:
            b[3] = b[1] + 4.5
        results.append(_line("Car", -1, -1, b, 1.5, 1.6, 3.9, t, 0.3, rng.uniform()))
    obj = np.concatenate(parts) if parts else np.zeros((0, 3))
    xyz = rect_to_velo(calib, obj)
    pts = np.concatenate([xyz, rng.uniform(0, 1, (len(xyz), 1))], 1).astype(np.float32)
    scan = np.concatenate([ks.kitti_scan(rng, calib, [], max(n_points - len(pts), 0)), pts])
    return scan[rng.permutation(len(scan))], calib, hw, labels, results


def fixture_scenes(z):
    """The frames of tests/golden/refine_extract.npz regenerated from their seeds and checked against the stored
    checksum -> (scans, calibs, image_hw, label lines, result lines), keyed by frame id."""
    ids = z["frame_ids"].tolist()
    scans, calibs, hws = {}, {}, {}
    for idx, seed in zip(ids, z["seeds"].tolist()):
        scans[idx], calibs[idx], hws[idx] = scene(seed)[:3]
    assert ks.checksum([scans[i] for i in ids]) == str(z["checksum"]), "the scene generator drifted from the fixture"
    labels = {i: [str(s) for s in z["labels_%d" % i]] for i in ids}
    results = {i: [str(s) for s in z["results_%d" % i]] for i in ids}
    return scans, calibs, hws, labels, results


def objects(lines):
    """{idx: [line]} -> {idx: [KittiObject]}."""
    from frustum_convnet_b200.refine_extract import KittiObject
    return {k: [KittiObject.parse(ln, "%06d.txt:%d" % (k, n + 1)) for n, ln in enumerate(v)] for k, v in lines.items()}


def large_scene(seed, n_frames=16, n_points=120000, n_objects=8):
    """KITTI-sized frames for the device-vs-oracle tests and the benchmark -> (scans, calibs, image_hw, label lines,
    result lines), keyed by frame id."""
    out = ({}, {}, {}, {}, {})
    for f in range(n_frames):
        idx = 200 + 3 * f
        for d, v in zip(out, scene(seed * 1000 + f, n_objects, n_points)):
            d[idx] = v
    return out
