"""Seeded synthetic KITTI scenes for the frustum extractor (frustum_convnet_b200/frustum_extract.py): Velodyne scans
(a ground plane, box-shaped objects and clutter, float32 x, y, z, intensity), KITTI-like calibration and 2-D detection
lines.  Everything is a pure function of its seed (numpy's PCG64), so tests regenerate the scans and compare a
checksum instead of storing them.

Two kinds of scene:
  exact      a dyadic calibration (Tr_velo_to_cam an axis permutation with dyadic translation, R0_rect = I, P2 with
             f = 512 and an integer principal point): every product and sum of the projection is exact, so any rounding
             order gives the same u, v and every edge is decided alike by any implementation.  Points are placed exactly
             on box and image edges (exact_scene lists the cases).
  realistic  a tilted, non-dyadic calibration near KITTI's and ~20k-point scans; 2-D boxes are the integer boxes of
             real detection lines with an object placed in each frustum.  `edges_clear` tells whether any u, v lies
             within 1e-9 px of a box or image edge (callers draw again until none does)."""
from __future__ import annotations

import hashlib

import numpy as np

H, W = 375, 1242
CU, CV = 609, 172                       # exact scenes: integer principal point
P03, P13 = 32.0, -16.0                  # and dyadic P2 translations


def exact_calib():
    P = np.array([[512.0, 0, CU, P03], [0, 512.0, CV, P13], [0, 0, 1, 0]])
    V2C = np.array([[0.0, -1, 0, 0.25], [0, 0, -1, -0.5], [1, 0, 0, -0.25]])
    return {"P2": P.reshape(12), "Tr_velo_to_cam": V2C.reshape(12), "R0_rect": np.eye(3).reshape(9)}


def exact_point(u, v, Z=16.0, inten=0.5):
    """The velo point that projects exactly to (u, v) at rect depth Z (a power of two) under exact_calib."""
    X = (Z * (u - CU) - P03) / 512.0
    Y = (Z * (v - CV) - P13) / 512.0
    p = np.array([Z + 0.25, 0.25 - X, -0.5 - Y, inten], dtype=np.float64)
    assert np.array_equal(p.astype(np.float32).astype(np.float64), p), (u, v, Z)
    return p.astype(np.float32)


def _clutter(rng, n):
    x = rng.uniform(-10, 60, n)
    y = rng.uniform(-30, 30, n)
    z = rng.uniform(-1.7, 0.5, n)
    return np.stack([x, y, z, rng.uniform(0, 1, n)], axis=1).astype(np.float32)


def _fill(rng, box, n):
    """n exact points strictly inside box (u, v on a 1/8 px grid, depths 8, 16 or 32)."""
    x0, y0, x1, y1 = box
    u = x0 + rng.integers(1, int((x1 - x0) * 8), n) / 8.0
    v = y0 + rng.integers(1, int((y1 - y0) * 8), n) / 8.0
    Z = rng.choice([8.0, 16.0, 32.0], n)
    return np.stack([exact_point(a, b, c, np.float32(rng.uniform())) for a, b, c in zip(u, v, Z)])


def _line(idx, typ, prob, box):
    return "%06d.png %s %s %s" % (idx, typ, repr(prob), " ".join(repr(float(b)) for b in box))


def exact_scene(seed):
    """-> (frames {idx: (scan, calib, (H, W))}, detection lines).  Cases (frame: what):
    3: u exactly on xmin (kept) and xmax (dropped), v on ymin / ymax likewise; u = 0 (in a box clipped from xmin < 0)
       and u = W; x_velo = 2.0f (dropped) and nextafter(2.0f, 3) (kept); NaN points; a box past the right edge (clipped
       to W - 1: u in [W - 1, W) drops out of it);
    5: a box exactly 5 px tall (kept), one 4.5 px tall and one 0.5 px wide (dropped), a box without points, a Pedestrian
       line (outside a Car whitelist), two overlapping boxes;
    8: no detection;  frames 3 and 5 alternate in the file (detections of a frame are not consecutive)."""
    rng = np.random.default_rng(seed)
    cal = exact_calib()
    b1, bu0, bedge, bx2 = (400, 150, 440, 190), (-20, 195, 30, 215), (1200, 100, 1300, 140), (620, 150, 640, 175)
    p3 = [_clutter(rng, 1500), _fill(rng, b1, 40), _fill(rng, (0, 195, 30, 215), 10), _fill(rng, (1200, 100, 1241, 140), 20)]
    edge = [exact_point(400, 170), exact_point(440, 170), exact_point(420, 150), exact_point(420, 190),
            exact_point(0, 200), exact_point(W, 200), exact_point(1241.5, 120), exact_point(1240.5, 120)]
    for xv in (np.float32(2.0), np.nextafter(np.float32(2.0), np.float32(3))):
        edge.append(np.array([xv, 0.25, -0.5, 0.25], dtype=np.float32))     # X = 0, Y = 0: (CU + 18.3, CV - 9.1)
    nanp = exact_point(420, 170)
    for k in range(3):
        q = nanp.copy()
        q[k] = np.nan
        edge.append(q)
    scan3 = np.concatenate(p3 + [np.stack(edge)])
    scan3 = scan3[rng.permutation(len(scan3))]
    b5, b45, bnarrow, bempty, bped, bo1, bo2 = ((500, 200, 540, 205), (560, 200, 600, 204.5), (700, 200, 700.5, 230),
                                                (300, 5, 360, 40), (800, 180, 840, 240), (900, 150, 960, 200),
                                                (930, 170, 1000, 230))
    p5 = [_clutter(rng, 1500)] + [_fill(rng, b, 30) for b in (b5, b45, bped, bo1, bo2)] + \
         [_fill(rng, (700, 200, 701, 230), 10)]
    scan5 = np.concatenate(p5)
    scan5 = scan5[rng.permutation(len(scan5))]
    scan8 = _clutter(rng, 800)
    frames = {3: (scan3, cal, (H, W)), 5: (scan5, cal, (H, W)), 8: (scan8, cal, (H, W))}
    lines = [_line(3, 2, 0.9, b1), _line(3, "Car", 0.8, bu0), _line(5, 2, 0.7, b5), _line(5, 2, 0.6, b45),
             _line(3, 2, 0.55, bedge), _line(3, 2, 0.5, bx2), _line(5, 2, 0.45, bnarrow), _line(5, 2, 0.4, bempty),
             _line(5, 1, 0.35, bped), _line(5, 2, 0.3, bo1), _line(5, "Car", 0.25, bo2)]
    return frames, lines


def _rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def kitti_calib(rng):
    """A tilted calibration near KITTI's (float64 values with full mantissas)."""
    f = 721.5377 + rng.normal(0, 5)
    P = np.array([[f, 0, 609.5593 + rng.normal(0, 3), 44.85728 + rng.normal(0, 1)],
                  [0, f, 172.854 + rng.normal(0, 3), 0.2163791 + rng.normal(0, 0.05)],
                  [0, 0, 1, 0.002745884 + rng.normal(0, 1e-4)]])
    perm = np.array([[0.0, -1, 0], [0, 0, -1], [1, 0, 0]])
    R = _rot(*rng.normal(0, 0.01, 3)) @ perm
    t = np.array([-0.004069766, -0.07631618, -0.2717806]) + rng.normal(0, 0.01, 3)
    V2C = np.concatenate([R, t[:, None]], axis=1)
    R0 = _rot(*rng.normal(0, 0.005, 3))
    return {"P2": P.reshape(12), "Tr_velo_to_cam": V2C.reshape(12), "R0_rect": R0.reshape(9)}


def _image_to_velo(calib, u, v, depth):
    P = calib["P2"].reshape(3, 4)
    V = calib["Tr_velo_to_cam"].reshape(3, 4)
    R0 = calib["R0_rect"].reshape(3, 3)
    x = ((u - P[0, 2]) * depth) / P[0, 0] + P[0, 3] / (-P[0, 0])
    y = ((v - P[1, 2]) * depth) / P[1, 1] + P[1, 3] / (-P[1, 1])
    ref = np.linalg.solve(R0, np.array([x, y, depth]))
    return V[:, :3].T @ (ref - V[:, 3])


def kitti_scan(rng, calib, boxes, n=20000):
    """~n points: a ground plane 1.73 m below the sensor, a box-shaped object in the frustum of each 2-D box (1.6 x 1.5 x
    3.9 m around the box centre's ray at 6-45 m), a few free-standing objects, uniform clutter."""
    n_obj = 150
    parts = []
    for b in boxes:
        c = _image_to_velo(calib, (b[0] + b[2]) / 2.0, (b[1] + b[3]) / 2.0, rng.uniform(6, 45))
        parts.append(c + rng.uniform(-1, 1, (n_obj, 3)) * np.array([1.95, 0.8, 0.75]))
    for _ in range(4):
        c = np.array([rng.uniform(5, 50), rng.uniform(-15, 15), -0.9])
        parts.append(c + rng.uniform(-1, 1, (n_obj, 3)) * np.array([1.95, 0.8, 0.75]))
    n_rest = max(n - n_obj * len(parts), 0)
    n_ground = n_rest * 3 // 4
    r = np.sqrt(rng.uniform(1, 70 ** 2, n_ground))
    a = rng.uniform(-np.pi, np.pi, n_ground)
    parts.append(np.stack([r * np.cos(a), r * np.sin(a), -1.73 + rng.normal(0, 0.03, n_ground)], axis=1))
    nc = n_rest - n_ground
    parts.append(np.stack([rng.uniform(-80, 80, nc), rng.uniform(-80, 80, nc), rng.uniform(-2, 3, nc)], axis=1))
    xyz = np.concatenate(parts)
    scan = np.concatenate([xyz, rng.uniform(0, 1, (len(xyz), 1))], axis=1).astype(np.float32)
    return scan[rng.permutation(len(scan))]


def edges_clear(u, v, hw, boxes, tol=1e-9):
    """No finite u within tol of 0, W or a clipped box's x edge, and no v likewise (boxes as read, clipped here)."""
    h, w = hw
    ex, ey = [0.0, float(w)], [0.0, float(h)]
    for b in boxes:
        b = np.asarray(b, dtype=np.float64)
        ex += list(np.clip(b[[0, 2]], 0, w - 1))
        ey += list(np.clip(b[[1, 3]], 0, h - 1))
    for c, edges in ((u, ex), (v, ey)):
        c = c[np.isfinite(c)]
        for e in edges:
            if np.any(np.abs(c - e) < tol):
                return False
    return True


def parse_line(line):
    t = line.rstrip().split(" ")
    return t[1], float(t[2]), np.array([float(x) for x in t[3:7]])


def realistic_scene(seed, lines, n=20000):
    """One frame for the detection lines of one image: (scan, calib, (H, W))."""
    rng = np.random.default_rng(seed)
    calib = kitti_calib(rng)
    hw = (int(rng.integers(370, 376)), int(rng.integers(1224, 1243)))
    boxes = [parse_line(ln)[2] for ln in lines]
    return kitti_scan(rng, calib, boxes, n), calib, hw


def fixture_scenes(z, part):
    """The scenes of tests/golden/frustum_extract.npz part 'exact' or 'real', regenerated from their seeds and checked
    against the stored checksum -> (scans, calibs, image_hw, detection lines)."""
    lines = [str(s) for s in z[part + "_lines"]]
    if part == "exact":
        frames, lines2 = exact_scene(int(z["exact_seed"]))
        assert lines2 == lines, "exact_scene's detection lines drifted from the fixture"
    else:
        frames = {}
        for idx, seed in zip(z["real_frame_ids"].tolist(), z["real_seeds"].tolist()):
            own = [ln for ln in lines if det_id(ln) == idx]
            frames[idx] = realistic_scene(seed, own)
    ids = sorted(frames)
    assert checksum([frames[i][0] for i in ids]) == str(z[part + "_checksum"]), \
        "the synthetic scan generator drifted from the fixture"
    return ({i: frames[i][0] for i in ids}, {i: frames[i][1] for i in ids}, {i: frames[i][2] for i in ids}, lines)


def det_id(line):
    return int(line.split(" ", 1)[0].rsplit("/", 1)[-1].split(".")[0])


def large_scene(seed, n_frames=16, n_points=120000, n_dets=30, empty_frame=None):
    """Random scenes for the device-vs-oracle tests and the benchmark: KITTI-like calibration and scans, n_dets boxes a
    frame (random sizes, overlapping, some past the image edge, some tiny), types drawn from Car / Pedestrian /
    Cyclist.  -> (scans, calibs, image_hw, id_list, type_list, prob_list, box2d_list), keyed by frame id; the frame
    `empty_frame` (if given) has no point."""
    rng = np.random.default_rng(seed)
    scans, calibs, hws = {}, {}, {}
    ids, types, probs, boxes = [], [], [], []
    for f in range(n_frames):
        idx = 100 + 7 * f
        calib = kitti_calib(rng)
        hw = (int(rng.integers(370, 376)), int(rng.integers(1224, 1243)))
        h, w = hw
        bx = []
        for _ in range(n_dets):
            bw, bh = np.exp(rng.uniform(np.log(0.4), np.log(400))), np.exp(rng.uniform(np.log(3), np.log(250)))
            x0, y0 = rng.uniform(-60, w + 20), rng.uniform(-30, h + 10)
            bx.append(np.array([x0, y0, x0 + bw, y0 + bh]).round(2))
        scans[idx] = (np.zeros((0, 4), np.float32) if f == empty_frame else
                      kitti_scan(rng, calib, bx[: n_dets // 2], n_points))
        calibs[idx], hws[idx] = calib, hw
        for b in bx:
            ids.append(idx)
            types.append(["Car", "Pedestrian", "Cyclist"][int(rng.integers(0, 3))])
            probs.append(float(rng.uniform()))
            boxes.append(b)
    order = rng.permutation(len(ids))              # frames interleave in the detection list
    pick = lambda a: [a[i] for i in order]
    return scans, calibs, hws, pick(ids), pick(types), pick(probs), pick(boxes)


def checksum(arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()
