"""TEST INFRASTRUCTURE ONLY - seeded SUN-RGBD frames for the frustum extractor: an (n, 6) float32 cloud (x, y, z,
r, g, b in upright depth coordinates), a calibration (tilted Rtilt, K with f_u != f_v) and label lines as the
reference's label files hold them ('class xmin ymin w h cx cy cz w l h b00 b01 b10 b11 o0 o1', l, w, h half extents).

The cloud is a depth grid (one point per pixel of an H x W image, at a random sub-pixel position and a smooth depth of
3-6 m, back-projected through K and Rtilt) plus, for each object, points drawn inside its 3-D box, which sits 1.2-2 m
from the camera.  An object's 2-D box is centred on its projection with a chosen size, so the frustum's point count
follows the box area (one grid point per pixel)."""
from __future__ import annotations

import numpy as np

from frustum_convnet_b200 import sunrgbd_extract as sx


def _rot(ax, ay):
    cx, sx_, cy, sy = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay)
    rx = np.array([[1, 0, 0], [0, cx, -sx_], [0, sx_, cx]])
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    return rx @ ry


def calib(rng, H, W):
    Rtilt = _rot(rng.uniform(0.05, 0.15), rng.uniform(-0.08, 0.08))
    fu = 0.75 * W * rng.uniform(0.95, 1.05)
    K = np.array([[fu, 0.0, W / 2 + rng.uniform(-3, 3)], [0.0, fu * rng.uniform(1.02, 1.06), H / 2 +
                  rng.uniform(-3, 3)], [0.0, 0.0, 1.0]])
    return {"Rtilt": Rtilt, "K": K}


def upright_of_pixel(u, v, d, cal):
    """Pixel (u, v) at depth d -> upright depth coordinates (project_image_to_camera, flip_axis_to_depth, Rtilt)."""
    K = cal["K"]
    cam = np.stack([(u - K[0, 2]) * d / K[0, 0], (v - K[1, 2]) * d / K[1, 1], d], -1).reshape(-1, 3)
    depth = sx.flip_axis_to_depth(cam)
    return (cal["Rtilt"] @ depth.T).T


def background(rng, H, W, cal):
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    u = u + rng.uniform(0, 1, u.shape)
    v = v + rng.uniform(0, 1, v.shape)
    a, b = rng.uniform(-1, 1, 2)
    d = 4.5 + a * (u / W - 0.5) + b * (v / H - 0.5) + 0.5 * np.sin(u / 23.0) * np.cos(v / 17.0)
    xyz = upright_of_pixel(u.reshape(-1), v.reshape(-1), d.reshape(-1), cal)
    return np.concatenate([xyz, rng.uniform(0, 1, (len(xyz), 3))], 1).astype(np.float32)


def label_line(cls, box2d, centroid, w, l, h, heading):
    """A label line whose parsed heading_angle is (up to rounding) `heading`: orientation (cos(-t), sin(-t))."""
    xmin, ymin, xmax, ymax = box2d
    vals = [xmin, ymin, xmax - xmin, ymax - ymin, *centroid, w, l, h, 0.0, 0.0, 0.0, 0.0, np.cos(-heading),
            np.sin(-heading)]
    return cls + " " + " ".join(repr(float(x)) for x in vals)


def make_object(rng, cal, cls, uc, vc, box_w, box_h, n_pts, half=None, zero_h=False):
    """An object seen at pixel (uc, vc), 1.2-2 m away, with a box_w x box_h px 2-D box around it and n_pts points in
    its 3-D box (half extents l, w, h from `half` or drawn) -> (label line, (n_pts, 6) float32 points)."""
    d = rng.uniform(1.2, 2.0)
    c = upright_of_pixel(np.array([uc]), np.array([vc]), np.array([d]), cal)[0]
    l, w, h = half if half is not None else rng.uniform(0.1, 0.35, 3)
    if zero_h:
        h = 0.0
    heading = rng.uniform(-np.pi, np.pi)
    box2d = [uc - box_w / 2, vc - box_h / 2, uc + box_w / 2, vc + box_h / 2]
    line = label_line(cls, box2d, c, w, l, h, heading)
    obj = sx.SUNObject3d(line)
    local = rng.uniform(-0.95, 0.95, (n_pts, 3)) * np.array([obj.l, obj.w, obj.h])
    t = -obj.heading_angle
    R = np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1]])
    xyz = local @ R.T + obj.centroid
    return line, np.concatenate([xyz, rng.uniform(0, 1, (n_pts, 3))], 1).astype(np.float32)


def frame(seed, H, W, specs):
    """specs: [(class, uc, vc, box_w, box_h, n_pts, dict(half=..., zero_h=...))] with uc, vc as fractions of W, H ->
    (cloud, calib, label lines).  The object points are interleaved with the grid in a seeded order."""
    rng = np.random.default_rng(seed)
    cal = calib(rng, H, W)
    pts, lines = [background(rng, H, W, cal)], []
    for cls, fu, fv, bw, bh, n, kw in specs:
        line, p = make_object(rng, cal, cls, fu * W, fv * H, bw, bh, n, **kw)
        lines.append(line)
        pts.append(p)
    cloud = np.concatenate(pts)
    return cloud[rng.permutation(len(cloud))], cal, lines


CLASSES = sx.TYPE_WHITELIST


def large_frame(seed, H=530, W=730, n_objects=8):
    """A frame at SUN-RGBD scale: an H x W grid and n_objects objects of the 10 classes plus one lamp, 2-D boxes of
    40-140 px a side (most frustums above 2048 points)."""
    rng = np.random.default_rng(10_000 + seed)
    specs = []
    for k in range(n_objects):
        specs.append((CLASSES[int(rng.integers(len(CLASSES)))], rng.uniform(0.15, 0.85), rng.uniform(0.15, 0.85),
                      rng.uniform(40, 140), rng.uniform(40, 140), int(rng.integers(20, 800)), {}))
    specs.append(("lamp", 0.5, 0.5, 60.0, 60.0, 50, {}))
    return frame(seed, H, W, specs)


def large_set(seed, n_frames=16, **kw):
    """-> (points {idx: cloud}, calibs {idx: calib}, labels {idx: [SUNObject3d]}, detection lists (ids, types,
    boxes, probs): for every label box a detection jittered off it, frames visited twice, non-contiguously)."""
    points, calibs, labels = {}, {}, {}
    for k in range(n_frames):
        idx = k + 1
        points[idx], calibs[idx], lines = large_frame(seed * 100 + k, **kw)
        labels[idx] = [sx.SUNObject3d(ln, "%d:%d" % (idx, n + 1)) for n, ln in enumerate(lines)]
    rng = np.random.default_rng(seed)
    ids, types, boxes, probs = [], [], [], []
    for rep in range(2):
        for idx in labels:
            for o in labels[idx][rep::2]:
                ids.append(idx)
                types.append(o.classname)
                boxes.append(o.box2d + rng.uniform(-4, 4, 4))
                probs.append(float(rng.uniform(0.1, 1.0)))
    return points, calibs, labels, (ids, types, boxes, probs)
