"""ORACLE: extract_frustum_data (sunrgbd/prepare_data.py:132-267) and extract_frustum_data_from_rgb_detection
(:270-381) restated in numpy, job by job in the reference's order, with the reference's generator calls in its order.

Every per-job constant (perturbation, frustum_angle, corners, size, heading, float32 box2d) comes from the host code
the device path uses (frustum_convnet_b200.sunrgbd_extract: the reference's own numpy expressions); the projection is
the reference's np.dot expression.  The labels are the float64 half-space test (in_box below, the test of
csrc/box_contains.cuh on sunrgbd_extract.box_record) instead of scipy's Delaunay over the corners; the two agree except
for points within rounding of a face (the fixture's scenes keep every point more than BAND from every face).
Returns the reference's dict (its keys) and a per-job trace (frame, n, labelled points in the box and among the kept
ones, skipped, choice drawn, kept)."""
from __future__ import annotations

import numpy as np

from frustum_convnet_b200 import sunrgbd_extract as sx

BAND = 1e-9           # m: no point this close to a face of a whitelisted label box
EDGE_BAND = 1e-7      # px: no point this close to an edge of a cutting box


def camera_points(pc):
    """pc_upright_camera of the reference: (x, -z, y, r, g, b), float32."""
    out = np.zeros_like(pc)
    out[:, 0:3] = sx.flip_axis_to_camera(pc[:, 0:3])
    out[:, 3:] = pc[:, 3:]
    return out


def image_coords(pc, calib):
    Rtilt, K = sx.calib_mats(calib)
    return sx.project_upright_depth_to_image(pc, Rtilt, K)


def cut(uv, box):
    xmin, ymin, xmax, ymax = box
    return (uv[:, 0] < xmax) & (uv[:, 0] >= xmin) & (uv[:, 1] < ymax) & (uv[:, 1] >= ymin)


def _local(pc_cam, obj):
    r = sx.box_record(obj)
    d = pc_cam[:, :3].astype(np.float64) - r["center"]
    return r, (r["cs"] * d[:, 0] - r["sn"] * d[:, 2]), d[:, 1], (r["sn"] * d[:, 0] + r["cs"] * d[:, 2])


def in_box(pc_cam, obj):
    """box3d_contains of csrc/box_contains.cuh on box_record(obj), elementwise in float64."""
    r, lx, ly, lz = _local(pc_cam, obj)
    return (np.abs(lx) <= r["half"][0]) & (np.abs(ly) <= r["half"][1]) & (np.abs(lz) <= r["half"][2])


def box_margin(pc_cam, obj):
    """Signed distance of each point to the faces of obj's box: > 0 inside."""
    r, lx, ly, lz = _local(pc_cam, obj)
    return np.minimum(np.minimum(r["half"][0] - np.abs(lx), r["half"][1] - np.abs(ly)), r["half"][2] - np.abs(lz))


class _Frames:
    def __init__(self, points, calibs):
        self.points, self.calibs, self.cache = points, calibs, {}

    def __getitem__(self, idx):
        if idx not in self.cache:
            pc = np.asarray(self.points[idx], dtype=np.float32)
            self.cache[idx] = (camera_points(pc), image_coords(pc, self.calibs[idx]))
        return self.cache[idx]


def _job(L, trace, frames, idx, box, typ, rng, calib, obj=None, prob=None):
    pc_cam, uv = frames[idx]
    inds = cut(uv, box)
    pts = pc_cam[inds]
    Rtilt, K = sx.calib_mats(calib)
    angle = sx.frustum_angle(box, Rtilt, K)
    t = dict(frame=idx, n=len(pts), skipped=False, choice=False, kept=False, in_box=None, chosen=None)
    trace.append(t)
    if obj is not None:
        if sx.zero_extent(obj):
            t["skipped"] = True
            return
        label = in_box(pts, obj)
        t["in_box"] = int(label.sum())
    if len(pts) > sx.CAP:
        choice = rng.choice(len(pts), sx.CAP, replace=False)
        t["choice"] = True
        pts = pts[choice]
        if obj is not None:
            label = label[choice]
    if obj is not None:
        t["chosen"] = int(label.sum())
        if np.sum(label) < sx.MIN_POINTS:
            return
    elif len(pts) < sx.MIN_POINTS:
        return
    t["kept"] = True
    L["id"].append(idx)
    L["type"].append(typ)
    L["input"].append(pts.astype(np.float32))
    L["frustum_angle"].append(angle)
    L["calib_K"].append(K)
    L["calib_R"].append(Rtilt)
    if obj is not None:
        L["box2d"].append(np.array([box[0], box[1], box[2], box[3]], dtype=np.float32))
        L["box3d"].append(sx.box3d_corners(obj))
        L["label"].append(label.astype(bool))
        L["box3d_heading"].append(obj.heading_angle)
        L["box3d_size"].append(np.array([2 * obj.l, 2 * obj.w, 2 * obj.h]))
    else:
        L["box2d"].append(box)
        L["box2d_prob"].append(prob)


def from_ground_truth(points, calibs, image_ids, gt, type_whitelist=sx.TYPE_WHITELIST, perturb=False, augment=1,
                      rng=np.random):
    """-> (the reference's dict, the per-job trace)."""
    L = {k: [] for k, _ in sx.GT_KEYS}
    trace, frames = [], _Frames(points, calibs)
    for idx in image_ids:
        for obj in gt[idx]:
            if obj.classname not in type_whitelist:
                continue
            for _ in range(augment):
                box = sx.random_shift_box2d(obj.box2d, rng) if perturb else obj.box2d
                _job(L, trace, frames, idx, box, obj.classname, rng, calibs[idx], obj=obj)
    return L, trace


def from_rgb_detections(points, calibs, id_list, type_list, box2d_list, prob_list, type_whitelist=sx.TYPE_WHITELIST,
                        valid_ids=None, rng=np.random):
    L = {k: [] for k, _ in sx.DET_KEYS}
    trace, frames = [], _Frames(points, calibs)
    for i in range(len(id_list)):
        idx = id_list[i]
        if valid_ids is not None and idx not in valid_ids:
            continue
        if type_list[i] not in type_whitelist:
            continue
        _job(L, trace, frames, idx, box2d_list[i], type_list[i], rng, calibs[idx], prob=prob_list[i])
    return L, trace


def counter(points, calibs, slots):
    """A count callable for sunrgbd_extract.replay computed here: the in-box counts of the live slots' jobs."""
    frames = _Frames(points, calibs)
    live = [s for s in slots if not s["skip"]]

    def count(begin, end, cuts):
        return np.array([int(cut(frames[live[j]["frame"]][1], c).sum()) for j, c in zip(range(begin, end), cuts)],
                        np.int64)
    return count
