"""ORACLE: the three extraction functions of kitti/prepare_data_refine.py (extract_frustum_data :239-403,
extract_frustum_det_data :406-592, extract_frustum_data_rgb_detection :649-773) restated in numpy, frame by frame.

The per-box constants and the job order come from the host code the device path uses
(frustum_convnet_b200.refine_extract.job_table: the reference's own numpy expressions, and the rng replay of
random_shift_rotate_box3d).  Two substitutions, shared with csrc/refine_extract.cu:
  in_box     "inside the box" is a float64 half-space test in the box's frame (every product and sum rounded
             separately, in the kernel's order) instead of scipy's Delaunay(corners).find_simplex >= 0; the two agree
             except for points within rounding of a face (box_margin gives the distance; the fixture's scenes keep
             every point more than BAND from every face of every box they test);
  match_iou  rbbox_iou_3d as its standup pre-filter (bbox_overlaps_3d, in the reference's order) and then
             oracle/box_iou.rbbox_iou_3d_pair's float64 clip instead of Boost.Geometry.
Returns the pickled lists of the reference's function, in its order (see LIST_NAMES)."""
from __future__ import annotations

import numpy as np

from frustum_convnet_b200 import _lib
from frustum_convnet_b200 import refine_extract as rx
from oracle import box_iou as obi
from oracle import frustum_extract as ofx

BAND = 1e-9
LIST_NAMES = {"gt": rx._GT_NAMES, "matched": rx._GT_NAMES, "det": rx._DET_NAMES}
MODES = {"gt": _lib.REFINE_GT, "matched": _lib.REFINE_MATCHED, "det": _lib.REFINE_DET}


def _local(pc, a):
    c, s = np.cos(a[6]), np.sin(a[6])
    d = pc[:, :3].astype(np.float64) - a[:3]
    return c * d[:, 0] - s * d[:, 2], d[:, 1], s * d[:, 0] + c * d[:, 2]


def in_box(pc, a):
    """Box array a = [cx, cy, cz, l, w, h, ry]: |R^T (p - c)| <= (l, h, w) / 2 per axis."""
    lx, ly, lz = _local(pc, a)
    return (np.abs(lx) <= a[3] / 2) & (np.abs(ly) <= a[5] / 2) & (np.abs(lz) <= a[4] / 2)


def box_margin(pc, a):
    """Signed distance of each point to the faces of box a: > 0 inside."""
    lx, ly, lz = _local(pc, a)
    return np.minimum(np.minimum(a[3] / 2 - np.abs(lx), a[5] / 2 - np.abs(ly)), a[4] / 2 - np.abs(lz))


def standup_iou(c, q):
    """bbox_overlaps_3d (ops/pybind11/rbbox_iou.py:62-96) of the standup boxes of corners c (8, 3) and q (8, 3)."""
    a = np.concatenate([c.min(0), c.max(0)])[[0, 2, 3, 5, 1, 4]]
    g = np.concatenate([q.min(0), q.max(0)])[[0, 2, 3, 5, 1, 4]]
    va = (a[2] - a[0]) * (a[3] - a[1]) * (a[5] - a[4])
    vg = (g[2] - g[0]) * (g[3] - g[1]) * (g[5] - g[4])
    ext = [max(min(a[2], g[2]) - max(a[0], g[0]), 0.0), max(min(a[3], g[3]) - max(a[1], g[1]), 0.0),
           max(min(a[5], g[5]) - max(a[4], g[4]), 0.0)]
    inter = ext[0] * ext[1] * ext[2]
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.float64(inter) / ((va + vg) - inter)


def match_iou(det_box, gt_boxes):
    """rbbox_iou_3d(det_box.reshape(-1, 7), gt_boxes)[0]: (G,) float64."""
    dc = rx.iou_corners(det_box)[0]
    gc = rx.iou_corners(np.stack(gt_boxes))
    out = np.zeros(len(gt_boxes))
    for g in range(len(gt_boxes)):
        if not standup_iou(dc, gc[g]) <= 0.0:
            out[g] = obi.rbbox_iou_3d_pair(dc[None], gc[g][None])[0, 1]
    return out


def fov_points(scan, calib, hw):
    """pc_rect[img_fov_inds] of the reference: float32 rect x, y, z and intensity of the in-image points."""
    scan = np.asarray(scan, dtype=np.float32)
    rect, u, v = ofx.project(scan, calib)
    keep = ofx.in_image(scan, u, v, hw[0], hw[1])
    return np.concatenate([rect, scan[:, 3:4]], axis=1)[keep]


def extract(mode, scans, calibs, image_hw, image_ids, objects=None, gt_objects=None, type_whitelist=("Car",),
            remove_diff=False, perturb=False, augment=1, rng=np.random):
    """mode 'gt', 'matched' or 'det' -> {list name: list} (the pickled lists, LIST_NAMES[mode] in order)."""
    m = MODES[mode]
    jobs, gts = rx.job_table(m, image_ids, objects, gt_objects, type_whitelist, remove_diff, perturb, augment, rng)
    thresh = 0.5 if "Car" in type_whitelist else 0.25
    L = {n: [] for n in LIST_NAMES[mode]}
    cache = {}
    for jb in jobs:
        idx = jb["frame"]
        if idx not in cache:
            cache[idx] = fov_points(scans[idx], calibs[idx], image_hw[idx])
        pc = cache[idx]
        cut = jb["cut"]
        pts = pc[in_box(pc, cut)]
        gt = None
        if mode == "gt":
            gt = gts[idx][jb["gt"]]
        elif mode == "matched":
            ov = match_iou(jb["box"], [rx.obj_array(o) for o in gts[idx]])
            if ov.max(0) < thresh:
                continue
            gt = gts[idx][int(ov.argmax(0))]
        if gt is not None:
            label = np.zeros(pts.shape[0])
            label[in_box(pts, rx.obj_array(gt))] = 1
            if np.sum(label) == 0:
                continue
        elif len(pts) < 1:
            continue
        obj = jb["obj"]
        L["id_list"].append(idx)
        L["input_list"].append(pts.astype(np.float32, copy=False))
        L["type_list"].append(obj.type)
        L["frustum_angle_list"].append(rx.frustum_angle(cut))
        L["calib_list"].append(calibs[idx])
        L["pred_box3d_list"].append(rx.compute_box_3d_obj_array(cut))
        L["pred_box3d_size_list"].append(cut[3:6])
        L["pred_box3d_angle_list"].append(cut[-1])
        if gt is None:
            L["box2d_list"].append(obj.box2d)
            L["prob_list"].append(obj.score)
        else:
            L["label_list"].append(label)
            L["box3d_list"].append(rx.compute_box_3d_obj_array(rx.obj_array(gt)))
            L["heading_list"].append(gt.ry)
            L["size_list"].append(np.array([gt.l, gt.w, gt.h]))
            L["box2d_list"].append(gt.box2d)
    return L
