"""ORACLE: extract_frustum_data_rgb_detection (kitti/prepare_data.py:462-568, kitti_util.py:172-210, draw_util.py:12-23)
restated in numpy with the projection evaluated elementwise in float64, in exactly the order of
csrc/frustum_extract.cu (fx_project): every product and sum rounded separately, each matrix row summed left to right
from column 0, the homogeneous 1 entering as the last column's value.  The reference's np.dot may round the float64
rect and image coordinates differently; the float32 points and every edge decision agree wherever no coordinate lies
within rounding of an edge, which the fixtures assert (oracle/make_golden_frustum_extract.py).

Returns the pickle's seven lists: id_list, box2d_list, input_list, type_list, frustum_angle_list, prob_list,
calib_list."""
from __future__ import annotations

import numpy as np


def _rows(M, cols, extra=None):
    """M (3, k) float64 times the column vectors `cols` (k arrays), each row ((m0 c0 + m1 c1) + m2 c2) (+ extra)."""
    out = []
    for i in range(3):
        acc = M[i, 0] * cols[0]
        for j in range(1, len(cols)):
            acc = acc + M[i, j] * cols[j]
        if extra is not None:
            acc = acc + M[i, extra]
        out.append(acc)
    return out


def project(scan, calib):
    """(n, 4) float32 scan -> (rect float32 (n, 3), u, v float64 (n,))."""
    P = np.asarray(calib["P2"], dtype=np.float64).reshape(3, 4)
    V = np.asarray(calib["Tr_velo_to_cam"], dtype=np.float64).reshape(3, 4)
    R = np.asarray(calib["R0_rect"], dtype=np.float64).reshape(3, 3)
    xyz = [scan[:, k].astype(np.float64) for k in range(3)]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        ref = _rows(V, xyz, extra=3)
        rect = _rows(R, ref)
        img = _rows(P, rect, extra=3)
        u, v = img[0] / img[2], img[1] / img[2]
    return np.stack(rect, axis=1).astype(np.float32), u, v


def in_image(scan, u, v, height, width, clip_distance=2.0):
    with np.errstate(invalid="ignore"):
        return (u < width) & (u >= 0) & (v < height) & (v >= 0) & (scan[:, 0] > clip_distance)


def extract(scans, calibs, image_hw, id_list, type_list, prob_list, box2d_list, type_whitelist=("Car",),
            img_height_threshold=5, lidar_point_threshold=1):
    out = {k: [] for k in ("id", "box2d", "input", "type", "angle", "prob", "calib")}
    cache_id, cache = None, None
    for det_idx in range(len(id_list)):
        data_idx = id_list[det_idx]
        if cache_id != data_idx:
            scan = np.asarray(scans[data_idx], dtype=np.float32)
            calib = calibs[data_idx]
            rect, u, v = project(scan, calib)
            pc_rect = np.concatenate([rect, scan[:, 3:4]], axis=1)
            h, w = image_hw[data_idx]
            fov = in_image(scan, u, v, h, w)
            cache, cache_id = (calib, pc_rect, u, v, fov, h, w), data_idx
        calib, pc_rect, u, v, fov, h, w = cache
        if type_list[det_idx] not in type_whitelist:
            continue
        box = np.asarray(box2d_list[det_idx], dtype=np.float64).copy()
        box[[0, 2]] = np.clip(box[[0, 2]], 0, w - 1)
        box[[1, 3]] = np.clip(box[[1, 3]], 0, h - 1)
        xmin, ymin, xmax, ymax = box
        with np.errstate(invalid="ignore"):
            inds = (u < xmax) & (u >= xmin) & (v < ymax) & (v >= ymin) & fov
        pts = pc_rect[inds, :]
        P = np.asarray(calib["P2"], dtype=np.float64).reshape(3, 4)
        c_u, c_v, f_u, f_v = P[0, 2], P[1, 2], P[0, 0], P[1, 1]
        b_x = P[0, 3] / (-f_u)
        cx = (xmin + xmax) / 2.0
        x = ((cx - c_u) * 20.0) / f_u + b_x
        angle = -1 * np.arctan2(20.0, x)
        if ymax - ymin < img_height_threshold or xmax - xmin < 1 or len(pts) < lidar_point_threshold:
            continue
        out["id"].append(data_idx)
        out["type"].append(type_list[det_idx])
        out["box2d"].append(np.array([xmin, ymin, xmax, ymax]))
        out["prob"].append(prob_list[det_idx])
        out["input"].append(pts.astype(np.float32, copy=False))
        out["angle"].append(angle)
        out["calib"].append(calib)
    return out["id"], out["box2d"], out["input"], out["type"], out["angle"], out["prob"], out["calib"]
