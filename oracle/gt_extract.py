"""ORACLE: extract_frustum_data (kitti/prepare_data.py:260-391) and extract_frustum_det_data (:102-257) restated in
numpy, frame by frame.

The job order, the perturbation replay, the 2-D matching and every per-box constant come from the host code the device
path uses (frustum_convnet_b200.gt_extract.job_table / job_lists: the reference's own numpy expressions).  The point
work is restated here:
  projection  oracle/frustum_extract.project and in_image: float64 velo -> rect -> image in the kernel's elementwise
              order, the in-image test of get_lidar_in_image_fov;
  2-D cut     u < xmax, u >= xmin, v < ymax, v >= ymin with the cutting box as given (:324-328);
  labels      oracle/refine_extract.in_box, the float64 half-space test, on the label box [tx, ty - h/2, tz, l, w, h,
              ry], instead of scipy's Delaunay over kitti_util.compute_box_3d's corners; the two agree except for
              points within rounding of a face (the fixture's scenes keep every point more than BAND from every face).
Returns the pickled lists of the reference's functions, in their order (gt_extract.NAMES)."""
from __future__ import annotations

import numpy as np

from frustum_convnet_b200 import gt_extract as gx
from frustum_convnet_b200 import refine_extract as rx
from oracle import frustum_extract as ofx
from oracle import refine_extract as orx


def fov_points(scan, calib, hw):
    """The in-image points of a frame: (float32 rect x, y, z and intensity (n, 4), float64 u (n,), v (n,))."""
    scan = np.asarray(scan, dtype=np.float32)
    rect, u, v = ofx.project(scan, calib)
    keep = ofx.in_image(scan, u, v, hw[0], hw[1])
    return np.concatenate([rect, scan[:, 3:4]], axis=1)[keep], u[keep], v[keep]


def cut(u, v, box):
    xmin, ymin, xmax, ymax = box
    return (u < xmax) & (u >= xmin) & (v < ymax) & (v >= ymin)


def jobs_of(mode, image_ids, gt_objects, type_whitelist, image_hw, perturb=False, augment=1, rng=np.random,
            dets=None):
    """mode 'gt' or 'matched' (dets: read_rgb_detections' four lists) -> gt_extract.job_table's jobs."""
    if mode == "gt":
        return gx.job_table(image_ids, gt_objects, type_whitelist, image_hw, perturb, augment, rng)
    thresh = 0.5 if "Car" in type_whitelist else 0.25
    return gx.job_table(image_ids, gt_objects, type_whitelist, image_hw, perturb, augment, rng,
                        gx.detection_table(*dets), thresh)


def extract(mode, scans, calibs, image_hw, image_ids, gt_objects, type_whitelist=("Car",), perturb=False, augment=1,
            rng=np.random, dets=None):
    """-> {list name: list} (the pickled lists, gt_extract.NAMES in order)."""
    jobs = jobs_of(mode, image_ids, gt_objects, type_whitelist, image_hw, perturb, augment, rng, dets)
    kept, inputs, labels, cache = [], [], [], {}
    for jb in jobs:
        idx = jb["frame"]
        if idx not in cache:
            cache[idx] = fov_points(scans[idx], calibs[idx], image_hw[idx])
        pc, u, v = cache[idx]
        pts = pc[cut(u, v, jb["cut"])]
        label = np.zeros(pts.shape[0])
        label[orx.in_box(pts, rx.obj_array(jb["obj"]))] = 1
        if np.sum(label) == 0:
            continue
        kept.append(jb)
        inputs.append(pts.astype(np.float32, copy=False))
        labels.append(label)
    L = gx.job_lists(kept, calibs)
    L["input_list"], L["label_list"] = inputs, labels
    return {n: L[n] for n in gx.NAMES}
