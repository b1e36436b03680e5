"""KITTI first-stage training frustums on the device: extract_frustum_data and extract_frustum_det_data of the
reference's kitti/prepare_data.py (--gen_train, --gen_val and the _det extension of provider_sample.py:110-125)
without their pickles, for a whole set of frames in one call.

    gx = GtFrustumExtractor(type_whitelist=("Car",))
    train = gx.from_ground_truth(scans, calibs, image_hw, train_ids, "label_2", perturb=True, augment=5, rng=np.random)
    val   = gx.from_ground_truth(scans, calibs, image_hw, val_ids, "label_2")
    ext   = gx.from_matched_detections(scans, calibs, image_hw, train_ids, ids, types, probs, boxes, "label_2",
                                       perturb=True, augment=5, rng=np.random)   # read_rgb_detections' four lists
    tb = TrainBatchBuilder.from_frustums(train, "det", strides=cfg.DATA.STRIDE, npoints=cfg.DATA.NUM_SAMPLES)

  from_ground_truth        extract_frustum_data (:260-391): every label line of a whitelisted type (exact match), in
                           line order, `augment` times; with perturb, each time its 2-D box shifted and scaled by
                           random_shift_box2d(., H, W, 0.1) (four rng.random() draws an attempt: cx, cy, h, w; the box
                           clipped to the image, drawn again while degenerate).  Labels: the points in its 3-D box.
  from_matched_detections  extract_frustum_det_data (:102-257): in the frames with whitelisted ground truth, every
                           whitelisted detection in line order gets the ground truth of the first maximum of
                           bbox_overlaps_2d (numpy, on the host: a NaN is the maximum) when that maximum is >= 0.5
                           (Car in the whitelist) or 0.25; it cuts with its own unclipped (or perturbed) box, `augment`
                           times, and is labelled with that ground truth's 3-D box.
A job whose label ground truth's 2-D box is under 25 px tall is dropped here on the host, after its perturbation draws
(the reference draws before it tests, :320 before :354).  A job without a labelled point is dropped on the device.
A whitelisted box with xmin >= xmax or ymin >= ymax raises ValueError naming its line when perturbed (where the
reference asserts); a non-finite 2-D box, or a label 3-D box that is not finite or has a non-positive extent (the
reference's Qhull would raise), always raises.

The points are the in-image points of section (15) (FrustumExtractor's projection), float32 rect x, y, z and intensity
in scan order, cut with xmin <= u < xmax and ymin <= v < ymax for the box as given (not clipped); "in the 3-D box" is
refine_extract's float64 half-space test (csrc/box_contains.cuh) where the reference triangulates the corners of
kitti_util.compute_box_3d with scipy's Delaunay: the two agree except for points within rounding (~1e-9 m) of a face.
Every per-box constant (perturbation, frustum_angle, corners, heading, size) is computed here on the host with the
reference's own numpy expressions; nothing random runs on the device.  One host sync per call, to learn the kept
frustums and their points.  No CPU fallback: CPU tensors and devices raise."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._host import cuda_device, upload
from .frustum_extract import LabelledFrustums, empty_outputs, frame_order, run_extract, scan_table
from .refine_extract import _check_box, box_record, iou_thresh, obj_array, objects_of

SHIFT_RATIO = 0.1          # random_shift_box2d(box2d, H, W, 0.1) of the training sets (prepare_data.py:187, :321)
MIN_HEIGHT = 25            # a ground truth whose 2-D box is shorter is rejected (:220, :354)
NAMES = ("id_list", "box2d_list", "box3d_list", "input_list", "label_list", "type_list", "heading_list", "size_list",
         "frustum_angle_list", "gt_box2d_list", "calib_list")          # the pickle's order (:244-255, :378-389)


# ------------------------------------------------------------------------------ per-box constants (host, float64)
def random_shift_box2d(box2d, img_height, img_width, shift_ratio=SHIFT_RATIO, rng=np.random):
    """prepare_data.py:55-77 with the generator as an argument; the reference's assert is the caller's check."""
    r = shift_ratio
    xmin, ymin, xmax, ymax = box2d
    h = ymax - ymin
    w = xmax - xmin
    cx = (xmin + xmax) / 2.0
    cy = (ymin + ymax) / 2.0
    while True:
        cx2 = cx + w * r * (rng.random() * 2 - 1)
        cy2 = cy + h * r * (rng.random() * 2 - 1)
        h2 = h * (1 + rng.random() * 2 * r - r)
        w2 = w * (1 + rng.random() * 2 * r - r)
        new_box2d = np.array([cx2 - w2 / 2.0, cy2 - h2 / 2.0, cx2 + w2 / 2.0, cy2 + h2 / 2.0])
        new_box2d[[0, 2]] = np.clip(new_box2d[[0, 2]], 0, img_width - 1)
        new_box2d[[1, 3]] = np.clip(new_box2d[[1, 3]], 0, img_height - 1)
        if new_box2d[0] < new_box2d[2] and new_box2d[1] < new_box2d[3]:
            return new_box2d


def bbox_overlaps_2d(anchors, gt_boxes):
    """ops/pybind11/rbbox_iou.py:34-59, the same numpy expression: (N, 4) x (K, 4) -> (N, K)."""
    N = anchors.shape[0]
    K = gt_boxes.shape[0]
    gt_boxes_area = ((gt_boxes[:, 2] - gt_boxes[:, 0]) * (gt_boxes[:, 3] - gt_boxes[:, 1])).reshape(1, K)
    anchors_area = ((anchors[:, 2] - anchors[:, 0]) * (anchors[:, 3] - anchors[:, 1])).reshape(N, 1)
    boxes = np.broadcast_to(anchors.reshape(N, 1, 4), (N, K, 4))
    query_boxes = np.broadcast_to(gt_boxes.reshape(1, K, 4), (N, K, 4))
    iw = (np.minimum(boxes[:, :, 2], query_boxes[:, :, 2]) - np.maximum(boxes[:, :, 0], query_boxes[:, :, 0]))
    iw[iw < 0] = 0
    ih = (np.minimum(boxes[:, :, 3], query_boxes[:, :, 3]) - np.maximum(boxes[:, :, 1], query_boxes[:, :, 1]))
    ih[ih < 0] = 0
    ua = anchors_area + gt_boxes_area - (iw * ih)
    return iw * ih / ua


def frustum_angle(box, calib):
    """-arctan2 of calib.project_image_to_rect of the box centre at depth 20 (prepare_data.py:334-340,
    kitti_util.py:222-234)."""
    P = np.reshape(calib["P2"], [3, 4])
    c_u, c_v, f_u, f_v = P[0, 2], P[1, 2], P[0, 0], P[1, 1]
    b_x, b_y = P[0, 3] / (-f_u), P[1, 3] / (-f_v)
    xmin, ymin, xmax, ymax = box
    uvdepth = np.zeros((1, 3))
    uvdepth[0, 0:2] = np.array([(xmin + xmax) / 2.0, (ymin + ymax) / 2.0])
    uvdepth[0, 2] = 20
    rect = np.zeros((1, 3))
    rect[:, 0] = ((uvdepth[:, 0] - c_u) * uvdepth[:, 2]) / f_u + b_x
    rect[:, 1] = ((uvdepth[:, 1] - c_v) * uvdepth[:, 2]) / f_v + b_y
    rect[:, 2] = uvdepth[:, 2]
    return -1 * np.arctan2(rect[0, 2], rect[0, 0])


def compute_box_3d(obj):
    """The corners (8, 3) of kitti_util.compute_box_3d (:324-354): bottom centre t, y from 0 to -h."""
    c, s = np.cos(obj.ry), np.sin(obj.ry)
    R = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    l, w, h = obj.l, obj.w, obj.h
    x_corners = [l / 2, l / 2, -l / 2, -l / 2, l / 2, l / 2, -l / 2, -l / 2]
    y_corners = [0, 0, 0, 0, -h, -h, -h, -h]
    z_corners = [w / 2, -w / 2, -w / 2, w / 2, w / 2, -w / 2, -w / 2, w / 2]
    corners_3d = np.dot(R, np.vstack([x_corners, y_corners, z_corners]))
    corners_3d[0, :] = corners_3d[0, :] + obj.t[0]
    corners_3d[1, :] = corners_3d[1, :] + obj.t[1]
    corners_3d[2, :] = corners_3d[2, :] + obj.t[2]
    return np.transpose(corners_3d)


def _check_box2d(box, where, perturb):
    if not np.isfinite(box).all():
        raise ValueError("%s: the 2-D box must be finite, got %s" % (where, box.tolist()))
    if perturb and not (box[0] < box[2] and box[1] < box[3]):
        raise ValueError("%s: a perturbed 2-D box needs xmin < xmax and ymin < ymax, got %s" % (where, box.tolist()))


def _cuts(box, hw, perturb, augment, rng):
    """The `augment` cutting boxes of one box, drawn in the reference's order."""
    return [random_shift_box2d(box, hw[0], hw[1], SHIFT_RATIO, rng) if perturb else box for _ in range(augment)]


def _frame_hw(image_hw, idx):
    return tuple(int(x) for x in image_hw[idx])


def job_table(image_ids, gt_objects, type_whitelist, image_hw, perturb=False, augment=1, rng=np.random, dets=None,
              thresh=None):
    """The jobs of one extraction in the reference's order -> a list of dicts (frame id, `cut` the (4,) float64
    cutting box, `obj` the label ground truth's KittiObject, `det` the detection line in matched mode).  dets: None
    (ground-truth mode) or {frame id: [(line, type, (4,) float64 box)]} in line order (matched mode)."""
    jobs = []
    for idx in image_ids:
        idx = int(idx)
        gts = [o for o in gt_objects[idx] if o.type in type_whitelist]
        if dets is None:
            for obj in gts:
                _check_box2d(obj.box2d, obj.line, perturb)
                _check_box(obj_array(obj), obj)
                for cut in _cuts(obj.box2d, _frame_hw(image_hw, idx), perturb, augment, rng):
                    if obj.box2d[3] - obj.box2d[1] >= MIN_HEIGHT:
                        jobs.append(dict(frame=idx, cut=cut, obj=obj))
            continue
        if not gts or idx not in dets:                                     # :149-150, :161-163
            continue
        for o in gts:
            _check_box2d(o.box2d, o.line, False)
        gt_boxes_2d = np.stack([o.box2d for o in gts], 0)
        for line, typ, box in dets[idx]:
            if typ not in type_whitelist:
                continue
            where = "detection line %d" % line
            _check_box2d(box, where, False)
            with np.errstate(all="ignore"):
                overlap = bbox_overlaps_2d(box.reshape(-1, 4), gt_boxes_2d)[0]
            if overlap.max(0) < thresh:
                continue
            obj = gts[overlap.argmax(0)]
            _check_box2d(box, where, perturb)
            _check_box(obj_array(obj), obj)
            for cut in _cuts(box, _frame_hw(image_hw, idx), perturb, augment, rng):
                if obj.box2d[3] - obj.box2d[1] >= MIN_HEIGHT:
                    jobs.append(dict(frame=idx, cut=cut, obj=obj, det=line))
    return jobs


def detection_table(id_list, type_list, prob_list, box2d_list):
    """read_rgb_detections' four lists -> {frame id: [(line, type, (4,) float64 box)]} in line order (all_boxes_2d,
    prepare_data.py:110-122)."""
    n = len(id_list)
    if len(type_list) != n or len(prob_list) != n or len(box2d_list) != n:
        raise ValueError("id_list, type_list, prob_list and box2d_list must have the same length")
    out = {}
    for i in range(n):
        out.setdefault(int(id_list[i]), []).append(
            (i, type_list[i], np.asarray(box2d_list[i], dtype=np.float64).reshape(4)))
    return out


def job_lists(jobs, calibs):
    """The provider's lists (all but input_list and label_list) of the jobs `jobs`, in order."""
    L = {n: [] for n in NAMES if n not in ("input_list", "label_list")}
    for jb in jobs:
        obj, cut = jb["obj"], jb["cut"]
        calib = calibs[jb["frame"]]
        L["id_list"].append(jb["frame"])
        L["box2d_list"].append(np.array([cut[0], cut[1], cut[2], cut[3]]))
        L["box3d_list"].append(compute_box_3d(obj))
        L["type_list"].append(obj.type)
        L["heading_list"].append(obj.ry)
        L["size_list"].append(np.array([obj.l, obj.w, obj.h]))
        L["frustum_angle_list"].append(frustum_angle(cut, calib))
        L["gt_box2d_list"].append(obj.box2d)
        L["calib_list"].append(calib)
    return L


# ------------------------------------------------------------------------------ result
class GtFrustums(LabelledFrustums):
    """One extraction (LabelledFrustums), always labelled; the lists are the provider's
    (datasets/provider_sample.py:97-108)."""

    pickle_names = NAMES

    def __init__(self, points, offsets, label, counts, job_index, lists, stream=None):
        super().__init__(points, offsets, label, counts, job_index, stream)
        for n in NAMES:
            if n not in ("input_list", "label_list"):
                setattr(self, n, lists[n])


class GtFrustumExtractor:
    def __init__(self, type_whitelist=("Car",), device=None):
        self.type_whitelist = tuple(type_whitelist)
        self.device = cuda_device(device, "GtFrustumExtractor")

    @property
    def iou_thresh(self):
        return iou_thresh(self.type_whitelist)

    def from_ground_truth(self, scans, calibs, image_hw, image_ids, gt, perturb=False, augment=1, rng=np.random,
                          stream=None, timer=None):
        """gt: a label_2 directory or {idx: [KittiObject]}.  rng: the np.random module or a RandomState."""
        gt = objects_of(gt, image_ids)
        jobs = job_table(image_ids, gt, self.type_whitelist, image_hw, perturb, int(augment), rng)
        return self._run(scans, calibs, image_hw, jobs, stream, timer)

    def from_matched_detections(self, scans, calibs, image_hw, image_ids, id_list, type_list, prob_list, box2d_list,
                                gt, perturb=False, augment=1, rng=np.random, stream=None, timer=None):
        """id_list ... box2d_list: read_rgb_detections' four lists; gt as for from_ground_truth."""
        dets = detection_table(id_list, type_list, prob_list, box2d_list)
        gt = objects_of(gt, image_ids)
        jobs = job_table(image_ids, gt, self.type_whitelist, image_hw, perturb, int(augment), rng, dets,
                         self.iou_thresh)
        return self._run(scans, calibs, image_hw, jobs, stream, timer)

    # ------------------------------------------------------------------ device call
    def _run(self, scans, calibs, image_hw, jobs, stream, timer):
        dev = self.device
        frame_ids, fpos = frame_order(jb["frame"] for jb in jobs)
        labels, label_of = [], {}
        for jb in jobs:
            if id(jb["obj"]) not in label_of:
                label_of[id(jb["obj"])] = len(labels)
                labels.append(jb["obj"])
        J, F = len(jobs), len(frame_ids)
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            if F == 0 or J == 0:
                return GtFrustums(*empty_outputs(dev, 4, True), np.zeros(0, np.int64), np.zeros(0, np.int64),
                                  job_lists([], calibs), stream)
            sc, frames, so = scan_table(scans, calibs, image_hw, frame_ids, dev, "GtFrustumExtractor")
            job_rec = np.zeros(J, dtype=np.dtype(_lib.GtJob))
            job_rec["box"] = np.stack([jb["cut"] for jb in jobs])
            job_rec["frame"] = [fpos[jb["frame"]] for jb in jobs]
            job_rec["label"] = [label_of[id(jb["obj"])] for jb in jobs]
            label_box = np.array([box_record(obj_array(o)) for o in labels], dtype=np.dtype(_lib.RefineBox))
            inp, ptrs = upload([bytes(frames), job_rec, label_box, so], dev)
            a = _lib.GtExtractArgs()
            a.num_frames, a.num_points, a.num_jobs, a.num_labels = F, int(so[-1]), J, len(labels)
            a.frames, a.jobs, a.label_boxes, a.scan_offsets = ptrs
            job_points, kept, out = run_extract(
                "gt_extract", a, sc, so, J, ("job_points",),
                lambda K, M, words: {"labels": torch.empty(M, dtype=torch.uint8, device=dev)},
                dev, stream, timer, "jobs reference no frame or label box")
        return GtFrustums(out["points"], out["offsets"], out["labels"], job_points[kept].astype(np.int64),
                          kept.astype(np.int64), job_lists([jobs[j] for j in kept.tolist()], calibs), stream)
