"""KITTI refinement frustums on the device: the three extraction functions of the reference's
kitti/prepare_data_refine.py without their pickles, for a whole set of frames in one call.

    rx = RefineFrustumExtractor(type_whitelist=("Car",))
    train = rx.from_ground_truth(scans, calibs, image_hw, train_ids, gt_dir, perturb=True, augment=5, rng=np.random)
    val   = rx.from_ground_truth(scans, calibs, image_hw, val_ids, gt_dir, remove_diff=True)
    vdet  = rx.from_matched_detections(scans, calibs, image_hw, val_ids, col.finalize(), gt_dir, remove_diff=True)
    test  = rx.from_detections(scans, calibs, image_hw, val_ids, col.finalize())    # or read_result_dir(...)
    tb = TrainBatchBuilder.from_frustums(test, "refine", strides=cfg.DATA.STRIDE, npoints=cfg.DATA.NUM_SAMPLES,
                                         labels=False)

  from_ground_truth        extract_frustum_data (:239-403): every ground-truth box of a whitelisted type (after the
                           remove_diff rule: occlusion > 2, truncation > 0.5 or a 2-D height < 25 drop it), enlarged
                           x1.2 and, with perturb, perturbed `augment` times in a chain (random_shift_rotate_box3d(.,
                           0.05), seven rng.random() draws an attempt); labels: the points in the ground-truth box.
  from_matched_detections  extract_frustum_det_data (:406-592): every whitelisted detection of a frame with ground
                           truth, enlarged x1.2; its ground truth is the first maximum of the 3-D IoU (rbbox_iou_3d,
                           float64, on the device) if that maximum is >= 0.5 (Car in the whitelist) or 0.25.
  from_detections          extract_frustum_data_rgb_detection (:649-773): every whitelisted detection, enlarged x1.2,
                           dropped when ymax - ymin < 5, xmax - xmin < 1 (the 2-D box as read, not clipped) or it
                           has no point; no labels, prob_list holds the scores.
A ground-truth or matched frustum without a labelled point is dropped.  Types match exactly (Object3d.type in
type_whitelist).  Every per-box constant (the box array, enlargement, perturbation, corners, sizes, angles,
frustum_angle) is computed here on the host with the reference's own numpy expressions; nothing random runs on the
device.  The points are the in-image points of section (15) (FrustumExtractor's projection), float32 rect x, y, z
and intensity in scan order; "in a box" is a float64 half-space test in the box's frame (csrc/refine_extract.cu)
where the reference triangulates the 8 corners with scipy's Delaunay: the two agree except for points within
rounding (~1e-9 m) of a face.  A box with a non-positive extent raises ValueError naming its line where the
reference's Qhull would raise (in matched mode: a matched detection and its ground truth only).  The matching IoU
substitutes the reference's Boost polygon clip with box_iou.cuh's clip_quads_area<double>; agreement with Boost is
not pinned.

Detections are the collector's {idx: {class: (n, 12)}} taken as the values the reference reads back from the text
write_detection_results writes (kitti_eval.detection_records), lines in class then row order; or the result files
themselves (read_result_dir).  Ground truth is a label_2 directory (or a {idx: [KittiObject]} dict).  One host sync
per call, to learn the kept frustums and their points.  No CPU fallback: CPU tensors and devices raise.

from_collected / from_matched_collected take DetectionCollector.finalize_device()'s CollectedDetections instead of the
dict: the rows stay on the device (csrc/refine_jobs.cu).  The host plans the jobs from segment metadata alone, the
device reads each row back as its text, builds and checks its box and writes the job; after the count pass it writes
the kept frustums' lists and their TrainBatchBuilder records (CollectedRefineFrustums).  Same one host read."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from ._host import csr_offsets, cuda_device, upload
from .frustum_extract import LabelledFrustums, empty_outputs, frame_order, run_extract, scan_table
from .kitti_eval import detection_records
from .train_inputs import KITTI_CLASSES

RATIO = 1.2                # the enlargement of every box that cuts points (prepare_data_refine.py:319, :489, :724)
PERTURB_RATIO = 0.05       # random_shift_rotate_box3d(., 0.05) of the training set (:328-329)
REFINE_STRIDES = (0.1, 0.2, 0.4, 0.8)   # cfg.DATA.STRIDE of cfgs/refine_car.yaml: the strides of the records


class KittiObject:
    """One label or result line, parsed as kitti_util.Object3d parses it."""

    def __init__(self, type, truncation, occlusion, alpha, box2d, h, w, l, t, ry, score=1, line=""):
        self.type, self.truncation, self.occlusion, self.alpha = type, truncation, occlusion, alpha
        self.box2d = np.array([box2d[0], box2d[1], box2d[2], box2d[3]])
        self.xmin, self.ymin, self.xmax, self.ymax = (float(v) for v in box2d)
        self.h, self.w, self.l, self.t, self.ry, self.score = h, w, l, tuple(t), ry, score
        self.line = line                 # "<file>:<line number>" for error messages

    @classmethod
    def parse(cls, text, where=""):
        data = text.split(" ")
        data[1:] = [float(x) for x in data[1:]]
        return cls(data[0], data[1], int(data[2]), data[3], data[4:8], data[8], data[9], data[10],
                   (data[11], data[12], data[13]), data[14], data[15] if len(data) > 15 else 1, where)


def read_objects(path):
    """A label or result file -> [KittiObject] (utils.read_label); a missing file raises, an empty one is empty."""
    with open(path) as f:
        return [KittiObject.parse(line.rstrip(), "%s:%d" % (path, n + 1)) for n, line in enumerate(f)]


def read_label_dir(label_dir, image_ids):
    return {int(i): read_objects(os.path.join(label_dir, "%06d.txt" % int(i))) for i in image_ids}


def objects_of(gt, image_ids):
    """Ground truth as the extractors take it, a label_2 directory or {idx: [KittiObject]} -> {int idx: objects}."""
    if isinstance(gt, (str, os.PathLike)):
        return read_label_dir(gt, image_ids)
    return {int(k): v for k, v in gt.items()}


def iou_thresh(type_whitelist):
    """The matching threshold of matched detections (prepare_data.py:141, prepare_data_refine.py:447)."""
    return 0.5 if "Car" in type_whitelist else 0.25


def read_result_dir(result_dir, image_ids):
    """Result files '%06d.txt' of every image of image_ids -> {idx: [KittiObject]}."""
    return read_label_dir(result_dir, image_ids)


def objects_from_detections(dets):
    """The collector's {idx: {class: float32 (n, 12)}} -> {idx: [KittiObject]}: the values utils.read_label reads
    back from the lines write_detection_results writes, in its line order (classes in dict order, then rows)."""
    out = {}
    for idx, per_class in dets.items():
        objs = []
        for cls_type, rows in per_class.items():
            for n, r in enumerate(detection_records(rows, cls_type)):
                objs.append(KittiObject(cls_type, -1.0, -1, float(r[1]), [float(v) for v in r[2:6]], float(r[6]),
                                        float(r[7]), float(r[8]), [float(v) for v in r[9:12]], float(r[12]),
                                        float(r[13]), "detections[%d][%r] row %d" % (idx, cls_type, n)))
        out[int(idx)] = objs
    return out


# ------------------------------------------------------------------------------ per-box constants (host, float64)
def obj_array(obj):
    """[cx, cy - h / 2, cz, l, w, h, ry] (prepare_data_refine.py:310-315)."""
    cx, cy, cz = obj.t
    return np.array([cx, cy - obj.h / 2, cz, obj.l, obj.w, obj.h, obj.ry])


def compute_box_3d_obj_array(a):
    """prepare_data_refine.py:56-79: the 8 corners (8, 3) of [cx, cy, cz, l, w, h, ry]."""
    cx, cy, cz, l, w, h, angle = a
    c, s = np.cos(angle), np.sin(angle)
    R = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    x_corners = [l / 2, l / 2, -l / 2, -l / 2, l / 2, l / 2, -l / 2, -l / 2]
    y_corners = [h / 2, h / 2, h / 2, h / 2, -h / 2, -h / 2, -h / 2, -h / 2]
    z_corners = [w / 2, -w / 2, -w / 2, w / 2, w / 2, -w / 2, -w / 2, w / 2]
    corners_3d = np.dot(R, np.vstack([x_corners, y_corners, z_corners]))
    corners_3d[0, :] = corners_3d[0, :] + cx
    corners_3d[1, :] = corners_3d[1, :] + cy
    corners_3d[2, :] = corners_3d[2, :] + cz
    return np.transpose(corners_3d, (1, 0))


def random_shift_rotate_box3d(a, r=PERTURB_RATIO, rng=np.random):
    """prepare_data_refine.py:203-236 with the generator as an argument: seven rng.random() draws an attempt (l, h, w,
    cx, cy, cz, angle), again while an extent is <= 0, the angle wrapped to [-pi, pi)."""
    cx, cy, cz, l, w, h, angle = a
    angle = angle + np.pi
    if not (l > 0 and w > 0 and h > 0):
        raise ValueError("a perturbed box needs positive extents, got l, w, h = %r, %r, %r" % (l, w, h))
    while True:
        l1 = l + l * r * (rng.random() * 2 - 1)
        h1 = h + h * r * (rng.random() * 2 - 1)
        w1 = w + w * r * (rng.random() * 2 - 1)
        cx1 = cx + l * r * (rng.random() * 2 - 1)
        cy1 = cy + h * r * (rng.random() * 2 - 1)
        cz1 = cz + w * r * (rng.random() * 2 - 1)
        angle1 = angle + r * (rng.random() * 2 - 1) * np.pi
        angle1 = angle1 % (2 * np.pi)
        if l1 > 0 and h1 > 0 and w1 > 0:
            return np.array([cx1, cy1, cz1, l1, w1, h1, angle1 - np.pi])


def iou_corners(boxes):
    """ops/pybind11/rbbox_iou.py:121-148 (boxes3d2corners): (n, 7) -> (n, 8, 3), as rbbox_iou_3d computes them."""
    boxes = np.asarray(boxes, dtype=np.float64).reshape(-1, 7)
    N = boxes.shape[0]
    l, w, h, hd = boxes[:, 3], boxes[:, 4], boxes[:, 5], boxes[:, 6]
    x = np.stack([l / 2, l / 2, -l / 2, -l / 2, l / 2, l / 2, -l / 2, -l / 2], 1)
    y = np.stack([h / 2, h / 2, h / 2, h / 2, -h / 2, -h / 2, -h / 2, -h / 2], 1)
    z = np.stack([w / 2, -w / 2, -w / 2, w / 2, w / 2, -w / 2, -w / 2, w / 2], 1)
    corners = np.stack([x, y, z], 1)
    c, s = np.cos(hd), np.sin(hd)
    one, zero = np.ones(N), np.zeros(N)
    R = np.stack([np.stack([c, zero, s], 1), np.stack([zero, one, zero], 1), np.stack([-s, zero, c], 1)], 1)
    out = np.einsum("bij,bjk->bik", R, corners) + np.expand_dims(boxes[:, :3], 2)
    return np.transpose(out, (0, 2, 1))


def box_record(a):
    """The half-space test's constants of box array a: centre, half extents (l, h, w) / 2, cos and sin of ry."""
    r = np.zeros(1, dtype=np.dtype(_lib.RefineBox))[0]
    r["center"] = a[:3]
    r["half"] = [a[3] / 2, a[5] / 2, a[4] / 2]
    r["cs"], r["sn"] = np.cos(a[6]), np.sin(a[6])
    return r


def _check_box(a, obj, extents=True):
    if not np.isfinite(a).all():
        raise ValueError("%s: the 3-D box must be finite, got %s" % (obj.line, a.tolist()))
    if extents and not (a[3] > 0 and a[4] > 0 and a[5] > 0):
        raise ValueError("%s: the 3-D box needs positive l, w, h, got %r, %r, %r" % (obj.line, a[3], a[4], a[5]))


def is_diff(obj):
    return obj.occlusion > 2 or obj.truncation > 0.5 or obj.ymax - obj.ymin < 25


def ground_truth_boxes(objects, type_whitelist, remove_diff):
    """extract_boxes (:25-53): the whitelisted (exact type) ground truth that remove_diff keeps, in line order."""
    return [o for o in objects if o.type in type_whitelist and not (remove_diff and is_diff(o))]


def job_table(mode, image_ids, objects, gt_objects, type_whitelist, remove_diff=False, perturb=False, augment=1,
              rng=np.random):
    """The jobs of one extraction in the reference's order, with every per-box constant.  -> (jobs, gts): jobs a list
    of dicts (frame id, the cutting box array `cut`, its object, `gt` the label ground truth's position in gts (GT
    mode), `det` the detection's position in the matched table); gts {frame id: [ground truth KittiObject]}."""
    jobs, gts = [], {}
    for idx in image_ids:
        idx = int(idx)
        if mode == _lib.REFINE_DET:
            for obj in objects[idx]:
                if obj.type not in type_whitelist:
                    continue
                a = obj_array(obj)
                _check_box(a, obj)
                if obj.ymax - obj.ymin < 5 or obj.xmax - obj.xmin < 1:     # :739-741, decided on the host
                    continue
                enl = a.copy()
                enl[3:6] = enl[3:6] * RATIO
                jobs.append(dict(frame=idx, obj=obj, cut=enl))
            continue
        g = ground_truth_boxes(gt_objects[idx], type_whitelist, remove_diff)
        if mode == _lib.REFINE_MATCHED:
            if not g:
                continue                                                     # :458-459
            gts[idx] = g
            for obj in objects[idx]:
                if obj.type not in type_whitelist:
                    continue
                a = obj_array(obj)
                _check_box(a, obj, extents=False)       # extents: once matched (check_matched_extents)
                enl = a.copy()
                enl[3:6] = enl[3:6] * RATIO
                jobs.append(dict(frame=idx, obj=obj, cut=enl, box=a))
            continue
        gts[idx] = g
        for k, obj in enumerate(g):
            a = obj_array(obj)
            _check_box(a, obj)
            enl = a.copy()
            enl[3:6] = enl[3:6] * RATIO
            for _ in range(augment):
                if perturb:
                    enl = random_shift_rotate_box3d(enl, PERTURB_RATIO, rng)
                jobs.append(dict(frame=idx, obj=obj, cut=enl, gt=k))
    return jobs, gts


def gt_table(frame_ids, gts):
    """The ground truth {frame id: [KittiObject]} of the frames frame_ids (none without an entry) -> (their objects
    in frame_ids order, each frame's first position among them: F + 1 int32 offsets)."""
    per_frame = [gts.get(k, []) for k in frame_ids]
    return [o for g in per_frame for o in g], csr_offsets([len(g) for g in per_frame])


def check_matched_extents(jobs, gt_flat, job_gt):
    """Matched mode: extract_frustum_det_data triangulates a detection's box and its ground truth's only once the
    detection is matched (:493-532), so only matched pairs need positive extents.  job_gt[j] >= 0: job j matched
    gt_flat[job_gt[j]]."""
    for j, g in enumerate(job_gt):
        if g >= 0:
            _check_box(jobs[j]["box"], jobs[j]["obj"])
            _check_box(obj_array(gt_flat[g]), gt_flat[g])


def frustum_angle(cut):
    return -1 * np.arctan2(cut[2], cut[0])


# ------------------------------------------------------------------------------ result
_GT_NAMES = ("id_list", "box3d_list", "input_list", "label_list", "type_list", "heading_list", "size_list",
             "frustum_angle_list", "box2d_list", "calib_list", "pred_box3d_list", "pred_box3d_size_list",
             "pred_box3d_angle_list")
_DET_NAMES = ("id_list", "box2d_list", "input_list", "type_list", "frustum_angle_list", "prob_list", "calib_list",
              "pred_box3d_list", "pred_box3d_size_list", "pred_box3d_angle_list")


class RefineFrustums(LabelledFrustums):
    """One extraction (LabelledFrustums) in `mode`, without labels (label None) for detections; the lists are the
    provider's (datasets/provider_sample_refine.py:85-117)."""

    def __init__(self, mode, points, offsets, label, counts, job_index, lists, stream=None):
        super().__init__(points, offsets, label, counts, job_index, stream)
        self.mode = mode
        self.has_labels = mode != _lib.REFINE_DET
        self.pickle_names = _GT_NAMES if self.has_labels else _DET_NAMES
        for n in ("id_list", "box2d_list", "type_list", "frustum_angle_list", "prob_list", "calib_list",
                  "box3d_list", "heading_list", "size_list", "pred_box3d_list", "pred_box3d_size_list",
                  "pred_box3d_angle_list"):
            setattr(self, n, lists.get(n))


class RefineFrustumExtractor:
    def __init__(self, type_whitelist=("Car",), device=None):
        self.type_whitelist = tuple(type_whitelist)
        self.device = cuda_device(device, "RefineFrustumExtractor")

    # ------------------------------------------------------------------ public modes
    def from_ground_truth(self, scans, calibs, image_hw, image_ids, gt, perturb=False, augment=1, rng=np.random,
                          remove_diff=False, stream=None, timer=None):
        """gt: a label_2 directory or {idx: [KittiObject]}.  rng: the np.random module or a RandomState."""
        gt = objects_of(gt, image_ids)
        jobs, gts = job_table(_lib.REFINE_GT, image_ids, None, gt, self.type_whitelist, remove_diff, perturb,
                              int(augment), rng)
        return self._run(_lib.REFINE_GT, scans, calibs, image_hw, jobs, gts, stream, timer)

    def from_matched_detections(self, scans, calibs, image_hw, image_ids, dets, gt, remove_diff=False, stream=None,
                                timer=None):
        """dets: the collector's dict or {idx: [KittiObject]} (read_result_dir); gt as for from_ground_truth."""
        dets, gt = self._dets(dets, image_ids), objects_of(gt, image_ids)
        jobs, gts = job_table(_lib.REFINE_MATCHED, image_ids, dets, gt, self.type_whitelist, remove_diff)
        return self._run(_lib.REFINE_MATCHED, scans, calibs, image_hw, jobs, gts, stream, timer)

    def from_detections(self, scans, calibs, image_hw, image_ids, dets, stream=None, timer=None):
        dets = self._dets(dets, image_ids)
        jobs, _ = job_table(_lib.REFINE_DET, image_ids, dets, None, self.type_whitelist)
        return self._run(_lib.REFINE_DET, scans, calibs, image_hw, jobs, {}, stream, timer)

    def from_collected(self, scans, calibs, image_hw, image_ids, collected, strides=REFINE_STRIDES, stream=None,
                       timer=None):
        """from_detections(.., collected.to_dict()) without the rows leaving the device -> CollectedRefineFrustums.
        collected: DetectionCollector.finalize_device()'s CollectedDetections; strides: those of the records."""
        return self._run_collected(_lib.REFINE_DET, scans, calibs, image_hw, image_ids, collected, None, False,
                                   strides, stream, timer)

    def from_matched_collected(self, scans, calibs, image_hw, image_ids, collected, gt, remove_diff=False,
                               strides=REFINE_STRIDES, stream=None, timer=None):
        """from_matched_detections(.., collected.to_dict(), gt, remove_diff) without the rows leaving the device."""
        return self._run_collected(_lib.REFINE_MATCHED, scans, calibs, image_hw, image_ids, collected, gt,
                                   remove_diff, strides, stream, timer)

    @property
    def iou_thresh(self):
        return iou_thresh(self.type_whitelist)

    @staticmethod
    def _dets(dets, image_ids):
        """Images without an entry have no detections (the collector's dict omits them)."""
        if any(len(v) and not isinstance(v, list) for v in dets.values()):
            dets = objects_from_detections(dets)
        return {int(i): list(dets.get(int(i), [])) for i in image_ids}

    # ------------------------------------------------------------------ device calls
    def _run(self, mode, scans, calibs, image_hw, jobs, gts, stream, timer):
        dev = self.device
        frame_ids, fpos = frame_order(jb["frame"] for jb in jobs)
        gt_flat, gt_off = gt_table(frame_ids, gts)
        J = len(jobs)
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            if J == 0:
                return self._result(mode, *empty_outputs(dev, 4, mode != _lib.REFINE_DET), np.zeros(0, np.int64),
                                    np.zeros(0, np.int64), np.zeros(0, np.int64), jobs, gt_flat, calibs, stream)
            job_frame = np.array([fpos[jb["frame"]] for jb in jobs], dtype=np.int32)
            if mode == _lib.REFINE_GT:
                job_ref = np.array([gt_off[f] + jb["gt"] for f, jb in zip(job_frame, jobs)], dtype=np.int32)
            elif mode == _lib.REFINE_MATCHED:
                job_ref = np.arange(J, dtype=np.int32)                 # one job per detection
            else:
                job_ref = np.zeros(J, dtype=np.int32)
            a = _lib.RefineExtractArgs()
            parts = [(a, "jobs", np.array([box_record(jb["cut"]) for jb in jobs], dtype=np.dtype(_lib.RefineBox))),
                     (a, "job_frame", job_frame), (a, "job_ref", job_ref)]
            if mode == _lib.REFINE_MATCHED:
                parts.append((a, "det_corners", iou_corners(np.stack([jb["box"] for jb in jobs]))))

            def check(words):
                if mode == _lib.REFINE_MATCHED:
                    check_matched_extents(jobs, gt_flat, words[J:2 * J])

            words, kept, out = self._extract(a, mode, scans, calibs, image_hw, frame_ids, gt_flat, gt_off, job_frame,
                                             parts, check, stream, timer)
        job_points, job_gt = words[:J], words[J:2 * J]
        return self._result(mode, out["points"], out["offsets"], out["labels"], job_points[kept].astype(np.int64),
                            kept.astype(np.int64), job_gt[kept].astype(np.int64), jobs, gt_flat, calibs, stream)

    def _run_collected(self, mode, scans, calibs, image_hw, image_ids, collected, gt, remove_diff, strides, stream,
                       timer):
        dev = self.device
        mark = timer if timer is not None else (lambda name: None)
        strides = [float(s) for s in strides]
        if not 1 <= len(strides) <= _lib.MAX_SCALES:
            raise ValueError("need 1..%d strides" % _lib.MAX_SCALES)
        gts = None
        if mode == _lib.REFINE_MATCHED:
            gt = objects_of(gt, image_ids)
            gts = {int(i): ground_truth_boxes(gt[int(i)], self.type_whitelist, remove_diff) for i in image_ids}
        plan = collected_plan(image_ids, collected, self.type_whitelist, gts)
        frame_ids, J = plan["frame_ids"], int(plan["offsets"][-1])
        gt_flat, gt_off = gt_table(frame_ids, gts or {})
        G = len(gt_flat)
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            if collected.stream.cuda_stream != stream.cuda_stream:
                stream.wait_stream(collected.stream)
            if J == 0:
                return CollectedRefineFrustums.empty(mode, dev, strides, stream)
            f64 = lambda *shape: torch.empty(shape, dtype=torch.float64, device=dev)
            i32 = lambda n: torch.empty(n, dtype=torch.int32, device=dev)
            jobs = f64(J, 8)                                       # fcn_refine_box
            job_frame, job_ref = i32(J), i32(J)
            job_data = torch.empty((J, C.sizeof(_lib.RefineJobData)), dtype=torch.uint8, device=dev)
            det_c = f64(J, 24) if mode == _lib.REFINE_MATCHED else None
            ja = _lib.RefineJobsArgs()
            ja.mode, ja.num_pieces, ja.num_jobs, ja.num_rows = mode, len(plan["row"]), J, collected.num_rows
            ja.rows = collected.rows.data_ptr()
            ja.host_piece_offsets, ja.host_piece_row = plan["offsets"].ctypes.data, plan["row"].ctypes.data
            ja.job_data = job_data.data_ptr()
            a = _lib.RefineExtractArgs()
            for args in (ja, a):                # the jobs ja writes and a reads
                args.jobs, args.job_frame, args.job_ref = jobs.data_ptr(), job_frame.data_ptr(), job_ref.data_ptr()
                args.det_corners = None if det_c is None else det_c.data_ptr()
            labels = mode == _lib.REFINE_MATCHED
            gt_arr = [obj_array(o) for o in gt_flat]
            terms = gt_terms(gt_flat, gt_arr) if labels else None       # host work, ahead of the device calls

            def count(words):                   # the jobs' status words follow job_points and job_gt
                ja.status = words.data_ptr() + 8 * J
                _lib.call("fcn_refine_jobs_from_rows", C.byref(ja), stream.cuda_stream)
                _lib.call("fcn_refine_extract_count", C.byref(a), stream.cuda_stream)
                mark("count")

            words, kept, out = self._extract(
                a, mode, scans, calibs, image_hw, frame_ids, gt_flat, gt_off,
                np.repeat(plan["frame"], np.diff(plan["offsets"])),
                [(ja, "piece_" + k, plan[k]) for k in ("offsets", "row", "frame", "image", "class")],
                lambda words: check_collected(mode, plan, collected, words[J:2 * J], words[2 * J:3 * J], gt_flat,
                                              gt_arr),
                stream, timer, count, J)
            K, S = len(kept), len(strides)
            tab, tptrs = upload([kept.astype(np.int32)] + ([words[J:2 * J], terms] if labels else []), dev)
            lists = f64(K, _lib.REFINE_LIST_COLS)
            records = torch.zeros((K, C.sizeof(_lib.TrainFrustum)), dtype=torch.uint8, device=dev)
            rwords = torch.empty((K, S + 1), dtype=torch.int32, device=dev)
            ta = _lib.RefineFrustumTableArgs()
            ta.mode, ta.labels, ta.num_kept, ta.num_jobs, ta.num_gt, ta.num_scales = mode, int(labels), K, J, G, S
            for q, st in enumerate(strides):
                ta.stride[q] = st
            ta.kept, ta.job_data = tptrs[0], job_data.data_ptr()
            if labels:
                ta.job_gt, ta.gt_terms = tptrs[1:]
            ta.lists, ta.records, ta.words = lists.data_ptr(), records.data_ptr(), rwords.data_ptr()
            mark("table_start")
            _lib.call("fcn_refine_frustum_table", C.byref(ta), stream.cuda_stream)
            mark("table")
        pk = np.searchsorted(plan["offsets"], kept, side="right") - 1
        kept_gt = words[J:2 * J][kept].astype(np.int64)
        return CollectedRefineFrustums(mode, out["points"], out["offsets"], out["labels"],
                                       words[kept].astype(np.int64), kept.astype(np.int64),
                                       plan["image"][pk].tolist(), [plan["types"][p] for p in pk.tolist()],
                                       bool((plan["class"][pk] >= 0).all()), lists, records, rwords, strides,
                                       kept_gt, gt_flat, calibs, stream)

    def _extract(self, a, mode, scans, calibs, image_hw, frame_ids, gt_flat, gt_off, job_frame, parts, check, stream,
                 timer, count=None, extra_words=0):
        """Both job sources' run_extract into the RefineExtractArgs `a`, jobs in frames job_frame.  The frames, the
        ground truth (gt_table's) and, in matched mode, its corners and pair offsets go up in one copy with `parts`,
        the job source's (struct, field, host array) triples, each field set to its array's device address.
        check(words) runs before the outputs are allocated.  -> run_extract's (words, kept, out)."""
        dev = self.device
        J, G = len(job_frame), len(gt_flat)
        sc, frames, so = scan_table(scans, calibs, image_hw, frame_ids, dev, "RefineFrustumExtractor")
        gt_arr = [obj_array(o) for o in gt_flat]
        common = [bytes(frames), so, np.array([box_record(g) for g in gt_arr], dtype=np.dtype(_lib.RefineBox))]
        if mode == _lib.REFINE_MATCHED:
            po = csr_offsets(np.diff(gt_off)[job_frame])
            common += [iou_corners(np.stack(gt_arr)) if G else np.zeros(0), gt_off, po]
        inp, ptrs = upload(common + [p for _, _, p in parts], dev)
        for (struct, field, _), ptr in zip(parts, ptrs[len(common):]):
            setattr(struct, field, ptr)
        a.mode, a.num_frames, a.num_points, a.num_jobs, a.num_gt = mode, len(frame_ids), int(so[-1]), J, G
        a.iou_thresh = self.iou_thresh
        a.frames, a.scan_offsets = ptrs[:2]
        a.gt_boxes = ptrs[2] if G > 0 else None
        if mode == _lib.REFINE_MATCHED:
            a.num_dets, a.num_pairs, a.det_frame = J, int(po[-1]), a.job_frame
            a.gt_corners, a.gt_offsets, a.pair_offsets = ptrs[3:6]

        def outputs(K, M, words):
            check(words)
            return {"labels": None if mode == _lib.REFINE_DET else torch.empty(M, dtype=torch.uint8, device=dev)}

        return run_extract("refine_extract", a, sc, so, J, ("job_points", "job_gt"), outputs, dev, stream, timer,
                           "jobs or pairs reference no frame or box", extra_words, count)

    @staticmethod
    def _result(mode, points, offsets, label, counts, kept, kept_gt, jobs, gt_flat, calibs, stream):
        L = {n: [] for n in ("id_list", "box2d_list", "type_list", "frustum_angle_list", "prob_list", "calib_list",
                             "box3d_list", "heading_list", "size_list", "pred_box3d_list", "pred_box3d_size_list",
                             "pred_box3d_angle_list")}
        for j, g in zip(kept.tolist(), kept_gt.tolist()):
            jb = jobs[j]
            obj, cut = jb["obj"], jb["cut"]
            L["id_list"].append(jb["frame"])
            L["type_list"].append(obj.type)
            L["frustum_angle_list"].append(frustum_angle(cut))
            L["calib_list"].append(calibs[jb["frame"]])
            L["pred_box3d_list"].append(compute_box_3d_obj_array(cut))
            L["pred_box3d_size_list"].append(cut[3:6])
            L["pred_box3d_angle_list"].append(cut[-1])
            if mode == _lib.REFINE_DET:
                L["box2d_list"].append(obj.box2d)
                L["prob_list"].append(obj.score)
            else:
                gt = gt_flat[g]
                L["box3d_list"].append(compute_box_3d_obj_array(obj_array(gt)))
                L["heading_list"].append(gt.ry)
                L["size_list"].append(np.array([gt.l, gt.w, gt.h]))
                L["box2d_list"].append(gt.box2d)
        if mode != _lib.REFINE_DET:
            L["prob_list"] = None
        else:
            for n in ("box3d_list", "heading_list", "size_list"):
                L[n] = None
        return RefineFrustums(mode, points, offsets, label, counts, kept, L, stream)


# ------------------------------------------------------------------------------ from the collector's device rows
def collected_plan(image_ids, collected, type_whitelist, gts=None):
    """The gather plan of fcn_refine_jobs_from_rows from the collector's segment metadata alone, in the dict path's job
    order: the images of image_ids (in matched mode, gts given, only those with ground truth), the whitelisted classes
    of each in the collector's dict order, their kept rows.  -> dict of the pieces (one per segment with kept rows):
    offsets (P + 1) int32 (the first job of each), row / frame / image / class (P) int32 (the first row, the frame's
    position in frame_ids, the image, the KITTI_CLASSES index or -1), types (P) class names, and frame_ids (the images
    with jobs, in first-appearance order)."""
    by_image = {}
    for s in collected.order.tolist():
        idx, ct = collected.segments[s]
        if ct in type_whitelist and collected.host_keep_count[s] > 0:
            by_image.setdefault(int(idx), []).append(s)
    segs, frame, pos = [], [], {}
    for idx in image_ids:
        idx = int(idx)
        if gts is not None and not gts[idx]:
            continue                                                     # :458-459
        for s in by_image.get(idx, ()):
            segs.append(s)
            frame.append(pos.setdefault(idx, len(pos)))
    segs = np.asarray(segs, dtype=np.int64)
    types = [collected.segments[s][1] for s in segs.tolist()]
    return {"offsets": csr_offsets(collected.host_keep_count[segs]),
            "row": np.ascontiguousarray(collected.host_seg_offsets[segs], dtype=np.int32),
            "frame": np.asarray(frame, dtype=np.int32),
            "image": np.array([int(collected.segments[s][0]) for s in segs.tolist()], dtype=np.int32),
            "class": np.array([KITTI_CLASSES.index(t) if t in KITTI_CLASSES else -1 for t in types], dtype=np.int32),
            "types": types, "segs": segs, "frame_ids": list(pos)}


def gt_terms(gt_flat, gt_arr):
    """The ground-truth terms of the refine records, per ground truth, with frustum_table's expressions."""
    t = np.zeros(len(gt_flat), dtype=np.dtype(_lib.RefineGtTerms))
    for r, o, a in zip(t, gt_flat, gt_arr):
        b3 = compute_box_3d_obj_array(a)
        size = np.array([o.l, o.w, o.h])
        l, w, h = size
        r["center"], r["heading"], r["size"] = (b3[0, :] + b3[6, :]) / 2, o.ry, size
        r["dist"] = np.sqrt(np.sum(l ** 2 + w ** 2))
    return t


def collected_object(plan, collected, j):
    """Job j's row as from_detections sees it: the KittiObject objects_from_detections makes (one row read)."""
    p = int(np.searchsorted(plan["offsets"], j, side="right") - 1)
    n = int(j - plan["offsets"][p])
    row = collected.rows[int(plan["row"][p]) + n].cpu().numpy()
    idx, ct = int(plan["image"][p]), plan["types"][p]
    r = detection_records(row.reshape(1, 12), ct)[0]
    return KittiObject(ct, -1.0, -1, float(r[1]), [float(v) for v in r[2:6]], float(r[6]), float(r[7]), float(r[8]),
                       [float(v) for v in r[9:12]], float(r[12]), float(r[13]), "detections[%d][%r] row %d" % (idx, ct, n))


def check_collected(mode, plan, collected, job_gt, status, gt_flat, gt_arr):
    """The ValueError the dict path raises for the same rows, from the jobs' status words (read back with the count):
    a non-finite box, or (in matched mode only for a matched pair, check_matched_extents) a non-positive extent."""
    bad = status & (_lib.REFINE_ROW_NONFINITE | (_lib.REFINE_ROW_EXTENTS if mode == _lib.REFINE_DET else 0))
    if bad.any():
        j = int(np.argmax(bad != 0))
        obj = collected_object(plan, collected, j)
        _check_box(obj_array(obj), obj, mode == _lib.REFINE_DET)
    if mode != _lib.REFINE_MATCHED:
        return
    m = np.flatnonzero(job_gt >= 0)
    gt_bad = np.array([not (np.isfinite(a).all() and a[3] > 0 and a[4] > 0 and a[5] > 0) for a in gt_arr], bool)
    bad = ((status[m] & _lib.REFINE_ROW_EXTENTS) != 0) | gt_bad[job_gt[m]] if len(m) else np.zeros(0, bool)
    if bad.any():
        j = int(m[np.argmax(bad)])
        obj = collected_object(plan, collected, j)
        _check_box(obj_array(obj), obj)
        g = gt_flat[job_gt[j]]
        _check_box(obj_array(g), g)


class CollectedRefineFrustums(RefineFrustums):
    """RefineFrustums from the collector's device rows.  Device: points, offsets, label as RefineFrustums; lists (K,
    FCN_REFINE_LIST_COLS) float64 and its views frustum_angle (K), pred_box3d (K, 8, 3), pred_box3d_size (K, 3),
    pred_box3d_angle (K), box2d (K, 4), prob (K); frustum_records (K fcn_train_frustum records for record_strides,
    which TrainBatchBuilder.from_frustums installs as they are) and record_words (K, S + 1) int32 (T per scale, the
    degenerate flag).  Host, at once: counts, job_index, id_list, type_list.  The provider's other lists are built on
    first use from one copy of `lists`."""

    _LAZY = ("box2d_list", "frustum_angle_list", "prob_list", "calib_list", "box3d_list", "heading_list", "size_list",
             "pred_box3d_list", "pred_box3d_size_list", "pred_box3d_angle_list")

    def __init__(self, mode, points, offsets, label, counts, job_index, id_list, type_list, classes_ok, lists,
                 records, record_words, strides, kept_gt, gt_flat, calibs, stream):
        LabelledFrustums.__init__(self, points, offsets, label, counts, job_index, stream)
        self.mode = mode
        self.has_labels = mode != _lib.REFINE_DET
        self.pickle_names = _GT_NAMES if self.has_labels else _DET_NAMES
        self.id_list, self.type_list = id_list, type_list
        K = len(id_list)
        self.lists = lists
        self.frustum_angle, self.pred_box3d = lists[:, 0], lists[:, 1:25].view(K, 8, 3)
        self.pred_box3d_size, self.pred_box3d_angle = lists[:, 25:28], lists[:, 28]
        self.box2d, self.prob = lists[:, 29:33], lists[:, 33]
        self.frustum_records, self.record_words = records, record_words
        self.record_strides, self.record_labels = list(strides), self.has_labels
        self.record_classes = KITTI_CLASSES if classes_ok else None
        self._kept_gt, self._gt_flat, self._calibs = kept_gt, gt_flat, calibs

    @classmethod
    def empty(cls, mode, dev, strides, stream):
        z = lambda *shape, dt=torch.float64: torch.zeros(shape, dtype=dt, device=dev)
        return cls(mode, *empty_outputs(dev, 4, mode != _lib.REFINE_DET), np.zeros(0, np.int64),
                   np.zeros(0, np.int64), [], [], True, z(0, _lib.REFINE_LIST_COLS),
                   z(0, C.sizeof(_lib.TrainFrustum), dt=torch.uint8), z(0, len(strides) + 1, dt=torch.int32), strides,
                   np.zeros(0, np.int64), [], {}, stream)

    def __getattr__(self, name):
        if name in CollectedRefineFrustums._LAZY:
            self._host_lists()
            return self.__dict__[name]
        raise AttributeError(name)

    def _host_lists(self):
        self.wait()
        L = self.lists.cpu().numpy()
        K = len(L)
        d = {"frustum_angle_list": list(L[:, 0]), "pred_box3d_list": list(L[:, 1:25].reshape(K, 8, 3)),
             "pred_box3d_size_list": list(L[:, 25:28]), "pred_box3d_angle_list": list(L[:, 28]),
             "calib_list": [self._calibs[k] for k in self.id_list]}
        if self.mode == _lib.REFINE_DET:
            d.update(box2d_list=list(L[:, 29:33]), prob_list=L[:, 33].tolist(), box3d_list=None, heading_list=None,
                     size_list=None)
        else:
            gts = [self._gt_flat[g] for g in self._kept_gt.tolist()]
            d.update(box2d_list=[g.box2d for g in gts], prob_list=None,
                     box3d_list=[compute_box_3d_obj_array(obj_array(g)) for g in gts],
                     heading_list=[g.ry for g in gts], size_list=[np.array([g.l, g.w, g.h]) for g in gts])
        self.__dict__.update(d)
