"""SUN-RGBD 3-D detection evaluation on the device: per-class average precision and precision / recall curves from the
detection dict, without the reference's per-pair Boost calls (train/sunrgbd_eval/eval_det.py, called after
write_detection_results in train/test_net_det_sunrgbd.py:264-276).

    gt = SunrgbdGroundTruth.from_gt_dir("train/sunrgbd_eval/gt_boxes")     # parsed and converted once, on the device
    res = SunrgbdEvaluator(gt).evaluate(col.finalize())   # DetectionCollector's {idx: {class: (n, 12)}}, or test()'s
    for line in res.lines():                              # '<class>: %.5f' in sorted class order, then 'mean_AP: %.5f'
        logging.info(line)
    res.ap["chair"], res.rec["chair"], res.prec["chair"]  # float, (nd,) float64, (nd,) float64

Semantics are those of eval_det(pred_all, gt_all, ovthresh=0.25, use_07_metric=False) (csrc/sunrgbd_eval.cu):
  * ground truth: '<class>_gt_boxes.dat' rows (four bird's-eye xy corners, zmin, zmax) with the image ids of
    '<class>_gt_imgids.txt', converted as get_gt_cls converts them (compare_matlab_python_eval.py:15-67);
  * detections: rows [x1,y1,x2,y2, tx,ty,tz, l,w,h, ry, score] as float32, corners by compute_box_3d
    (datasets/data_utils.py:44-70: float32 cos / sin of the float32 angle, float64 corners), gathered per class in
    dict order, then row order (write_detection_results, eval_det_cls :116-126); ``evaluate_corners`` takes the
    reference's own {class: {idx: [(corners (8, 3), score)]}} instead;
  * order: score descending, STABLE - of two equal scores the earlier detection in gather order ranks first, and -0.0
    equals 0.0 (the reference's np.argsort(-confidence) leaves the tie order to numpy's sort implementation);
  * matching: the 3-D IoU of rbbox_iou_3d_pair<double> against the same image's ground truth of the class, the first
    maximum; a TP needs IoU > ovthresh and a ground truth not yet taken, with no fall-back to another one;
  * rec and prec are bit-identical to the reference's; ap (voc_ap) is summed in a fixed order, within a few ulps of
    numpy's pairwise sum; mean_ap is np.mean of the per-class APs.
Divergence: a class with ground truth and no detection gets AP 0 and empty curves (the reference raises KeyError).
Detections of classes without ground truth are ignored, as in the reference.  Image ids are integers (integral floats
are accepted).  Detections in images without ground truth of their class are false positives, as in the reference;
when the ground truth is given the split's ``image_ids``, an id in neither raises KeyError.  No CPU fallback: a CPU
device raises.  PR-curve plots are not drawn: the curves are returned as arrays."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from ._host import csr_offsets, cuda_device, upload, workspace

CLASS_NAMES = ("bed", "table", "sofa", "chair", "toilet", "desk", "dresser", "night_stand", "bookshelf", "bathtub")
_RES = C.sizeof(_lib.SunrgbdEvalResult)


def image_key(idx) -> int:
    """An image id as an int; ids are integers, and floats are accepted only when integral (the id files hold them
    as floats)."""
    if isinstance(idx, (int, np.integer)):
        return int(idx)
    f = float(idx)
    if not f.is_integer():
        raise ValueError("image id %r is not an integer" % (idx,))
    return int(f)


def read_gt_files(gt_boxes_dir, classname):
    """'<class>_gt_boxes.dat' and '<class>_gt_imgids.txt' as np.loadtxt reads them -> ((n, 10) float64 rows, (n,)
    int64 image ids).  A one-row class stays (1, 10)."""
    boxes = np.loadtxt(os.path.join(gt_boxes_dir, "%s_gt_boxes.dat" % classname), ndmin=2)
    ids = np.loadtxt(os.path.join(gt_boxes_dir, "%s_gt_imgids.txt" % classname), ndmin=1)
    if boxes.size == 0:
        boxes = boxes.reshape(0, 10)
    if boxes.shape[1] != 10:
        raise ValueError("%s_gt_boxes.dat: rows of 10 values are required, got %d" % (classname, boxes.shape[1]))
    if len(ids) != len(boxes):
        raise ValueError("%s: %d boxes but %d image ids" % (classname, len(boxes), len(ids)))
    return boxes, np.array([image_key(i) for i in ids.tolist()], dtype=np.int64)


def gt_corners(boxes):
    """(n, 10) ground-truth rows -> (n, 8, 3) float64 corners: the xy ring made clockwise (is_clockwise), zmax on
    corners 0-3 and zmin on 4-7 (box_conversion), to camera axes (x, -z, y) (flip_axis_to_camera), then the two
    halves swapped (wrapper), so corners 0-3 have y = -zmin and 4-7 y = -zmax."""
    b = np.asarray(boxes, dtype=np.float64).reshape(-1, 10)
    xy = b[:, :8].reshape(-1, 4, 2)
    x, y = xy[..., 0], xy[..., 1]
    cw = (x * np.roll(y, 1, axis=1)).sum(1) - (y * np.roll(x, 1, axis=1)).sum(1) > 0
    xy = np.where(cw[:, None, None], xy, xy[:, ::-1])
    out = np.empty((len(b), 8, 3), dtype=np.float64)
    out[:, :, 0] = np.tile(xy[..., 0], 2)
    out[:, :, 2] = np.tile(xy[..., 1], 2)
    out[:, :4, 1] = -b[:, 8:9]
    out[:, 4:, 1] = -b[:, 9:10]
    return out


def det_corners(rows):
    """(n, 12) detection rows -> (n, 8, 3) float64 corners of compute_box_3d(row[4:7], row[7:10], row[10]) on the
    float32 row: float32 cos / sin and half sizes, then the rotation about y and the translation in float64."""
    r = np.asarray(rows, dtype=np.float32).reshape(-1, 12)
    c = np.cos(r[:, 10]).astype(np.float64)[:, None]
    s = np.sin(r[:, 10]).astype(np.float64)[:, None]
    hl, hw, hh = ((r[:, k] / np.float32(2)).astype(np.float64)[:, None] for k in (7, 8, 9))
    sx = np.array([1, 1, -1, -1, 1, 1, -1, -1], dtype=np.float64)
    sy = np.array([1, 1, 1, 1, -1, -1, -1, -1], dtype=np.float64)
    sz = np.array([1, -1, -1, 1, 1, -1, -1, 1], dtype=np.float64)
    xc, yc, zc = hl * sx, hh * sy, hw * sz
    out = np.empty((len(r), 8, 3), dtype=np.float64)
    out[:, :, 0] = (c * xc + s * zc) + r[:, 4:5].astype(np.float64)
    out[:, :, 1] = yc + r[:, 5:6].astype(np.float64)
    out[:, :, 2] = (-s * xc + c * zc) + r[:, 6:7].astype(np.float64)
    return out


class SunrgbdGroundTruth:
    """The ground truth of every class, converted once and kept on the device: rows grouped per class, and within a
    class per image (in file order, so the first of two equal overlaps wins as in the reference).

    ``gt`` maps each class, in evaluation order, to (corners (n, 8, 3), image ids (n,)).  ``image_ids`` (optional, a
    split's full id list) names the images detections may come from: with it, a detection image found neither there
    nor in the ground truth raises KeyError (a mismatched id map); without it every integral id is accepted."""

    def __init__(self, gt, image_ids=None, device=None):
        self.device = cuda_device(device, "SunrgbdGroundTruth")
        self.classes = tuple(gt)
        if len(self.classes) > _lib.SUNRGBD_MAX_CLASSES:
            raise ValueError("at most %d classes" % _lib.SUNRGBD_MAX_CLASSES)
        self.class_index = {c: i for i, c in enumerate(self.classes)}
        corners, seg_counts, cls_counts = [], [], []
        self.segment_of = {}                      # (class index, image id) -> segment
        for ci, name in enumerate(self.classes):
            cor, ids = gt[name]
            cor = np.asarray(cor, dtype=np.float64).reshape(-1, 8, 3)
            keys = np.array([image_key(i) for i in np.asarray(ids).reshape(-1).tolist()], dtype=np.int64)
            if len(keys) != len(cor):
                raise ValueError("%s: %d boxes but %d image ids" % (name, len(cor), len(keys)))
            if not np.isfinite(cor).all():
                raise ValueError("%s: non-finite ground-truth corners" % name)
            order = np.argsort(keys, kind="stable")
            uniq, counts = np.unique(keys[order], return_counts=True)
            for k in uniq.tolist():
                self.segment_of[(ci, k)] = len(seg_counts)
                seg_counts.append(0)
            seg_counts[len(seg_counts) - len(uniq):] = counts.tolist()
            corners.append(cor[order])
            cls_counts.append(len(cor))
        self.known_images = (None if image_ids is None else
                             {k for (_, k) in self.segment_of} | {image_key(i) for i in image_ids})
        self.host_segment_offsets = csr_offsets(seg_counts)
        self.host_class_offsets = csr_offsets(cls_counts)
        self.num_gt = int(self.host_class_offsets[-1])
        self.num_segments = len(seg_counts)
        flat = np.concatenate(corners) if corners else np.zeros((0, 8, 3))
        self.corners = torch.from_numpy(np.ascontiguousarray(flat)).to(self.device)
        self.segment_offsets = torch.from_numpy(self.host_segment_offsets).to(self.device)
        self.class_offsets = torch.from_numpy(self.host_class_offsets).to(self.device)

    @classmethod
    def from_gt_dir(cls, gt_boxes_dir, classes=CLASS_NAMES, image_ids=None, device=None):
        gt = {}
        for name in classes:
            boxes, ids = read_gt_files(gt_boxes_dir, name)
            gt[name] = (gt_corners(boxes), ids)
        return cls(gt, image_ids, device)


class SunrgbdEvalResult:
    """Per class (every class of the ground truth): rec[c], prec[c] ((nd_c,) float64, in score order), ap[c],
    npos[c], nd[c]; mean_ap over the classes."""

    def __init__(self, classes, raw, rec, prec, det_off):
        self.classes = classes
        self.rec, self.prec, self.ap, self.npos, self.nd = {}, {}, {}, {}, {}
        for i, name in enumerate(classes):
            a, b = int(det_off[i]), int(det_off[i + 1])
            self.rec[name], self.prec[name] = rec[a:b].copy(), prec[a:b].copy()
            self.ap[name], self.npos[name], self.nd[name] = float(raw[i].ap), int(raw[i].npos), int(raw[i].nd)
        self.mean_ap = float(np.mean([self.ap[c] for c in classes])) if classes else float("nan")

    def lines(self):
        """The lines eval_det logs: '<class>: %.5f' in sorted class-name order, then 'mean_AP: %.5f'."""
        return ["%s: %.5f" % (c, self.ap[c]) for c in sorted(self.ap)] + ["mean_AP: %.5f" % self.mean_ap]


class SunrgbdEvaluator:
    def __init__(self, gt: SunrgbdGroundTruth):
        self.gt = gt
        self.device = gt.device

    def _check_image(self, idx):
        key = image_key(idx)
        if self.gt.known_images is not None and key not in self.gt.known_images:
            raise KeyError("detections for image %d, which is neither in the ground truth nor in its image_ids" % key)
        return key

    def _segments(self, ci, key, n):
        return np.full(n, self.gt.segment_of.get((ci, key), -1), dtype=np.int32)

    def evaluate(self, det_results, ovthresh=0.25, stream=None, timer=None):
        """{idx: {class: (n, 12) rows}} (DetectionCollector.finalize() or test()'s dict) -> SunrgbdEvalResult."""
        rows = [[] for _ in self.gt.classes]
        segs = [[] for _ in self.gt.classes]
        for idx, by_class in det_results.items():
            key = self._check_image(idx)
            for name, dets in by_class.items():
                ci = self.gt.class_index.get(name)
                if ci is None:
                    continue
                d = np.asarray(dets, dtype=np.float32).reshape(-1, 12)
                rows[ci].append(d)
                segs[ci].append(self._segments(ci, key, len(d)))
        flat = [r for per in rows for r in per]
        allrows = np.concatenate(flat) if flat else np.zeros((0, 12), np.float32)
        counts = [sum(len(r) for r in per) for per in rows]
        seg = np.concatenate([s for per in segs for s in per]) if flat else np.zeros(0, np.int32)
        return self._run(det_corners(allrows), allrows[:, 11].astype(np.float64), seg, counts, ovthresh, stream, timer)

    def evaluate_corners(self, pred_all, ovthresh=0.25, stream=None, timer=None):
        """The reference's pred_all, {class: {idx: [(corners (8, 3), score)]}} (write_detection_results' return
        value) -> SunrgbdEvalResult."""
        corners, scores, segs, counts = [], [], [], []
        for ci, name in enumerate(self.gt.classes):
            n = 0
            for idx, lst in pred_all.get(name, {}).items():
                key = self._check_image(idx)
                segs.append(self._segments(ci, key, len(lst)))
                for box, score in lst:
                    corners.append(np.asarray(box, dtype=np.float64).reshape(8, 3))
                    scores.append(float(score))
                n += len(lst)
            counts.append(n)
        for name, by_img in pred_all.items():
            if name not in self.gt.class_index:
                for idx in by_img:
                    self._check_image(idx)
        cor = np.stack(corners) if corners else np.zeros((0, 8, 3))
        seg = np.concatenate(segs) if segs else np.zeros(0, np.int32)
        return self._run(cor, np.asarray(scores, dtype=np.float64), seg, counts, ovthresh, stream, timer)

    def gather_plan(self, collected):
        """The host half of ``evaluate_collected``, from segment metadata only -> (seg_dst, seg_gt, det_class_offsets):
        per segment of the collector the first detection it owns in the gather order of ``evaluate`` (class after
        class, images in dict order, then rows; -1: not written, as for a class without ground truth), its ground-truth
        segment (or -1), and the (num_classes + 1) offsets of that order.  Every image of the dict is checked as
        ``evaluate`` checks it."""
        gt = self.gt
        S, order = collected.num_segments, collected.order
        _, img_rank = collected.image_order()
        seg_ci = np.full(len(order), -1, dtype=np.int64)
        seg_gt = np.full(S, -1, dtype=np.int32)
        checked = {}
        for j, s in enumerate(order.tolist()):
            idx, name = collected.segments[s]
            key = checked.get(idx)
            if key is None:
                key = checked[idx] = self._check_image(idx)
            ci = gt.class_index.get(name)
            if ci is not None:
                seg_ci[j] = ci
                seg_gt[s] = gt.segment_of.get((ci, key), -1)
        sel = seg_ci >= 0
        rank = np.lexsort((img_rank[sel], seg_ci[sel]))                  # class, then the image's dict position
        gathered = order[sel][rank]
        counts = collected.host_keep_count[gathered].astype(np.int64)
        seg_dst = np.full(S, -1, dtype=np.int32)
        seg_dst[gathered] = (np.cumsum(counts) - counts).astype(np.int32)
        per_class = np.bincount(seg_ci[sel], weights=collected.host_keep_count[order[sel]].astype(np.int64),
                                minlength=len(gt.classes)).astype(np.int64)
        return seg_dst, seg_gt, csr_offsets(per_class)

    def evaluate_collected(self, collected, ovthresh=0.25, stream=None, timer=None):
        """DetectionCollector.finalize_device()'s CollectedDetections -> the SunrgbdEvalResult ``evaluate`` gives for
        its dict, without the rows crossing to the host: corners, scores and ground-truth segments are written on the
        device (``fcn_det_sunrgbd_feed``) in ``evaluate``'s gather order, the plan coming from the segment keys alone.
        cos and sin are the correctly rounded float32 values (numpy's float32 loops can differ in the last bit, so a
        corner can move by an ulp or two of its magnitude)."""
        dev = self.device
        seg_dst, seg_gt, det_off = self.gather_plan(collected)
        D = int(det_off[-1])
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            if collected.stream.cuda_stream != stream.cuda_stream:
                stream.wait_stream(collected.stream)
            buf, (p_dst, p_gt, p_off) = upload([seg_dst, seg_gt, det_off], dev)
            det = torch.empty(max(D, 1) * 26 + 1, dtype=torch.float64, device=dev)    # corners | scores | segments
            dp = det.data_ptr()
            status = torch.zeros(1, dtype=torch.int32, device=dev)
            if timer is not None:
                timer("feed_start")
            a = collected.feed_args(seg_dst, seg_gt, D, (p_dst, p_gt))
            a.corners, a.scores, a.segments = dp, dp + 8 * 24 * max(D, 1), dp + 8 * 25 * max(D, 1)
            a.status = status.data_ptr()
            _lib.call("fcn_det_sunrgbd_feed", C.byref(a), stream.cuda_stream)
            return self._launch(a.corners, a.scores, a.segments, p_off, det_off, D, ovthresh, stream, timer, status)

    def _run(self, corners, scores, seg, counts, ovthresh, stream, timer):
        """(D, 8, 3) corners, (D,) scores and ground-truth segments, gathered class after class -> result.  One upload
        of the detections, one read-back of the result.  `timer(name)` (optional) is called before the first device
        call ("start") and after each of the two is enqueued (benchmarks)."""
        if not np.isfinite(scores).all():
            raise ValueError("detection scores must be finite")
        if not np.isfinite(corners).all():
            raise ValueError("detection corners must be finite")
        D = len(scores)
        det_off = csr_offsets(counts)
        dev = self.device
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            buf, ptrs = upload([np.asarray(corners, np.float64), np.asarray(scores, np.float64),
                                np.asarray(seg, np.int32), det_off], dev)
            return self._launch(*ptrs, det_off, D, ovthresh, stream, timer)

    def _launch(self, corners, scores, seg, det_off_dev, det_off, D, ovthresh, stream, timer, status=None):
        """The two evaluator entries on `stream` (current, on the evaluator's device) over device detections -> result
        after the one read back.  `status` (optional, device int32): the feed's flags, read back with the result; a
        non-finite corner or score raises ValueError as ``evaluate`` does."""
        gt, dev = self.gt, self.device
        Cn = len(gt.classes)
        a = _lib.SunrgbdEvalArgs()
        a.num_classes, a.num_gt, a.num_gt_segments, a.num_det = Cn, gt.num_gt, gt.num_segments, D
        a.ovthresh = float(ovthresh)
        a.gt_corners, a.gt_segment_offsets, a.gt_class_offsets = (gt.corners.data_ptr(),
                                                                  gt.segment_offsets.data_ptr(),
                                                                  gt.class_offsets.data_ptr())
        a.det_corners, a.det_scores, a.det_segments, a.det_class_offsets = corners, scores, seg, det_off_dev
        a.host_gt_segment_offsets = gt.host_segment_offsets.ctypes.data
        a.host_gt_class_offsets = gt.host_class_offsets.ctypes.data
        a.host_det_class_offsets = det_off.ctypes.data
        ws, nbytes = workspace("fcn_sunrgbd_eval_workspace_bytes", dev, C.byref(a))
        out = torch.zeros(Cn * _RES + 16 * D + 16, dtype=torch.uint8, device=dev)     # results | rec | prec | status
        ob = out.data_ptr()
        a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
        a.result, a.rec, a.prec = ob, ob + Cn * _RES, ob + Cn * _RES + 8 * D
        if timer is not None:
            timer("start")
        for name in ("fcn_sunrgbd_eval_match", "fcn_sunrgbd_eval_curves"):
            _lib.call(name, C.byref(a), stream.cuda_stream)
            if timer is not None:
                timer(name)
        if status is not None:
            out[Cn * _RES + 16 * D:Cn * _RES + 16 * D + 4].copy_(status.view(torch.uint8))
        back = out.cpu().numpy()                                             # the one read back
        flags = int(back[Cn * _RES + 16 * D:Cn * _RES + 16 * D + 4].view(np.int32)[0])
        if flags & _lib.DET_FEED_NONFINITE:
            raise ValueError("detection scores and corners must be finite")
        raw = (_lib.SunrgbdEvalResult * Cn).from_buffer_copy(back[:Cn * _RES].tobytes()) if Cn else []
        bad = [gt.classes[i] for i in range(Cn) if raw[i].status]
        if bad:
            raise RuntimeError("sunrgbd_eval: detection segments outside their class's ground truth: %s" % bad)
        rec = back[Cn * _RES:Cn * _RES + 8 * D].view(np.float64)
        prec = back[Cn * _RES + 8 * D:Cn * _RES + 16 * D].view(np.float64)
        return SunrgbdEvalResult(gt.classes, raw, rec, prec, det_off)
