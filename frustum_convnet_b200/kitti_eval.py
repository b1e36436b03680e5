"""KITTI object evaluation on the device: 2-D, AOS, bird's-eye-view and 3-D average precision from the detection
dict, without result files and without the reference's CPU evaluator (train/kitti_eval/evaluate_object_3d_offline,
called after write_detection_results in train/test_net_det.py:302-315).

    gt = KittiGroundTruth.from_label_dir("kitti/training/label_2", image_ids)   # parsed once, kept on the device
    ev = KittiEvaluator(gt)
    res = ev.evaluate(col.finalize())          # DetectionCollector's {idx: {class: (n, 12)}}, or test()'s dict
    print("\\n".join(res.lines()))             # the evaluator's "car_detection AP: e m h" lines
    res.ap["3d"]["car"]                        # (3,) easy / moderate / hard, as printed

Semantics are the evaluator's (csrc/kitti_eval.cu): the 41-point precision and AOS vectors per metric, class and
difficulty, and the printed AP (every 4th point / 11 * 100, summed in float32).  The detections are the text the
reference writes, without the text: alpha = compute_alpha(tx, tz, ry) on the float32 rows
(datasets/provider_sample.py:389-394), every field rounded as '%.4f' and the score as '%f', then read back
(``quantize``).  Every image of ``image_ids`` counts, with or without detections, as fill_files makes it count.
``evaluate_dir`` reads result files instead, like the evaluator's loadDetections.  A class that is never detected is
not evaluated and is absent from the result.  No CPU fallback: a CPU device raises."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from ._host import csr_offsets, cuda_device, upload, workspace

CLASS_NAMES = ("car", "pedestrian", "cyclist")
METRICS = ("image", "ground", "3d")
TYPE_CODES = {"car": _lib.KITTI_CAR, "pedestrian": _lib.KITTI_PEDESTRIAN, "cyclist": _lib.KITTI_CYCLIST,
              "van": _lib.KITTI_VAN, "person_sitting": _lib.KITTI_PERSON_SITTING, "dontcare": _lib.KITTI_DONTCARE}
OTHER = _lib.KITTI_OTHER
GT_COLS, DET_COLS, PTS = _lib.KITTI_GT_COLS, _lib.KITTI_DET_COLS, _lib.KITTI_PTS


def type_code(name: str) -> int:
    """Type names match case-insensitively (strcasecmp); every type other than the six named ones is OTHER."""
    return TYPE_CODES.get(name.lower(), OTHER)


def quantize(v, decimals):
    """'%.<decimals>f' followed by strtod, for float32 values: a float32 times 10^4 or 10^6 is exact in float64, so
    rounding that product to an integer (ties to even, as printf rounds an exact tie) and dividing gives the double
    strtod reads back."""
    s = 10.0 ** decimals
    return np.rint(np.asarray(v, dtype=np.float32).astype(np.float64) * s) / s


def compute_alpha(x, z, ry):
    """datasets/provider_sample.py:389-394 on float32 arrays (float32 results, as for the reference's float32 rows)."""
    beta = np.arctan2(z, x)
    return -np.sign(beta) * np.pi / 2 + beta + ry


def _parse_tokens(path, width, what):
    with open(path) as f:
        tok = f.read().split()
    n = len(tok) // width
    if n * width != len(tok):
        raise ValueError("%s: %d fields are not a whole number of %d-field %s lines" % (path, len(tok), width, what))
    return [tok[i * width:(i + 1) * width] for i in range(n)]


def parse_label_file(path):
    """A label_2 file -> (n, 15) float64 records (loadGroundtruth, :180-204)."""
    rows = []
    for t in _parse_tokens(path, 15, "label"):
        rows.append([type_code(t[0]), float(t[1]), int(t[2])] + [float(x) for x in t[3:15]])
    return np.asarray(rows, dtype=np.float64).reshape(-1, GT_COLS)


def parse_result_file(path):
    """A result file -> (n, 14) float64 records (loadDetections, :133-178; the two fields after the type are
    unused)."""
    rows = []
    for t in _parse_tokens(path, 16, "result"):
        rows.append([type_code(t[0])] + [float(x) for x in t[3:16]])
    return np.asarray(rows, dtype=np.float64).reshape(-1, DET_COLS)


def detection_records(dets, class_type):
    """Rows [x1,y1,x2,y2, tx,ty,tz, h,w,l, ry, score] (float32, as DetectionCollector.finalize() and the reference's
    test() return them) -> (n, 14) float64 records of the lines write_detection_results writes (:88-123)."""
    d = np.asarray(dets, dtype=np.float32).reshape(-1, 12)
    out = np.empty((d.shape[0], DET_COLS), dtype=np.float64)
    out[:, 0] = type_code(class_type)
    out[:, 1] = quantize(compute_alpha(d[:, 4], d[:, 6], d[:, 10]), 4)
    out[:, 2:6] = quantize(d[:, 0:4], 4)                          # x1, y1, x2, y2
    out[:, 6:9] = quantize(d[:, 7:10], 4)                         # h, w, l
    out[:, 9:12] = quantize(d[:, 4:7], 4)                         # tx, ty, tz
    out[:, 12] = quantize(d[:, 10], 4)                            # ry
    out[:, 13] = quantize(d[:, 11], 6)                            # score, '%f'
    return out


class KittiGroundTruth:
    """label_2 records of a list of images, parsed once and kept on the device."""

    def __init__(self, image_ids, records, device=None):
        self.image_ids = [int(i) for i in image_ids]
        if len(set(self.image_ids)) != len(self.image_ids):
            raise ValueError("image_ids must be unique")
        if len(records) != len(self.image_ids):
            raise ValueError("one record array per image is required")
        self.device = cuda_device(device, "KittiGroundTruth")
        self.records = [np.asarray(r, dtype=np.float64).reshape(-1, GT_COLS) for r in records]
        self.index = {idx: i for i, idx in enumerate(self.image_ids)}
        self.host_offsets = csr_offsets([len(r) for r in self.records])
        flat = np.concatenate(self.records) if self.records else np.zeros((0, GT_COLS))
        self.gt = torch.from_numpy(np.ascontiguousarray(flat)).to(self.device)
        self.offsets = torch.from_numpy(self.host_offsets).to(self.device)

    @classmethod
    def from_label_dir(cls, label_dir, image_ids, device=None):
        ids = [int(i) for i in image_ids]
        return cls(ids, [parse_label_file(os.path.join(label_dir, "%06d.txt" % i)) for i in ids], device)

    @property
    def num_gt(self):
        return int(self.host_offsets[-1])


class KittiEvalResult:
    """precision[metric][class] (3, 41) float64 (rows easy, moderate, hard); aos[class] (3, 41) (image metric, when
    no alpha is -10); ap[metric][class] (3,) and ap_aos[class] (3,): the printed AP; n_thresholds, n_gt likewise.
    Only evaluated classes are present."""

    def __init__(self, raw):
        self.raw = raw
        self.compute_aos = bool(raw.compute_aos)
        prec = np.ctypeslib.as_array(raw.precision).reshape(3, 3, 3, PTS)
        aos = np.ctypeslib.as_array(raw.aos).reshape(3, 3, PTS)
        ap = np.ctypeslib.as_array(raw.ap).reshape(3, 3, 3)
        ap_aos = np.ctypeslib.as_array(raw.ap_aos).reshape(3, 3)
        nthr = np.ctypeslib.as_array(raw.n_thresholds).reshape(3, 3, 3)
        ngt = np.ctypeslib.as_array(raw.n_gt).reshape(3, 3, 3)
        ev = np.ctypeslib.as_array(raw.evaluated).reshape(3, 3)
        self.evaluated = {METRICS[m]: tuple(CLASS_NAMES[c] for c in range(3) if ev[m, c]) for m in range(3)}
        self.precision, self.ap, self.n_thresholds, self.n_gt = ({m: {} for m in METRICS} for _ in range(4))
        self.aos, self.ap_aos = {}, {}
        for m in range(3):
            for c in range(3):
                if not ev[m, c]:
                    continue
                name = CLASS_NAMES[c]
                self.precision[METRICS[m]][name] = prec[m, c].copy()
                self.ap[METRICS[m]][name] = ap[m, c].astype(np.float64)
                self.n_thresholds[METRICS[m]][name] = nthr[m, c].copy()
                self.n_gt[METRICS[m]][name] = ngt[m, c].copy()
                if m == 0 and self.compute_aos:
                    self.aos[name] = aos[c].copy()
                    self.ap_aos[name] = ap_aos[c].astype(np.float64)

    def lines(self):
        """The evaluator's printed AP lines, in its order (image + orientation per class, then ground, then 3-D)."""
        out = []
        for m, suffix in zip(METRICS, ("_detection", "_detection_ground", "_detection_3d")):
            for name in CLASS_NAMES:
                if name in self.ap[m]:
                    out.append("%s AP: %f %f %f" % ((name + suffix,) + tuple(self.ap[m][name])))
                    if m == "image" and name in self.aos:
                        out.append("%s AP: %f %f %f" % ((name + "_orientation",) + tuple(self.ap_aos[name])))
        return out


class KittiEvaluator:
    def __init__(self, gt: KittiGroundTruth):
        self.gt = gt
        self.device = gt.device

    def evaluate(self, det_results, stream=None, timer=None):
        """{idx: {class_type: (n, 12)}} -> KittiEvalResult over every image of the ground truth (`stream`, `timer`:
        as for ``evaluate_records``)."""
        per_image = [[] for _ in self.gt.image_ids]
        for idx, by_class in det_results.items():
            i = self.gt.index.get(int(idx))
            if i is None:
                raise KeyError("detections for image %s, which is not in the ground truth's image_ids" % idx)
            for class_type, dets in by_class.items():
                if len(dets):
                    per_image[i].append(detection_records(dets, class_type))
        return self.evaluate_records([np.concatenate(p) if p else np.zeros((0, DET_COLS)) for p in per_image], stream,
                                     timer)

    def evaluate_dir(self, result_dir):
        """Result files result_dir/data/<index>.txt (the evaluator's layout) -> KittiEvalResult over the images that
        have a file, like the evaluator; every such image must be in the ground truth."""
        data = os.path.join(result_dir, "data")
        recs = {}
        for name in os.listdir(data):
            if len(name) < 10:
                continue
            idx = int(name[-10:].split(".")[0])
            if idx not in self.gt.index:
                raise KeyError("result file %s has no ground truth" % name)
            recs[idx] = parse_result_file(os.path.join(data, name))
        ids = sorted(recs)
        sub = KittiGroundTruth(ids, [self.gt.records[self.gt.index[i]] for i in ids], self.device)
        return KittiEvaluator(sub).evaluate_records([recs[i] for i in ids])

    def gather_plan(self, collected):
        """The host half of ``evaluate_collected``, from segment metadata only -> (seg_dst, seg_code, det_offsets):
        per segment of the collector the first record it owns in the per-image CSR of ``evaluate`` (-1: not written)
        and its type code, and the (num_images + 1) offsets of that CSR.  Within an image its classes keep the dict
        order, then the row order.  An image of the dict that is not in the ground truth raises KeyError."""
        S = collected.num_segments
        order = collected.order
        gt_index = np.empty(len(order), dtype=np.int64)
        seen = {}
        for j, s in enumerate(order.tolist()):
            idx = collected.segments[s][0]
            i = seen.get(idx)
            if i is None:
                i = self.gt.index.get(int(idx))
                if i is None:
                    raise KeyError("detections for image %s, which is not in the ground truth's image_ids" % idx)
                seen[idx] = i
            gt_index[j] = i
        kept = collected.host_keep_count[order].astype(np.int64)
        by_image = order[np.argsort(gt_index, kind="stable")]        # images in ground-truth order, dict order within
        seg_dst = np.full(S, -1, dtype=np.int32)
        counts = collected.host_keep_count[by_image].astype(np.int64)
        seg_dst[by_image] = (np.cumsum(counts) - counts).astype(np.int32)
        seg_code = np.array([type_code(ct) for _, ct in collected.segments], dtype=np.int32)
        det_off = csr_offsets(np.bincount(gt_index, weights=kept, minlength=len(self.gt.image_ids)).astype(np.int64))
        return seg_dst, seg_code, det_off

    def evaluate_collected(self, collected, stream=None, timer=None):
        """DetectionCollector.finalize_device()'s CollectedDetections -> the KittiEvalResult ``evaluate`` gives for
        its dict, without the rows crossing to the host: the records are written on the device
        (``fcn_det_kitti_records``) into the per-image order ``evaluate`` builds, the gather plan coming from the
        segment keys alone.  Alpha uses the correctly rounded float32 atan2 (numpy's float32 arctan2 can differ from it
        in the last bit, by at most one '%.4f' step after the rounding); every other field is identical."""
        dev = self.device
        seg_dst, seg_code, det_off = self.gather_plan(collected)
        num_det = int(det_off[-1])
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            if collected.stream.cuda_stream != stream.cuda_stream:
                stream.wait_stream(collected.stream)
            buf, (p_dst, p_code, p_off) = upload([seg_dst, seg_code, det_off], dev)
            det = torch.empty((max(num_det, 1), DET_COLS), dtype=torch.float64, device=dev)
            if timer is not None:
                timer("feed_start")
            a = collected.feed_args(seg_dst, seg_code, num_det, (p_dst, p_code))
            a.records = det.data_ptr()
            _lib.call("fcn_det_kitti_records", C.byref(a), stream.cuda_stream)
            return self._launch(det.data_ptr(), p_off, det_off, stream, timer)

    def evaluate_records(self, det_records, stream=None, timer=None):
        """One (nd_i, 14) float64 record array per image of the ground truth, in its order -> KittiEvalResult.
        `timer(name)` (optional) is called before the first device call ("start") and after each of the three is
        enqueued (benchmarks)."""
        if len(det_records) != len(self.gt.image_ids):
            raise ValueError("one detection record array per ground-truth image is required")
        dev = self.device
        det_records = [np.asarray(r, dtype=np.float64).reshape(-1, DET_COLS) for r in det_records]
        host_det_off = csr_offsets([len(r) for r in det_records])
        flat = np.concatenate(det_records) if det_records else np.zeros((0, DET_COLS))
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            det = torch.from_numpy(np.ascontiguousarray(flat)).to(dev, non_blocking=False)
            det_off = torch.from_numpy(host_det_off).to(dev)
            return self._launch(det.data_ptr(), det_off.data_ptr(), host_det_off, stream, timer)

    def _launch(self, det, det_off, host_det_off, stream, timer):
        """The three evaluator entries on `stream` (current, on the evaluator's device) over device records `det` with
        device offsets `det_off` and their host copy -> KittiEvalResult after the one read back."""
        dev = self.device
        a = _lib.KittiEvalArgs()
        a.num_images, a.num_gt, a.num_det = len(self.gt.image_ids), self.gt.num_gt, int(host_det_off[-1])
        a.gt, a.det = self.gt.gt.data_ptr(), det
        a.gt_offsets, a.det_offsets = self.gt.offsets.data_ptr(), det_off
        a.host_gt_offsets = self.gt.host_offsets.ctypes.data
        a.host_det_offsets = host_det_off.ctypes.data
        ws, nbytes = workspace("fcn_kitti_eval_workspace_bytes", dev, C.byref(a))
        res = torch.zeros(C.sizeof(_lib.KittiEvalResult), dtype=torch.uint8, device=dev)   # + tail padding
        a.workspace, a.workspace_bytes, a.result = ws.data_ptr(), nbytes, res.data_ptr()
        if timer is not None:
            timer("start")
        for name in ("fcn_kitti_eval_overlaps", "fcn_kitti_eval_thresholds", "fcn_kitti_eval_statistics"):
            _lib.call(name, C.byref(a), stream.cuda_stream)
            if timer is not None:
                timer(name)
        raw = _lib.KittiEvalResult.from_buffer_copy(res.cpu().numpy().tobytes())   # the one read back
        return KittiEvalResult(raw)
