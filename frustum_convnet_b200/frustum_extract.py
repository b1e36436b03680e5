"""KITTI frustums from raw LiDAR scans and 2-D detections on the device: extract_frustum_data_rgb_detection of the
reference (kitti/prepare_data.py:462-568) without its pickle, for a whole set of frames in one call.

    ids, types, probs, boxes = read_rgb_detections(open("rgb_detection_val.txt"))
    fr = FrustumExtractor(type_whitelist=("Car",)).extract(scans, calibs, image_hw, ids, types, probs, boxes)
    fb.set_frustums_device(fr.points, fr.offsets, fr.frustum_angle, fr.box2d, fr.P)   # FrustumBatchBuilder
    col = DetectionCollector(fr.id_list, fr.type_list, fr.box2d_list)

``scans[data_idx]`` is an (n, 4) float32 scan (x, y, z, intensity in Velodyne coordinates; numpy or a CUDA tensor),
``calibs[data_idx]`` a dict with 'P2', 'Tr_velo_to_cam' and 'R0_rect' (the calib file's float64 values) and
``image_hw[data_idx]`` the image's (height, width).  The result holds what the reference pickles: device tensors
``points`` (M, 4) float32, ``offsets`` (K + 1) int32, ``frustum_angle`` (K) float64, ``box2d`` (K, 4) float64 and
``P`` (K, 12) float64; host ``counts`` and the lists ``id_list``, ``type_list``, ``box2d_list``, ``prob_list``,
``calib_list`` in the pickle's order.  Points, counts, boxes and order are bit-identical to the reference's wherever
its matmul rounding and the kernel's fixed elementwise order (csrc/frustum_extract.cu) agree on a point's side of an
edge; the angle comes from CUDA's atan2 (within 2 ulp of glibc's).  The thresholds (5 px, 1 point) and the 2 m
distance are the reference's.  One host sync per call, to learn K and M.  No CPU fallback: CPU tensors raise."""
from __future__ import annotations

import ctypes as C
import os
import pickle

import numpy as np
import torch

from . import _lib
from ._host import csr_offsets, cuda_device, on_device, upload, workspace

DET_ID2STR = {1: "Pedestrian", 2: "Car", 3: "Cyclist"}


def read_rgb_detections(lines):
    """Lines 'path type prob xmin ymin xmax ymax' (read_det_file, prepare_data.py:428-446) ->
    (id_list, type_list, prob_list, box2d_list); the type is a detector id of DET_ID2STR or a type name."""
    id_list, type_list, prob_list, box2d_list = [], [], [], []
    for line in lines:
        t = line.rstrip().split(" ")
        id_list.append(int(os.path.basename(t[0]).rstrip(".png")))
        try:
            cls_type = DET_ID2STR[int(t[1])]
        except ValueError:
            if t[1] not in DET_ID2STR.values():
                raise ValueError("unknown detection type %r" % t[1])
            cls_type = t[1]
        type_list.append(cls_type)
        prob_list.append(float(t[2]))
        box2d_list.append(np.array([float(t[i]) for i in range(3, 7)]))
    return id_list, type_list, prob_list, box2d_list


class Frustums:
    """One extraction: K kept detections and their M points (see the module docstring)."""

    def __init__(self, points, offsets, frustum_angle, box2d, P, counts, id_list, type_list, box2d_list, prob_list,
                 calib_list, det_index):
        self.points, self.offsets, self.frustum_angle, self.box2d, self.P = points, offsets, frustum_angle, box2d, P
        self.counts = counts
        self.id_list, self.type_list, self.box2d_list = id_list, type_list, box2d_list
        self.prob_list, self.calib_list = prob_list, calib_list
        self.det_index = det_index          # (K,) host int64: the detection line of each kept frustum

    def __len__(self):
        return len(self.id_list)


def _frame_record(calib, hw):
    f = _lib.FrustumFrame()
    for name, key, n in (("P", "P2", 12), ("V2C", "Tr_velo_to_cam", 12), ("R0", "R0_rect", 9)):
        v = np.asarray(calib[key], dtype=np.float64).reshape(-1)
        if v.size != n:
            raise ValueError("calib %s must hold %d values, got %d" % (key, n, v.size))
        getattr(f, name)[:] = v.tolist()
    h, w = (int(x) for x in hw)
    if h <= 0 or w <= 0:
        raise ValueError("image size must be positive, got %r" % (hw,))
    f.height, f.width = h, w
    return f


def _scan(scan, dev, who, cols=4):
    if isinstance(scan, torch.Tensor):
        if not on_device(scan, dev):
            raise RuntimeError("%s: scans must be numpy arrays or CUDA tensors on %s" % (who, dev))
        if scan.dtype != torch.float32 or scan.dim() != 2 or scan.shape[1] != cols:
            raise ValueError("a scan must be an (n, %d) float32 array" % cols)
        return scan
    a = np.asarray(scan)
    if a.dtype != np.float32 or a.ndim != 2 or a.shape[1] != cols:
        raise ValueError("a scan must be an (n, %d) float32 array" % cols)
    return a


def scan_table(scans, calibs, image_hw, frame_ids, dev, who):
    """The frames of every extractor (this module's, refine_extract's and gt_extract's), in frame_ids order, checked
    on the host -> (their scans, the fcn_frustum_frame array, the host scan offsets)."""
    sc = [_scan(scans[k], dev, who) for k in frame_ids]
    frames = (_lib.FrustumFrame * len(frame_ids))(*[_frame_record(calibs[k], image_hw[k]) for k in frame_ids])
    return sc, frames, csr_offsets([s.shape[0] for s in sc])


def upload_scans(sc, dev):
    """scan_table's scans -> one (N, 4) float32 tensor on dev (N, 6 for SUN-RGBD clouds)."""
    if all(isinstance(s, np.ndarray) for s in sc):
        return torch.from_numpy(np.concatenate(sc)).to(dev)
    return torch.cat([s if isinstance(s, torch.Tensor) else torch.from_numpy(s).to(dev) for s in sc]).contiguous()


def frame_order(frames):
    """Frame ids (one per job, several jobs a frame) -> (the distinct ids in first-appearance order, {id: position})."""
    pos = {}
    for k in frames:
        pos.setdefault(k, len(pos))
    return list(pos), pos


def read_counts(summary, n, who, bad_what):
    """The count pass's summary, read back once (the extraction's one host sync): int64 info (K kept records, M
    points, bad references, -), then int32 words, the first n of them each record's point count (-1: dropped).
    -> (K, M, the int32 words, the kept records)."""
    back = summary.cpu().numpy()
    K, M, bad = int(back[0]), int(back[1]), int(back[2])
    if bad:
        raise RuntimeError("%s: %d %s" % (who, bad, bad_what))
    if M >= 2 ** 31:
        raise RuntimeError("%s: %d frustum points do not fit int32 offsets" % (who, M))
    words = back[4:].view(np.int32)
    kept = np.flatnonzero(words[:n] >= 0)
    assert len(kept) == K and int(words[kept].sum()) == M
    return K, M, words, kept


def run_extract(family, a, sc, so, n, word_fields, outputs, dev, stream, timer, bad_what, extra_words=0, count=None,
                cols=4):
    """The two device calls of an extractor family ('frustum_extract', 'refine_extract', 'gt_extract',
    'sunrgbd_extract') on the current stream `stream`.  a: the family's args struct with its counts and inputs filled;
    sc, so: the frames' scans and host scan offsets.  Uploads the scans, queries the workspace, runs the count into one
    summary (info, then the per-job int32 words: n of them for each args field of word_fields, then extra_words more),
    reads it back once (read_counts, naming bad_what), then runs fcn_<family>_write into new points (M, cols),
    offsets and the tensors of outputs(K, M, words), a dict {args field: tensor or None}.
    count(the summary's int32 words on the device) enqueues the count-side device work and marks its own timer
    names; the default runs fcn_<family>_count and marks "count".  A family whose count is several calls, or which
    builds its jobs on the device (writing per-job words into the extra words), passes its own.  `timer(name)`
    (optional) also marks "start" before the count, "write_start" and "write".
    -> (the int32 words, the kept jobs, {args field: output tensor}, points and offsets included)."""
    mark = timer if timer is not None else (lambda name: None)
    if count is None:
        def count(words):
            _lib.call("fcn_%s_count" % family, C.byref(a), stream.cuda_stream)
            mark("count")
    scan_dev = upload_scans(sc, dev)            # like so and the caller's upload, alive until the write is enqueued
    a.scans = scan_dev.data_ptr() if int(so[-1]) > 0 else None
    a.host_scan_offsets = so.ctypes.data
    ws, nbytes = workspace("fcn_%s_workspace_bytes" % family, dev, C.byref(a))
    summary = torch.empty(4 + (len(word_fields) * n + extra_words + 1) // 2, dtype=torch.int64, device=dev)
    words_dev = summary[4:].view(torch.int32)
    a.workspace, a.workspace_bytes, a.info = ws.data_ptr(), nbytes, summary.data_ptr()
    for k, field in enumerate(word_fields):
        setattr(a, field, words_dev.data_ptr() + 4 * n * k)
    mark("start")
    count(words_dev)
    K, M, words, kept = read_counts(summary, n, "fcn_" + family, bad_what)
    out = {"points": torch.empty((M, cols), dtype=torch.float32, device=dev),
           "offsets": torch.empty(K + 1, dtype=torch.int32, device=dev), **outputs(K, M, words)}
    a.num_kept, a.num_out_points = K, M
    for field, t in out.items():
        setattr(a, field, None if t is None else t.data_ptr())
    mark("write_start")
    _lib.call("fcn_%s_write" % family, C.byref(a), stream.cuda_stream)
    mark("write")
    return words, kept, out


def empty_outputs(dev, cols, labels):
    """The device tensors of an extraction without frustums: points (0, cols) float32, offsets [0] int32 and label
    (0,) uint8, or None without labels."""
    return (torch.zeros((0, cols), dtype=torch.float32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev),
            torch.zeros(0, dtype=torch.uint8, device=dev) if labels else None)


class LabelledFrustums:
    """The result of refine_extract's, gt_extract's and sunrgbd_extract's extractors: K kept frustums and their M
    points.  Device: points (M, 4) float32 ((M, 6) for SUN-RGBD), offsets (K + 1) int32, label (M) uint8 (None without labels), written on the extraction's
    stream.  Host: counts (K,) and job_index (K,) (the job, i.e. box and augmentation, of each frustum), int64, and
    the provider's lists.  input_list(), label_list() and TrainBatchBuilder.from_frustums make the current stream wait
    for that stream first (wait()); other readers of the tensors on another stream call wait() themselves."""

    has_labels = True
    pickle_names = ()          # the lists in the order the reference pickles them

    def __init__(self, points, offsets, label, counts, job_index, stream):
        self.points, self.offsets, self.label = points, offsets, label
        self.stream = stream
        self.counts = counts
        self.job_index = job_index

    def __len__(self):
        return len(self.id_list)

    def _split(self, t):
        off = np.concatenate([[0], np.cumsum(self.counts)])
        return [t[off[k]:off[k + 1]] for k in range(len(self))]

    def wait(self):
        """Make the current stream of the tensors' device wait for the extraction's stream."""
        if self.stream is not None:
            torch.cuda.current_stream(self.points.device).wait_stream(self.stream)

    def input_list(self):
        """The per-frustum (n, 4) (SUN-RGBD: (n, 6)) float32 point arrays, copied to the host."""
        self.wait()
        return self._split(self.points.cpu().numpy())

    def label_list(self):
        """The per-frustum (n,) float64 labels (1 inside the ground-truth box), copied to the host."""
        if not self.has_labels:
            raise ValueError("frustums from detections have no labels")
        self.wait()
        return self._split(self.label.cpu().numpy().astype(np.float64))

    def to_pickle(self, path):
        """The lists in the order the reference's function pickles them (readable by the reference's provider)."""
        values = {"input_list": self.input_list()}
        if self.has_labels:
            values["label_list"] = self.label_list()
        with open(path, "wb") as fp:
            for n in self.pickle_names:
                pickle.dump(values[n] if n in values else getattr(self, n), fp, -1)


class FrustumExtractor:
    def __init__(self, type_whitelist=("Car",), device=None):
        self.type_whitelist = tuple(type_whitelist)
        self.device = cuda_device(device, "FrustumExtractor")

    def extract(self, scans, calibs, image_hw, id_list, type_list, prob_list, box2d_list, stream=None, timer=None):
        """-> Frustums.  Runs on `stream` (default: the current stream of the extractor's device).  `timer(name)`
        (optional, benchmarks) is called around the two device calls: "start", "count", "write_start", "write"."""
        n = len(id_list)
        if len(type_list) != n or len(prob_list) != n or len(box2d_list) != n:
            raise ValueError("id_list, type_list, prob_list and box2d_list must have the same length")
        lines = [i for i in range(n) if type_list[i] in self.type_whitelist]
        frame_ids, frame_of = frame_order(id_list[i] for i in lines)
        boxes = np.array([np.asarray(box2d_list[i], dtype=np.float64).reshape(4) for i in lines],
                         dtype=np.float64).reshape(-1, 4)
        if not np.isfinite(boxes).all():
            raise ValueError("2-D boxes must be finite")
        det_frame = np.array([frame_of[id_list[i]] for i in lines], dtype=np.int32)
        dev = self.device
        sc, frames, so = scan_table(scans, calibs, image_hw, frame_ids, dev, "FrustumExtractor")
        F, D, N = len(frame_ids), len(lines), int(so[-1])
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            if F == 0 or D == 0:
                return self._result(*empty_outputs(dev, 4, False)[:2], *self._empty(dev), np.zeros(0, np.int64), [],
                                    id_list, type_list, prob_list, box2d_list, calibs, image_hw)
            inp, ptrs = upload([bytes(frames), boxes, so, det_frame], dev)
            a = _lib.FrustumExtractArgs()
            a.num_frames, a.num_points, a.num_dets = F, N, D
            a.frames, a.boxes, a.scan_offsets, a.det_frame = ptrs
            det_points, kept, out = run_extract(
                "frustum_extract", a, sc, so, D, ("det_points",),
                lambda K, M, words: {"frustum_angle": torch.empty(K, dtype=torch.float64, device=dev),
                                     "box2d": torch.empty((K, 4), dtype=torch.float64, device=dev),
                                     "P": torch.empty((K, 12), dtype=torch.float64, device=dev),
                                     "det_index": torch.empty(K, dtype=torch.int32, device=dev)},
                dev, stream, timer, "detections reference no frame")
        line_idx = np.asarray(lines, dtype=np.int64)[kept]
        return self._result(out["points"], out["offsets"], out["frustum_angle"], out["box2d"], out["P"],
                            det_points[kept].astype(np.int64), line_idx, id_list, type_list, prob_list, box2d_list,
                            calibs, image_hw)

    @staticmethod
    def _empty(dev):
        return (torch.zeros(0, dtype=torch.float64, device=dev), torch.zeros((0, 4), dtype=torch.float64, device=dev),
                torch.zeros((0, 12), dtype=torch.float64, device=dev))

    @staticmethod
    def _result(points, offsets, angle, box2d, P, counts, line_idx, id_list, type_list, prob_list, box2d_list, calibs,
                image_hw):
        ids = [id_list[i] for i in line_idx]
        boxes = []
        for i, k in zip(line_idx, ids):              # the reference's own clip (prepare_data.py:522-524), on the host
            h, w = image_hw[k]
            b = np.asarray(box2d_list[i], dtype=np.float64).reshape(4).copy()
            b[[0, 2]] = np.clip(b[[0, 2]], 0, w - 1)
            b[[1, 3]] = np.clip(b[[1, 3]], 0, h - 1)
            boxes.append(b)
        return Frustums(points, offsets, angle, box2d, P, counts, ids, [type_list[i] for i in line_idx], boxes,
                        [prob_list[i] for i in line_idx], [calibs[k] for k in ids], np.asarray(line_idx, np.int64))
