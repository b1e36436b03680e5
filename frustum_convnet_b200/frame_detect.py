"""KITTI first-stage detection of single frames in fixed capacities: scans and 2-D detections to 3-D boxes with no
host round trip, so a serving loop can capture one call in a CUDA graph and replay it on every new frame.

    fd = FrameDetector(model, type_whitelist=("Car",), frames=1, points=131072, dets=8)
    inp = fd.inputs()                                  # fixed device buffers, filled in place for every frame
    fd.stage(inp, [(scan, calib, (h, w), [("Car", 0.9, box2d), ...])])
    out = fd.detect(*inp)                              # no host sync
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                          # after one eager call
        out = fd.detect(*inp)
    fd.stage(inp, next_frames); g.replay()
    results = out.to_dict()                            # {frame: {class: float32 (n, 12)}}, the one host read

The chain is the offline one (FrustumExtractor, FrustumBatchBuilder, the model, DetectionCollector) in capacity
mode (C ABI section (21)): the extraction runs over all F * D detection slots, the resampling indices are drawn on
the device (csrc/resample.cu), the forward runs on the model's plan for (F * D, N, T) and the collector's finalize
reads its sizes on the device.  The batch holds the kept frustums in (frame, detection) order, then dummy entries
that add no row.  The resampling does not reproduce numpy's stream: each draw is a Philox4x32-10 value keyed on
(seed, call counter, detection slot, point), so a replay draws fresh indices and a given key repeats bit for bit.
Given the same `choice` (FrameDetections.choice), rows, offsets and keep counts equal the offline chain's bit for bit.

Capacities that a call exceeds set bits of FrameDetections.status (a device int32; FCN_FRAME_* of the C header):
  1  a frame had more than P scan points (its first P were used)
  2  a frame had more than D detections (its first D were used)
  4  a frame's kept frustums had more than P_out points (those past the budget were dropped)
  8  the frustums gave more candidate rows than R (the rows past R were not recorded; the result is incomplete)
  16 a detection had a class outside Car / Pedestrian / Cyclist or a non-finite box (it was not extracted)
No store lands outside a buffer whatever the inputs."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._host import check_tensors, cuda_device, workspace
from .input_builder import FrustumBatchBuilder
from .refine_extract import REFINE_STRIDES
from .train_inputs import SUNRGBD_CLASSES

CLASSES = ("Car", "Pedestrian", "Cyclist")          # det_class values 0, 1, 2 (the model's one-hot index)
_FRAME_BYTES = C.sizeof(_lib.FrustumFrame)         # 33 float64 (P2, Tr_velo_to_cam, R0_rect), then height, width


class FrameDetections:
    """The result of one FrameDetector.detect, on the device (overwritten by the next call).

    rows (R, 12) float32: kept row k of segment s at seg_offsets[s] + k, k < keep_count[s], in the row layout of
    DetectionCollector.finalize_device(); segment s = C f + r (C = len(classes)) is frame f's r-th class by first
    appearance among its kept detections, seg_class[f, r] that class (-1: none).  status: the capacity bits.  choice
    (F * D, N) int32: the resampling indices of the batch entries (kept frustums first).  classes: the names of the
    class indices, dataset: "KITTI" or "SUNRGBD".  cap_choice (SunrgbdFrameDetector only, else None): the 2048-point
    cap draws of the detection slots."""

    cap_choice = None

    def __init__(self, rows, seg_offsets, keep_count, seg_class, status, choice, valid, classes=CLASSES,
                 dataset="KITTI"):
        self.rows, self.seg_offsets, self.keep_count = rows, seg_offsets, keep_count
        self.seg_class, self.status, self.choice, self.valid = seg_class, status, choice, valid
        self.classes, self.dataset = tuple(classes), dataset

    def to_dict(self, frame_ids=None):
        """-> {frame id: {class name: float32 (n, 12)}} in the reference's dict order (frames with a kept frustum, each
        class by first appearance), what DetectionCollector.finalize() gives; frame_ids names frame f (default f).
        Reads the result back once (a host sync)."""
        F, C = self.seg_class.shape
        S = C * F
        meta = torch.cat([self.seg_offsets, self.keep_count, self.seg_class.reshape(-1), self.status]).cpu().numpy()
        n = int(meta[S])
        rows = self.rows[:max(n, 1)].cpu().numpy()
        off, kc, cls = meta[:S + 1], meta[S + 1:2 * S + 1], meta[2 * S + 1:3 * S + 1]
        res = {}
        for s in range(S):
            if cls[s] < 0:
                continue
            f = s // C
            key = f if frame_ids is None else frame_ids[f]
            res.setdefault(key, {})[self.classes[cls[s]]] = rows[off[s]:off[s] + kc[s]].copy()
        return res

    def collected(self, frame_ids=None):
        """-> detect.CollectedDetections over the same device rows, segments (frame id, class name) in to_dict's order
        (frame_ids names frame f, default f), so a frame call's rows go to KittiEvaluator.evaluate_collected (or
        SunrgbdEvaluator.evaluate_collected) and RefineFrustumExtractor.from_collected without leaving the device.
        Reads the offsets, keep counts and classes back once (a host sync); a segment of no class is named ""."""
        from .detect import CollectedDetections
        F, C = self.seg_class.shape
        S = C * F
        meta = torch.cat([self.seg_offsets, self.keep_count, self.seg_class.reshape(-1)]).cpu().numpy()
        off, kc, cls = meta[:S + 1], meta[S + 1:2 * S + 1], meta[2 * S + 1:3 * S + 1]
        ids = list(range(F)) if frame_ids is None else list(frame_ids)
        segments = [(ids[s // C], self.classes[cls[s]] if cls[s] >= 0 else "") for s in range(S)]
        order = [s for s in range(S) if cls[s] >= 0]
        return CollectedDetections(self.dataset, self.rows, self.seg_offsets, self.keep_count, off, kc, segments, order,
                                   torch.cuda.current_stream(self.rows.device))

    def status_bits(self):
        """The status word, read back (a host sync)."""
        return int(self.status.item())


class _CapacityStage:
    """What the detection and refinement stages share: the model's eval forward on its plan for (B, N, T) and the
    collector's candidates and capacity finalize over B entries, of which only the valid ones add rows.  A subclass
    calls _settings, sets model, device, F, B, N, T (sections per scale), R and the entry tables seg, valid, box2d32
    and seg_class, then calls _init_collector.  Each frame has one segment per class of `classes`."""

    classes, dataset = CLASSES, _lib.DET_KITTI

    def _settings(self, who, classes, type_whitelist, method, thresh, top_k, seed):
        """class_mask of type_whitelist (names of `classes`; any other raises ValueError before a device is
        touched), the collector's method, thresh and top_k, and the resampling seed."""
        bad = [t for t in type_whitelist if t not in classes]
        if bad:
            raise ValueError("%s: unknown types %s (classes: %s)" % (who, bad, classes))
        self.class_mask = sum(1 << classes.index(t) for t in set(type_whitelist))
        self.method = 0 if method == "nms" else 1
        self.thresh, self.top_k, self.seed = float(thresh), int(top_k), int(seed) & (2 ** 64 - 1)

    def _init_resample(self, index):
        """The fcn_resample_choice arguments: N indices into each of the B entries' points (offsets) written to
        choice, drawn under the key (seed, call, index[k], point)."""
        r = _lib.ResampleArgs()
        r.B, r.N, r.seed = self.B, self.N, self.seed
        r.offsets, r.det_index, r.call, r.choice = (self.offsets.data_ptr(), index.data_ptr(), self.call.data_ptr(),
                                                    self.choice.data_ptr())
        self._ra = r

    def _init_fixed_batch(self, kind, num_classes, max_depth, keys):
        """The fixed-width batch of fcn_build_train_inputs_fixed over points3, offsets64 and frustum_records (the
        extraction's records, zeroed here): the tensors `keys` of point_cloud, rot_angle, ref_center, rgb_prob and
        one_hot, then center_ref1.. of widths T at the strides."""
        dev, B, N, S = self.device, self.B, self.N, len(self.strides)
        e = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
        self.offsets64 = torch.empty(B + 1, dtype=torch.int64, device=dev)
        self.frustum_records = torch.zeros((B, C.sizeof(_lib.TrainFrustum)), dtype=torch.uint8, device=dev)
        self.index = torch.arange(B, dtype=torch.int32, device=dev)
        shapes = {"point_cloud": (B, 3, N), "rot_angle": (B,), "ref_center": (B, 3), "rgb_prob": (B,),
                  "one_hot": (B, num_classes)}
        self.batch = {k: e(*shapes[k]) for k in keys}
        for s, w in enumerate(self.T):
            self.batch["center_ref%d" % (s + 1)] = e(B, 3, w)
        t = _lib.TrainInputArgs()
        t.kind, t.labels, t.rtc, t.extra_feat = kind, 0, 1, 0
        t.B, t.N, t.num_scales, t.num_classes, t.num_frustums = B, N, S, num_classes, B
        for s in range(S):
            t.stride[s] = self.strides[s]
            t.centers[s] = self.batch["center_ref%d" % (s + 1)].data_ptr()
        t.max_depth = max_depth
        t.points, t.point_offsets, t.frustums = (self.points3.data_ptr(), self.offsets64.data_ptr(),
                                                 self.frustum_records.data_ptr())
        t.index, t.choice = self.index.data_ptr(), self.choice.data_ptr()
        for k in keys:
            setattr(t, k, self.batch[k].data_ptr())
        self._ta = t
        self._widths = (C.c_int32 * S)(*self.T)

    def _init_collector(self, per_frame):
        """The collector's buffers; per_frame: the most entries of one frame (a segment holds rows of at most that
        many entries)."""
        dev, F, R, T2 = self.device, self.F, self.R, self.T[1]
        S = len(self.classes) * F
        e = lambda *shape, dtype=torch.int32: torch.empty(shape, dtype=dtype, device=dev)
        self.counter = torch.zeros(1, dtype=torch.int32, device=dev)
        self.records = e(R, 12)
        self.rows = e(R, 12, dtype=torch.float32)
        self.seg_offsets, self.keep_count = e(S + 1), e(S)
        self.info = e(4, dtype=torch.int64)
        m = min(R, per_frame * T2)                      # the most rows one (frame, class) segment can hold
        self.mask = e(max(R * ((m + 31) // 32), 1))
        with torch.cuda.device(dev):
            self._det_ws, det_bytes = workspace("fcn_det_workspace_bytes", dev, R, S)
        fa = _lib.DetFinalizeArgs()
        fa.num_segments, fa.num_frustums, fa.capacity, fa.method, fa.dataset = S, self.B, R, self.method, self.dataset
        fa.top_k, fa.thresh = self.top_k, self.thresh
        fa.counter, fa.records, fa.box2d = self.counter.data_ptr(), self.records.data_ptr(), self.box2d32.data_ptr()
        fa.workspace, fa.workspace_bytes, fa.info = self._det_ws.data_ptr(), det_bytes, self.info.data_ptr()
        fa.seg_offsets, fa.keep_count, fa.rows = (self.seg_offsets.data_ptr(), self.keep_count.data_ptr(),
                                                  self.rows.data_ptr())
        fa.mask, fa.mask_words = self.mask.data_ptr(), self.mask.numel()
        self._fa = fa
        self._plan = None
        self._keep = None

    def _forward(self, data):
        """The model's eval forward on its plan for (B, N, T), launched on the current stream (no graph of its own,
        so an enclosing capture records the kernels)."""
        pc = data["point_cloud"]
        centers = [data["center_ref%d" % (s + 1)] for s in range(len(self.T))]
        oh = data.get("one_hot") if self.model.num_vec > 0 else None
        first = self._plan is None
        if first:
            self._plan = self.model.engine().plan(self.B, self.N, self.T)
        return self._plan.run(pc, centers, oh, use_graph=False, copy_out=False, trusted=not first)

    def _collect(self, out, rot_angle, rgb_prob, ref_center, st):
        """Candidates of the valid entries, then the capacity finalize (box2d32 filled by the caller)."""
        cls_probs, center, heading, size, _, size_probs = out
        ts = [t.contiguous() for t in (cls_probs, center, heading, size, size_probs)]
        a = _lib.DetCandidateArgs()
        a.B, a.T2, a.NS, a.dataset, a.method = self.B, self.T[1], int(ts[4].shape[-1]), self.dataset, self.method
        a.first, a.num_frustums, a.capacity = 0, self.B, self.R
        a.cls_probs, a.center, a.heading, a.size, a.size_probs = (t.data_ptr() for t in ts)
        a.rot_angle, a.rgb_prob = rot_angle.data_ptr(), rgb_prob.data_ptr()
        a.ref_center = None if ref_center is None else ref_center.data_ptr()
        a.seg_of_frustum, a.counter, a.records = self.seg.data_ptr(), self.counter.data_ptr(), self.records.data_ptr()
        _lib.call("fcn_det_candidates_valid", C.byref(a), self.valid.data_ptr(), st)
        _lib.call("fcn_det_finalize_capacity", C.byref(self._fa), self.status.data_ptr(), st)
        self._keep = ts

    def _result(self):
        return FrameDetections(self.rows, self.seg_offsets, self.keep_count, self.seg_class, self.status,
                               self.choice, self.valid, self.classes,
                               "SUNRGBD" if self.dataset == _lib.DET_SUNRGBD else "KITTI")


class FrameDetector(_CapacityStage):
    def __init__(self, model, type_whitelist=("Car",), method="nms", thresh=0.1, top_k=300, seed=0, frames=1,
                 points=131072, dets=8, rows=None, frustum_points=None, strides=None, max_depth=None, npoints=None,
                 device=None):
        """model: an eval-mode det_base.PointNetDet.  frames F, points P, dets D: the capacities of one call;
        rows R (default F * D * T2, every position of every entry) and frustum_points P_out (default P) those of
        the collector and of each frame's frustum points.  strides, max_depth, npoints: the input cfg (default: the
        current cfg's DATA.STRIDE, MAX_DEPTH, NUM_SAMPLES).  method / thresh / top_k: the collector's."""
        from .config import get_cfg
        cfg = get_cfg()
        self._settings("FrameDetector", CLASSES, type_whitelist, method, thresh, top_k, seed)
        self.model = model
        self.device = cuda_device(device, "FrameDetector")
        self.F, self.P, self.D = int(frames), int(points), int(dets)
        self.B = self.F * self.D
        self.fb = FrustumBatchBuilder(cfg.DATA.STRIDE if strides is None else strides,
                                      cfg.DATA.MAX_DEPTH if max_depth is None else max_depth,
                                      cfg.DATA.NUM_SAMPLES if npoints is None else npoints, device=self.device)
        self.N, self.T = self.fb.N, list(self.fb.T)
        self.T2 = self.T[1]
        self.R = int(rows) if rows is not None else self.B * self.T2
        self.P_out = int(frustum_points) if frustum_points is not None else self.P
        if min(self.F, self.P, self.D, self.R, self.P_out) < 1:
            raise ValueError("FrameDetector: every capacity must be >= 1")
        dev, B, F = self.device, self.B, self.F
        e = lambda *shape, dtype=torch.int32: torch.empty(shape, dtype=dtype, device=dev)
        f64 = torch.float64
        self._frames = torch.zeros((F, _FRAME_BYTES), dtype=torch.uint8, device=dev)
        self.points4 = e(F * self.P_out + B, 4, dtype=torch.float32)
        self.points3 = e(F * self.P_out + B, 3, dtype=torch.float32)
        self.offsets, self.angle, self.box2d, self.Pm = e(B + 1), e(B, dtype=f64), e(B, 4, dtype=f64), \
            e(B, 12, dtype=f64)
        self.det_index, self.valid, self.cls_index, self.seg = e(B), e(B), e(B), e(B)
        self.seg_class, self.rgb_prob = e(F, 3), e(B, dtype=torch.float32)
        self.box2d32 = e(B, 4, dtype=torch.float32)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self.call = torch.zeros(1, dtype=torch.int64, device=dev)
        self.choice = e(B, self.N)
        self.fb.set_frustums_device(self.points3, self.offsets, self.angle, self.box2d, self.Pm, self.cls_index)

        a = _lib.FrameExtractArgs()
        a.num_frames, a.scan_capacity, a.det_capacity, a.out_capacity = F, self.P, self.D, self.P_out
        a.class_mask = self.class_mask
        a.frames = self._frames.data_ptr()
        a.status, a.points, a.offsets = self.status.data_ptr(), self.points4.data_ptr(), self.offsets.data_ptr()
        a.frustum_angle, a.box2d, a.P = self.angle.data_ptr(), self.box2d.data_ptr(), self.Pm.data_ptr()
        a.det_index, a.valid, a.cls_index = self.det_index.data_ptr(), self.valid.data_ptr(), self.cls_index.data_ptr()
        a.seg, a.seg_class, a.rgb_prob = self.seg.data_ptr(), self.seg_class.data_ptr(), self.rgb_prob.data_ptr()
        with torch.cuda.device(dev):
            self._ws, a.workspace_bytes = workspace("fcn_frame_extract_workspace_bytes", dev, C.byref(a))
            a.workspace = self._ws.data_ptr()
        self._xa = a
        self._init_resample(self.det_index)
        self._init_collector(self.D)

    # ------------------------------------------------------------------ inputs
    def inputs(self):
        """Fresh device input buffers of this detector's capacities, zero counts: (scans, calibs, image_hw, dets) with
        scans = (points (F, P, 4) float32, counts (F,) int32), calibs (F, 33) float64 (P2, Tr_velo_to_cam, R0_rect
        row-major), image_hw (F, 2) int32 and dets = (boxes (F, D, 4) float64, classes (F, D) int32 (index in
        CLASSES), probs (F, D) float32, counts (F,) int32)."""
        dev, F, P, D = self.device, self.F, self.P, self.D
        z = lambda *shape, dtype=torch.int32: torch.zeros(shape, dtype=dtype, device=dev)
        return ((z(F, P, 4, dtype=torch.float32), z(F)), z(F, 33, dtype=torch.float64), z(F, 2),
                (z(F, D, 4, dtype=torch.float64), z(F, D), z(F, D, dtype=torch.float32), z(F)))

    def stage(self, inputs, frames):
        """Copy host frames into `inputs` (this detector's inputs()): frames is a list of at most F tuples
        (scan (n, 4) float32, calib dict with 'P2', 'Tr_velo_to_cam', 'R0_rect', (height, width),
        [(type name, prob, box2d), ...]); frames past the list get zero counts.  Rows past a capacity are copied up
        to it and the counts are kept, so detect reports the overflow."""
        (pts, npts), calib, hw, (boxes, cls, prob, ndet) = inputs
        F, P, D = self.F, self.P, self.D
        if len(frames) > F:
            raise ValueError("FrameDetector.stage: %d frames for a capacity of %d" % (len(frames), F))
        h_pts = np.zeros((F, P, 4), np.float32)
        h_calib, h_hw = np.zeros((F, 33)), np.zeros((F, 2), np.int32)
        h_box, h_cls = np.zeros((F, D, 4)), np.zeros((F, D), np.int32)
        h_prob, h_n, h_nd = np.zeros((F, D), np.float32), np.zeros(F, np.int32), np.zeros(F, np.int32)
        for f, (scan, cal, size, det) in enumerate(frames):
            scan = np.asarray(scan, np.float32).reshape(-1, 4)
            h_n[f], h_nd[f] = len(scan), len(det)
            h_pts[f, :min(len(scan), P)] = scan[:P]
            h_calib[f] = np.concatenate([np.asarray(cal[k], np.float64).reshape(-1)
                                         for k in ("P2", "Tr_velo_to_cam", "R0_rect")])
            h_hw[f] = size
            for j, (t, p, b) in enumerate(det[:D]):
                h_cls[f, j] = CLASSES.index(t) if t in CLASSES else -1
                h_prob[f, j], h_box[f, j] = p, np.asarray(b, np.float64).reshape(4)
        for dst, src in ((pts, h_pts), (npts, h_n), (calib, h_calib), (hw, h_hw), (boxes, h_box), (cls, h_cls),
                         (prob, h_prob), (ndet, h_nd)):
            dst.copy_(torch.from_numpy(src), non_blocking=False)

    # ------------------------------------------------------------------ the call
    @torch.no_grad()
    def detect(self, scans, calibs, image_hw, dets):
        """One call on the current stream: no host sync, no allocation after the first call, so it can be captured
        with torch.cuda.graph once it has run eagerly (the capture keeps the input tensors' addresses).
        -> FrameDetections (this detector's buffers, overwritten by the next call)."""
        (pts, npts), (boxes, cls, prob, ndet) = scans, dets
        F, P, D = self.F, self.P, self.D
        check_tensors("FrameDetector.detect", self.device, (
            ("scan points", pts, (F, P, 4), torch.float32), ("scan counts", npts, (F,), torch.int32),
            ("calibs", calibs, (F, 33), torch.float64), ("image_hw", image_hw, (F, 2), torch.int32),
            ("boxes", boxes, (F, D, 4), torch.float64), ("classes", cls, (F, D), torch.int32),
            ("probs", prob, (F, D), torch.float32), ("det counts", ndet, (F,), torch.int32)))
        dev = self.device
        with torch.cuda.device(dev):
            st = torch.cuda.current_stream(dev).cuda_stream
            self.status.zero_()
            self.counter.zero_()
            self._frames[:, :264].view(torch.float64).copy_(calibs)
            self._frames[:, 264:272].view(torch.int32).copy_(image_hw)
            a = self._xa
            a.scans, a.scan_counts, a.boxes = pts.data_ptr(), npts.data_ptr(), boxes.data_ptr()
            a.det_class, a.det_prob, a.det_counts = cls.data_ptr(), prob.data_ptr(), ndet.data_ptr()
            _lib.call("fcn_frame_extract", C.byref(a), st)
            self.points3.copy_(self.points4[:, :3])
            _lib.call("fcn_resample_choice", C.byref(self._ra), st)
            self.call.add_(1)
            data = self.fb.build(self.choice)
            out = self._forward(data)
            self.box2d32.copy_(self.box2d)
            self._collect(out, data["rot_angle"], self.rgb_prob, None, st)
        return self._result()


def section_widths(max_width, strides):
    """W[s] = len(np.arange(-w / 2, w / 2, s)) for w = max_width: the sections of a refinement record whose enlarged
    box is max_width wide, at every stride s."""
    w = float(max_width)
    return [len(np.arange(-w / 2, w / 2, float(s))) for s in strides]


class FrameRefiner(_CapacityStage):
    """The second stage of the KITTI cascade for a FrameDetector's results, in the same fixed capacities: refinement
    frustums cut around the first stage's kept rows, device resampling, the refinement forward and the collector, with
    no host sync (C ABI section (22)).  A detect and a refine call can be captured in one CUDA graph.

        fd = FrameDetector(det_model, ("Car",), frames=F, points=P, dets=D)
        fr = FrameRefiner(fd, refine_model, type_whitelist=("Car",), jobs=2 * D, max_width=4.8, seed=1)
        inp = fd.inputs(); fd.stage(inp, frames)
        out = fr.refine(inp, fd.detect(*inp))          # FrameDetections of the second stage

    The chain is the offline one (RefineFrustumExtractor.from_collected, TrainBatchBuilder.from_frustums(..,
    "refine", labels=False), the model, DetectionCollector) in capacity mode.  Frame f's jobs are the first stage's
    kept rows of its whitelisted classes in to_dict order (slot f * J + j); the batch holds the kept frustums in slot
    order, then dummy entries that add no row.  Batch width: the offline path pads each refinement batch to its own
    widest item, so a refined box depends on its batch-mates; here every batch is padded to the fixed W[s], and the
    result equals the offline path's for a batch padded to W.  Resampling draws are keyed on (seed, this refiner's
    call counter, slot, point); the counter has bit 63 set, so no draw coincides with a first-stage draw.

    Status: the result's status word is the first stage's with the second stage's FCN_FRAME_* bits OR-ed in:
      4  a frame's refinement frustums had more than P2_out points (those past the budget were dropped)
      8  the refinement gave more candidate rows than R2 (the result is incomplete)
      16 a first-stage row had a non-finite box or a non-positive extent (it was not refined)
      32 a frame had more than J whitelisted first-stage rows (the first J were refined)
      64 a refinement frustum needed more sections than W[s] (it was dropped)"""

    def __init__(self, detector, model, type_whitelist=("Car",), jobs=None, max_width=4.8, sections=None,
                 frustum_points=None, rows=None, strides=REFINE_STRIDES, npoints=512, method="nms", thresh=0.1,
                 top_k=300, seed=0):
        """detector: the FrameDetector whose results this refines (its frames F, scan capacity P and device).
        model: an eval-mode refinement det_base.PointNetDet (cfgs/refine_car.yaml: strides REFINE_STRIDES, npoints
        512; the global cfg is the first stage's and is not read).  jobs J (default 2 * D) and max_width (4.8 m, the
        widest enlarged box kept) are guesses, not measured distributions: size them to the first stage's rows per
        frame and the boxes it produces.  sections=(W[0], ...) overrides the widths max_width gives; they must halve
        from scale to scale like the model's section pyramid.
        frustum_points P2_out (default P) and rows R2 (default B2 * W[1], B2 = F * J): the capacities of each frame's
        frustum points and of the collector.  method / thresh / top_k: the collector's."""
        self._settings("FrameRefiner", CLASSES, type_whitelist, method, thresh, top_k, seed)
        self.fd, self.model, self.device = detector, model, detector.device
        self.F, self.P = detector.F, detector.P
        self.J = int(jobs) if jobs is not None else 2 * detector.D
        self.strides = [float(s) for s in strides]
        self.N = int(npoints)
        self.T = [int(w) for w in (sections if sections is not None else section_widths(max_width, self.strides))]
        if len(self.T) != len(self.strides):
            raise ValueError("FrameRefiner: %d sections for %d strides" % (len(self.T), len(self.strides)))
        if any(self.T[s] != (self.T[s - 1] + 1) // 2 for s in range(1, len(self.T))):
            raise ValueError("FrameRefiner: sections %s must halve from scale to scale (W[s] = (W[s-1] + 1) // 2), as "
                             "the model's section pyramid does" % (self.T,))
        self.B = self.F * self.J
        self.P_out = int(frustum_points) if frustum_points is not None else self.P
        self.R = int(rows) if rows is not None else self.B * self.T[1]
        if min([self.J, self.P_out, self.R, self.N] + self.T) < 1:
            raise ValueError("FrameRefiner: every capacity must be >= 1")
        dev, B, F, S = self.device, self.B, self.F, len(self.strides)
        e = lambda *shape, dtype=torch.int32: torch.empty(shape, dtype=dtype, device=dev)
        self.points4 = e(F * self.P_out + B, 4, dtype=torch.float32)
        self.points3 = e(F * self.P_out + B, 3, dtype=torch.float32)
        self.offsets = e(B + 1)
        self.job_index, self.valid, self.cls_index, self.seg = e(B), e(B), e(B), e(B)
        self.seg_class, self.box2d32 = e(F, 3), e(B, 4, dtype=torch.float32)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self.call = torch.full((1,), -2 ** 63, dtype=torch.int64, device=dev)     # bit 63 set: stage 2's draws
        self.choice = e(B, self.N)
        self._init_fixed_batch(_lib.TRAIN_REFINE, len(CLASSES), 1.0,
                               ("point_cloud", "rot_angle", "ref_center", "rgb_prob", "one_hot"))

        a = _lib.FrameRefineArgs()
        a.num_frames, a.scan_capacity, a.job_capacity, a.out_capacity = F, self.P, self.J, self.P_out
        a.num_rows, a.num_scales, a.class_mask = detector.R, S, self.class_mask
        for s in range(S):
            a.stride[s], a.widths[s] = self.strides[s], self.T[s]
        a.frames = detector._frames.data_ptr()              # the calibs and image sizes its detect() packed
        a.rows, a.seg_offsets = detector.rows.data_ptr(), detector.seg_offsets.data_ptr()
        a.keep_count, a.seg_class = detector.keep_count.data_ptr(), detector.seg_class.data_ptr()
        a.status, a.points, a.offsets = self.status.data_ptr(), self.points4.data_ptr(), self.offsets.data_ptr()
        a.job_index, a.valid, a.cls_index = self.job_index.data_ptr(), self.valid.data_ptr(), self.cls_index.data_ptr()
        a.seg, a.seg_class_out = self.seg.data_ptr(), self.seg_class.data_ptr()
        a.records, a.box2d = self.frustum_records.data_ptr(), self.box2d32.data_ptr()
        with torch.cuda.device(dev):
            self._ws, a.workspace_bytes = workspace("fcn_frame_refine_extract_workspace_bytes", dev, C.byref(a))
            a.workspace = self._ws.data_ptr()
        self._xa = a
        self._init_resample(self.job_index)
        self._init_collector(self.J)

    @torch.no_grad()
    def refine(self, inputs, first):
        """inputs: the detector's inputs() the first stage read; first: its detect() result of this call (the
        calibrations and image sizes are those that detect() packed from the same inputs).  One call
        on the current stream: no host sync, no allocation after the first call, so detect and refine can be captured
        in one CUDA graph once both have run eagerly.  -> FrameDetections of the second stage (this refiner's
        buffers, overwritten by the next call); choice holds the stage-2 resampling indices."""
        (pts, npts), _, _, _ = inputs
        if first.rows.data_ptr() != self.fd.rows.data_ptr():
            raise ValueError("FrameRefiner.refine: `first` is not the result of this refiner's detector")
        F, P = self.F, self.P
        check_tensors("FrameRefiner.refine", self.device, (("scan points", pts, (F, P, 4), torch.float32),
                                                           ("scan counts", npts, (F,), torch.int32)))
        dev = self.device
        with torch.cuda.device(dev):
            st = torch.cuda.current_stream(dev).cuda_stream
            self.status.copy_(first.status)
            self.counter.zero_()
            a = self._xa
            a.scans, a.scan_counts = pts.data_ptr(), npts.data_ptr()
            _lib.call("fcn_frame_refine_extract", C.byref(a), st)
            self.points3.copy_(self.points4[:, :3])
            self.offsets64.copy_(self.offsets)
            _lib.call("fcn_resample_choice", C.byref(self._ra), st)
            self.call.add_(1)
            _lib.call("fcn_build_train_inputs_fixed", C.byref(self._ta), self._widths, st)
            data = dict(self.batch)
            out = self._forward(data)
            self._collect(out, self.batch["rot_angle"], self.batch["rgb_prob"], self.batch["ref_center"], st)
        return self._result()


_SUNRGBD_FRAME_BYTES = C.sizeof(_lib.SunrgbdFrame)  # Rtilt, then K: 18 float64


class SunrgbdFrameDetector(_CapacityStage):
    """SUN-RGBD detection of single RGB-D frames in fixed capacities: depth clouds and 2-D detections to 3-D boxes with
    no host round trip, so a serving loop can capture one call in a CUDA graph (C ABI section (23)).

        fd = SunrgbdFrameDetector(model, frames=1, points=393216, dets=16)
        inp = fd.inputs()
        fd.stage(inp, [(cloud, {"Rtilt": Rtilt, "K": K}, [("chair", 0.9, box2d), ...])])
        out = fd.detect(*inp)                              # no host sync; capturable after one eager call
        results = out.to_dict()                            # {frame: {class: float32 (n, 12)}}

    The chain is the offline one (SunrgbdFrustumExtractor.from_rgb_detections, TrainBatchBuilder.from_frustums(..,
    "sunrgbd", labels=False), the model, DetectionCollector(dataset="SUNRGBD")) in capacity mode: the extraction runs
    over all F * D detection slots, the reference's 2048-point cap (np.random.choice(n, 2048, replace=False)) and the
    provider's resampling are drawn on the device, the forward runs on the model's plan for (F * D, N, T) and the
    collector's finalize reads its sizes there.  The batch holds the kept frustums in (frame, detection) order, then
    dummy entries that add no row.  Both draws are Philox4x32-10 values keyed on (seed, call counter, slot, point), as
    FrameDetector's: the cap's counter has bit 62 set, so the two never coincide.  Given the same cap rows
    (FrameDetections.cap_choice) and `choice`, frustums, rows, offsets and keep counts equal the offline chain's bit
    for bit.

    Capacities that a call exceeds set bits of FrameDetections.status (FCN_FRAME_* of the C header):
      1  a frame had more than P cloud points (its first P were used)
      2  a frame had more than D detections (its first D were used)
      4  a frame's kept frustums had more than P_out points (those past the budget were dropped)
      8  the frustums gave more candidate rows than R (the result is incomplete)
      16 a detection had a class index outside SUNRGBD_CLASSES or a non-finite box (it was not extracted)
    No store lands outside a buffer whatever the inputs.

    From depth images instead of clouds (C ABI section (24), the reference's read_3d_points on the device):
        inp = fd.inputs_depth(530, 730)
        fd.stage_depth(inp, [(depth_uint16, rgb_uint8_or_None, {"Rtilt": Rtilt, "K": K}, dets)])
        out = fd.detect_depth(*inp)                        # the conversion, then detect()'s chain
    which adds status bit 128 for an image larger than the buffers."""

    dataset = _lib.DET_SUNRGBD

    def __init__(self, model, type_whitelist=SUNRGBD_CLASSES, method="top", thresh=0.1, top_k=300, seed=0, frames=1,
                 points=393216, dets=16, rows=None, frustum_points=None, strides=None, max_depth=None, npoints=None,
                 device=None):
        """model: an eval-mode det_base_sunrgbd.PointNetDet.  type_whitelist: classes of SUNRGBD_CLASSES to detect
        frames F, points P (< 2^24), dets D (<= 64): the capacities of one call; rows R (default
        F * D * T2) and frustum_points P_out (default D * 2048, which no frame can exceed) those of the collector and
        of each frame's frustum points.  strides, max_depth, npoints: the input cfg (default: the current cfg's
        DATA.STRIDE, MAX_DEPTH, NUM_SAMPLES; cfgs/det_sample_sunrgbd.yaml).  method / thresh / top_k: the
        collector's (the reference's SUN-RGBD cfg tests with "top")."""
        from .config import get_cfg
        cfg = get_cfg()
        self.classes = SUNRGBD_CLASSES
        self._settings("SunrgbdFrameDetector", SUNRGBD_CLASSES, type_whitelist, method, thresh, top_k, seed)
        self.model = model
        self.device = cuda_device(device, "SunrgbdFrameDetector")
        self.F, self.P, self.D = int(frames), int(points), int(dets)
        self.B = self.F * self.D
        self.strides = [float(s) for s in (cfg.DATA.STRIDE if strides is None else strides)]
        self.max_depth = float(cfg.DATA.MAX_DEPTH if max_depth is None else max_depth)
        self.N = int(cfg.DATA.NUM_SAMPLES if npoints is None else npoints)
        if len(self.strides) != 5:
            raise ValueError("SunrgbdFrameDetector: the SUN-RGBD model takes 5 strides, got %d" % len(self.strides))
        self.T = [len(np.arange(0, self.max_depth, s)) for s in self.strides]
        self.T2 = self.T[1]
        self.R = int(rows) if rows is not None else self.B * self.T2
        self.P_out = int(frustum_points) if frustum_points is not None else self.D * _lib.SUNRGBD_MAX_POINTS
        if min(self.F, self.P, self.D, self.R, self.P_out, self.N) < 1:
            raise ValueError("SunrgbdFrameDetector: every capacity must be >= 1")
        if self.D > _lib.SUNRGBD_FRAME_MAX_DETS or self.P >= 2 ** 24 or self.N > _lib.SUNRGBD_MAX_POINTS:
            raise ValueError("SunrgbdFrameDetector: need dets <= %d, points < 2^24 and npoints <= 2048"
                             % _lib.SUNRGBD_FRAME_MAX_DETS)
        dev, B, F, S, NC = self.device, self.B, self.F, len(self.strides), len(SUNRGBD_CLASSES)
        e = lambda *shape, dtype=torch.int32: torch.empty(shape, dtype=dtype, device=dev)
        f32 = torch.float32
        self._frames = torch.zeros((F, _SUNRGBD_FRAME_BYTES), dtype=torch.uint8, device=dev)
        self.points = e(F * self.P_out + B, 6, dtype=f32)
        self.points3 = e(F * self.P_out + B, 3, dtype=f32)
        self.offsets = e(B + 1)
        self.det_index, self.valid, self.cls_index, self.seg = e(B), e(B), e(B), e(B)
        self.seg_class, self.rgb_prob, self.box2d32 = e(F, NC), e(B, dtype=f32), e(B, 4, dtype=f32)
        self.cap_choice = e(B, _lib.SUNRGBD_MAX_POINTS)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self.call = torch.zeros(1, dtype=torch.int64, device=dev)
        self.cap_call = torch.full((1,), 2 ** 62, dtype=torch.int64, device=dev)    # bit 62 set: the cap's draws
        self.choice = e(B, self.N)
        self._init_fixed_batch(_lib.TRAIN_SUNRGBD, NC, self.max_depth, ("point_cloud", "rot_angle", "rgb_prob",
                                                                        "one_hot"))

        a = _lib.SunrgbdFrameExtractArgs()
        a.num_frames, a.point_capacity, a.det_capacity, a.out_capacity = F, self.P, self.D, self.P_out
        a.class_mask, a.num_scales, a.seed, a.max_depth = self.class_mask, S, self.seed, self.max_depth
        for s in range(S):
            a.stride[s] = self.strides[s]
        a.frames, a.call, a.status = self._frames.data_ptr(), self.cap_call.data_ptr(), self.status.data_ptr()
        a.points, a.xyz, a.offsets = self.points.data_ptr(), self.points3.data_ptr(), self.offsets.data_ptr()
        a.det_index, a.valid, a.cls_index = self.det_index.data_ptr(), self.valid.data_ptr(), self.cls_index.data_ptr()
        a.seg, a.seg_class, a.rgb_prob = self.seg.data_ptr(), self.seg_class.data_ptr(), self.rgb_prob.data_ptr()
        a.box2d, a.cap_choice = self.box2d32.data_ptr(), self.cap_choice.data_ptr()
        a.records = self.frustum_records.data_ptr()
        with torch.cuda.device(dev):
            self._ws, a.workspace_bytes = workspace("fcn_sunrgbd_frame_extract_workspace_bytes", dev, C.byref(a))
            a.workspace = self._ws.data_ptr()
        self._xa = a
        self._init_resample(self.det_index)
        self._init_collector(self.D)
        self._depth = None              # detect_depth's conversion and its (F, P, 6) clouds, made on its first call

    # ------------------------------------------------------------------ inputs
    def inputs(self):
        """Fresh device input buffers of this detector's capacities, zero counts: (clouds, calibs, dets) with
        clouds = (points (F, P, 6) float32, counts (F,) int32), calibs (F, 18) float64 (Rtilt, then K, row-major)
        and dets = (boxes (F, D, 4) float64, classes (F, D) int32 (index in SUNRGBD_CLASSES), probs (F, D) float32,
        counts (F,) int32)."""
        dev, F, P, D = self.device, self.F, self.P, self.D
        z = lambda *shape, dtype=torch.int32: torch.zeros(shape, dtype=dtype, device=dev)
        return ((z(F, P, 6, dtype=torch.float32), z(F)), z(F, 18, dtype=torch.float64),
                (z(F, D, 4, dtype=torch.float64), z(F, D), z(F, D, dtype=torch.float32), z(F)))

    def stage(self, inputs, frames):
        """Copy host frames into `inputs` (this detector's inputs()): frames is a list of at most F tuples
        (cloud (n, 6) float32, calib dict with 'Rtilt' and 'K' (3 x 3), [(type name, prob, box2d), ...]); frames past
        the list get zero counts.  Detections whose type is not one of SUNRGBD_CLASSES are skipped, as the offline
        extractor's whitelist skips them (a 19-class 2-D detector is the usual input).  Rows past a capacity are
        copied up to it and the counts are kept, so detect reports the overflow."""
        (pts, npts), calib, dets = inputs
        F, P = self.F, self.P
        if len(frames) > F:
            raise ValueError("SunrgbdFrameDetector.stage: %d frames for a capacity of %d" % (len(frames), F))
        h_pts, h_n = np.zeros((F, P, 6), np.float32), np.zeros(F, np.int32)
        for f, (cloud, _, _) in enumerate(frames):
            cloud = np.asarray(cloud, np.float32).reshape(-1, 6)
            h_n[f] = len(cloud)
            h_pts[f, :min(len(cloud), P)] = cloud[:P]
        for dst, src in ((pts, h_pts), (npts, h_n)):
            dst.copy_(torch.from_numpy(src), non_blocking=False)
        self._stage_calib_dets(calib, dets, [(cal, det) for _, cal, det in frames])

    def _stage_calib_dets(self, calib, dets, frames):
        """stage()'s calibrations and detections: frames is a list of (calib, [(type name, prob, box2d), ...])."""
        boxes, cls, prob, ndet = dets
        F, D = self.F, self.D
        h_calib = np.zeros((F, 18))
        h_box, h_cls = np.zeros((F, D, 4)), np.zeros((F, D), np.int32)
        h_prob, h_nd = np.zeros((F, D), np.float32), np.zeros(F, np.int32)
        for f, (cal, det) in enumerate(frames):
            h_calib[f] = np.concatenate([np.asarray(cal[k], np.float64).reshape(9) for k in ("Rtilt", "K")])
            det = [d for d in det if d[0] in self.classes]
            h_nd[f] = len(det)
            for j, (t, p, b) in enumerate(det[:D]):
                h_cls[f, j] = self.classes.index(t)
                h_prob[f, j], h_box[f, j] = p, np.asarray(b, np.float64).reshape(4)
        for dst, src in ((calib, h_calib), (boxes, h_box), (cls, h_cls), (prob, h_prob), (ndet, h_nd)):
            dst.copy_(torch.from_numpy(src), non_blocking=False)

    # ------------------------------------------------------------------ the call
    @torch.no_grad()
    def detect(self, clouds, calibs, dets):
        """One call on the current stream: no host sync, no allocation after the first call, so it can be captured
        with torch.cuda.graph once it has run eagerly (the capture keeps the input tensors' addresses).
        -> FrameDetections (this detector's buffers, overwritten by the next call), with cap_choice (F * D, 2048):
        the cap draw of every candidate slot with more than 2048 in-box points, in draw order."""
        (pts, npts), (boxes, cls, prob, ndet) = clouds, dets
        F, P, D = self.F, self.P, self.D
        check_tensors("SunrgbdFrameDetector.detect", self.device, (
            ("cloud points", pts, (F, P, 6), torch.float32), ("cloud counts", npts, (F,), torch.int32),
            ("calibs", calibs, (F, 18), torch.float64), ("boxes", boxes, (F, D, 4), torch.float64),
            ("classes", cls, (F, D), torch.int32), ("probs", prob, (F, D), torch.float32),
            ("det counts", ndet, (F,), torch.int32)))
        dev = self.device
        with torch.cuda.device(dev):
            self.status.zero_()
            return self._chain(clouds, calibs, dets)

    def _chain(self, clouds, calibs, dets):
        """The extraction, the resampling, the forward and the collector on the current stream, with the status as the
        caller left it."""
        (pts, npts), (boxes, cls, prob, ndet) = clouds, dets
        st = torch.cuda.current_stream(self.device).cuda_stream
        self.counter.zero_()
        self._frames.view(torch.float64).copy_(calibs)
        a = self._xa
        a.clouds, a.cloud_counts, a.boxes = pts.data_ptr(), npts.data_ptr(), boxes.data_ptr()
        a.det_class, a.det_prob, a.det_counts = cls.data_ptr(), prob.data_ptr(), ndet.data_ptr()
        _lib.call("fcn_sunrgbd_frame_extract", C.byref(a), st)
        self.cap_call.add_(1)
        self.offsets64.copy_(self.offsets)
        _lib.call("fcn_resample_choice", C.byref(self._ra), st)
        self.call.add_(1)
        _lib.call("fcn_build_train_inputs_fixed", C.byref(self._ta), self._widths, st)
        data = dict(self.batch)
        out = self._forward(data)
        self._collect(out, self.batch["rot_angle"], self.batch["rgb_prob"], None, st)
        res = self._result()
        res.cap_choice = self.cap_choice
        return res

    # ------------------------------------------------------------------ from depth images (C ABI section (24))
    def inputs_depth(self, height, width, rgb=True):
        """Fresh device input buffers for frames of at most height x width pixels, zero sizes and counts:
        (images, calibs, dets) with images = (depth (F, H, W) uint16, rgb (F, H, W, 3) uint8 or None (rgb=False),
        image_hw (F, 2) int32), and calibs and dets as inputs() makes them."""
        dev, F, D, H, W = self.device, self.F, self.D, int(height), int(width)
        if min(H, W) < 1:
            raise ValueError("SunrgbdFrameDetector.inputs_depth: height and width must be >= 1")
        z = lambda *shape, dtype=torch.int32: torch.zeros(shape, dtype=dtype, device=dev)
        depth = z(F, H, W, dtype=torch.int16).view(torch.uint16)
        images = (depth, z(F, H, W, 3, dtype=torch.uint8) if rgb else None, z(F, 2))
        return (images, z(F, 18, dtype=torch.float64),
                (z(F, D, 4, dtype=torch.float64), z(F, D), z(F, D, dtype=torch.float32), z(F)))

    def stage_depth(self, inputs, frames):
        """Copy host frames into `inputs` (this detector's inputs_depth()): frames is a list of at most F tuples
        (depth (h, w) uint16, rgb (h, w, 3) uint8 in RGB order or None, calib dict with 'Rtilt' and 'K' (3 x 3),
        [(type name, prob, box2d), ...]); frames past the list get zero sizes and counts.  An image larger than the
        buffers is copied as its top-left crop with its own size kept, so detect_depth reports it; a None rgb gives
        that frame colour 0 (the rgb buffer's zeros) and needs no rgb buffer.  Detections as stage() takes them."""
        (depth, rgb, hw), calib, dets = inputs
        F, (H, W) = self.F, depth.shape[1:]
        if len(frames) > F:
            raise ValueError("SunrgbdFrameDetector.stage_depth: %d frames for a capacity of %d" % (len(frames), F))
        h_depth, h_hw = np.zeros((F, H, W), np.uint16), np.zeros((F, 2), np.int32)
        h_rgb = np.zeros((F, H, W, 3), np.uint8)
        for f, (d, c, _, _) in enumerate(frames):
            d = np.asarray(d)
            if d.ndim != 2 or d.dtype != np.uint16:
                raise ValueError("SunrgbdFrameDetector.stage_depth: frame %d's depth must be (h, w) uint16" % f)
            h_hw[f] = d.shape
            h, w = min(d.shape[0], H), min(d.shape[1], W)
            h_depth[f, :h, :w] = d[:h, :w]
            if c is not None:
                if rgb is None:
                    raise ValueError("SunrgbdFrameDetector.stage_depth: an rgb image for inputs without rgb buffers")
                c = np.asarray(c, np.uint8)
                if c.shape != d.shape + (3,):
                    raise ValueError("SunrgbdFrameDetector.stage_depth: frame %d's rgb must be (h, w, 3)" % f)
                h_rgb[f, :h, :w] = c[:h, :w]
        self._stage_calib_dets(calib, dets, [(cal, det) for _, _, cal, det in frames])
        depth.view(torch.int16).copy_(torch.from_numpy(h_depth.view(np.int16)))
        hw.copy_(torch.from_numpy(h_hw))
        if rgb is not None:
            rgb.copy_(torch.from_numpy(h_rgb))

    @torch.no_grad()
    def detect_depth(self, images, calibs, dets):
        """detect() from depth images (inputs_depth()'s buffers): the status cleared, the frames converted into this
        detector's internal (F, P, 6) clouds (fcn_sunrgbd_depth_cloud), then detect()'s chain.  One call on the current
        stream with no host sync; it allocates on the first call for an image size only, so it can be captured with
        torch.cuda.graph after one eager call.  Status bits besides detect()'s:
          1   a frame had more than P valid pixels (its first P in row-major order were used)
          128 a frame's image_hw was larger than the buffers (their top-left crop was read)"""
        depth, rgb, hw = images
        (boxes, cls, prob, ndet) = dets
        F, D = self.F, self.D
        if depth.dim() != 3:
            raise ValueError("SunrgbdFrameDetector.detect_depth: depth must be (F, H, W)")
        H, W = depth.shape[1:]
        if self._depth is None or (self._depth.H, self._depth.W) != (H, W):
            from .sunrgbd_depth import DepthCloudStage
            dev = self.device
            self._depth = DepthCloudStage(F, H, W, self.P, dev)
            self._depth_clouds = (torch.empty((F, self.P, 6), dtype=torch.float32, device=dev),
                                  torch.empty(F, dtype=torch.int32, device=dev))
        self._depth.check("SunrgbdFrameDetector.detect_depth", depth, rgb, hw, calibs)
        check_tensors("SunrgbdFrameDetector.detect_depth", self.device, (
            ("boxes", boxes, (F, D, 4), torch.float64), ("classes", cls, (F, D), torch.int32),
            ("probs", prob, (F, D), torch.float32), ("det counts", ndet, (F,), torch.int32)))
        with torch.cuda.device(self.device):
            self.status.zero_()
            pts, npts = self._depth_clouds
            self._depth.run(depth, rgb, hw, calibs, pts, npts, self.status,
                            torch.cuda.current_stream(self.device).cuda_stream)
            return self._chain(self._depth_clouds, calibs, dets)


class FrameStore:
    """The kept rows of many calls of one frame stage (FrameDetector, FrameRefiner or SunrgbdFrameDetector) collected
    on the device (C ABI section (25)), so a whole split run through the stage's CUDA graph is scored or refined from
    one table: every append is one launch sequence with no host sync, captured in the same graph as the call.

        store = FrameStore(fd, rows=200000, segments=30000)
        with torch.cuda.graph(g):                          # after one eager detect
            out = fd.detect(*inp); store.append(out)
        store.reset()
        for frames, ids in split:                          # at most F frames a call
            fd.stage(inp, frames); store.stage_ids(ids); g.replay()
        res = KittiEvaluator(...).evaluate_collected(store.collected())

    A call's segments (frame slot, then class by first appearance, as FrameDetections.to_dict orders them) are those of
    slots with an id >= 0; they are appended with their rows copied bit for bit, zero-row segments included.  A call
    is stored whole or not at all: when its rows or segments do not fit, nothing of it is stored and the store's
    status gets FCN_STORE_ROWS (1) or FCN_STORE_SEGMENTS (2); earlier calls stay intact.  Each stored call's own
    status word (FCN_FRAME_*) is OR-ed into the store's frame status, so one read at the end tells whether any call
    of the split hit a frame capacity."""

    def __init__(self, stage, rows, segments):
        """stage: the frame stage whose results are appended (its frames F, classes, dataset, device and result
        buffers); rows, segments: the store's capacities."""
        self.stage, self.device = stage, stage.device
        self.F, self.classes = stage.F, tuple(stage.classes)
        self.dataset = "SUNRGBD" if stage.dataset == _lib.DET_SUNRGBD else "KITTI"
        self.row_capacity, self.segment_capacity = int(rows), int(segments)
        if min(self.row_capacity, self.segment_capacity) < 1 or max(self.row_capacity, self.segment_capacity) >= 2 ** 31:
            raise ValueError("FrameStore: rows and segments must lie in [1, 2^31)")
        dev, n = self.device, self.segment_capacity
        e = lambda *shape, dtype=torch.int32: torch.empty(shape, dtype=dtype, device=dev)
        self.rows = e(self.row_capacity, 12, dtype=torch.float32)
        self.image, self.seg_class, self.frame = e(n, dtype=torch.int64), e(n), e(n)
        self.seg_offsets, self.keep_count = torch.zeros(n + 1, dtype=torch.int32, device=dev), e(n)
        self.cursor = torch.zeros(C.sizeof(_lib.FrameStoreCursor) // 4, dtype=torch.int32, device=dev)
        self.ids = torch.full((self.F,), -1, dtype=torch.int64, device=dev)
        a = _lib.FrameStoreArgs()
        a.num_frames, a.num_classes, a.num_rows = self.F, len(self.classes), stage.R
        a.row_capacity, a.segment_capacity = self.row_capacity, n
        a.rows, a.seg_offsets, a.keep_count = stage.rows.data_ptr(), stage.seg_offsets.data_ptr(), \
            stage.keep_count.data_ptr()
        a.seg_class, a.status, a.ids = stage.seg_class.data_ptr(), stage.status.data_ptr(), self.ids.data_ptr()
        a.store_rows, a.store_image, a.store_class = self.rows.data_ptr(), self.image.data_ptr(), \
            self.seg_class.data_ptr()
        a.store_frame, a.store_offset, a.store_keep = self.frame.data_ptr(), self.seg_offsets.data_ptr(), \
            self.keep_count.data_ptr()
        a.cursor = self.cursor.data_ptr()
        with torch.cuda.device(dev):
            self._ws, a.workspace_bytes = workspace("fcn_frame_store_append_workspace_bytes", dev, C.byref(a))
            a.workspace = self._ws.data_ptr()
        self._a = a

    def stage_ids(self, ids):
        """Copy the image ids of the next call's frame slots into `ids`: at most F values, slots past them get -1 (a
        slot with a negative id contributes nothing)."""
        ids = list(ids)
        if len(ids) > self.F:
            raise ValueError("FrameStore.stage_ids: %d ids for %d frame slots" % (len(ids), self.F))
        h = np.full(self.F, -1, np.int64)
        h[:len(ids)] = ids
        self.ids.copy_(torch.from_numpy(h), non_blocking=False)

    def append(self, out):
        """Append `out`, the stage's result of this call, on the current stream: no host sync, no allocation, so it is
        captured in the same CUDA graph as the call."""
        if out.rows.data_ptr() != self.stage.rows.data_ptr():
            raise ValueError("FrameStore.append: `out` is not a result of this store's stage")
        with torch.cuda.device(self.device):
            _lib.call("fcn_frame_store_append", C.byref(self._a), torch.cuda.current_stream(self.device).cuda_stream)

    def reset(self):
        """Empty the store on the current stream (capturable): zeroes the cursor block, status words included."""
        with torch.cuda.device(self.device):
            self.cursor.zero_()

    def collected(self):
        """-> detect.CollectedDetections over the store's device rows, segments (image id, class name) in append
        order, for KittiEvaluator / SunrgbdEvaluator.evaluate_collected and RefineFrustumExtractor.from_collected.
        One host read, of the cursor block and the segment table; no row crosses to the host.  Raises RuntimeError
        when a call did not fit (a store status bit is set) and ValueError naming an image id that was appended from
        two frame slots."""
        from .detect import CollectedDetections
        n = self.segment_capacity
        with torch.cuda.device(self.device):
            meta = torch.cat([t.view(torch.uint8).reshape(-1) for t in (self.cursor, self.image, self.seg_class,
                                                                         self.frame, self.seg_offsets,
                                                                         self.keep_count)]).cpu().numpy()
        cur = meta[:self.cursor.numel() * 4].view(np.int32)
        pieces, at = [], len(cur) * 4
        for dt, k in ((np.int64, n), (np.int32, n), (np.int32, n), (np.int32, n + 1), (np.int32, n)):
            size = np.dtype(dt).itemsize * k
            pieces.append(meta[at:at + size].view(dt))
            at += size
        image, cls, frame, off, kc = pieces
        used, total, status = int(cur[0]), int(cur[1]), int(cur[3])
        if status:
            raise RuntimeError("FrameStore: store status %d: a call's %s did not fit and was not stored (capacities: "
                               "%d rows, %d segments)" % (status, " and ".join(
                                   w for b, w in ((_lib.STORE_ROWS, "rows"), (_lib.STORE_SEGMENTS, "segments"))
                                   if status & b), self.row_capacity, n))
        image, frame = image[:used], frame[:used]
        pairs = np.unique(np.stack([image, frame.astype(np.int64)], axis=1), axis=0)
        twice = pairs[1:, 0][pairs[1:, 0] == pairs[:-1, 0]]
        if len(twice):
            raise ValueError("FrameStore: image id %d was appended from two frame slots" % int(twice[0]))
        segments = [(int(i), self.classes[c]) for i, c in zip(image.tolist(), cls[:used].tolist())]
        return CollectedDetections(self.dataset, self.rows, self.seg_offsets, self.keep_count,
                                   np.append(off[:used], total), kc[:used], segments, np.arange(used),
                                   torch.cuda.current_stream(self.device))

    def to_dict(self):
        """-> {image id: {class name: float32 (n, 12)}}: collected().to_dict()."""
        return self.collected().to_dict()

    def status_bits(self):
        """-> (the store's FCN_STORE_* bits, the OR of the stored calls' FCN_FRAME_* words), read back (a host sync)."""
        cur = self.cursor.cpu().numpy()
        return int(cur[3]), int(cur[4])
