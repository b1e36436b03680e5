"""numpy restatement of fcn_sunrgbd_frame_extract (C ABI section (23), csrc/sunrgbd_frame.cu): the clamped frame
inputs and status bits, the extraction of each clamped frame by oracle/sunrgbd_extract with the cap draws injected from
tests/resample_ref.choice_row under the cap's key, each frame's P_out budget, the ten-class ranks, the B = F * D batch
entries with their dummy tail, and the fcn_train_frustum records (frustum_table of the kept frustums; the frustum
angle is sunrgbd_extract.frustum_angle)."""
from functools import partial

import numpy as np

from frame_ref import budget, class_ranks as _class_ranks
from frustum_convnet_b200 import _lib
from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES, frustum_table
from oracle import sunrgbd_extract as ox
from resample_ref import choice_row

SCAN_POINTS, DETS, OUT_POINTS, BAD_DET = 1, 2, 4, 16          # FCN_FRAME_* bits of the C header
CAP, MIN_POINTS, NC = 2048, 5, len(SUNRGBD_CLASSES)
class_ranks = partial(_class_ranks, num_classes=NC)          # KITTI's budget and ranks over ten classes


def synth_frames(seed, F, H=240, W=320, n_objects=6):
    """F seeded sunrgbd_scene_synth frames: [(cloud (n, 6) float32, calib, [(class index, prob, box2d), ...])], one
    detection per label box of the ten classes (jittered; the first cut to 30 x 30 px, so each frame has frustums on
    both sides of the 2048-point cap)."""
    from frustum_convnet_b200 import sunrgbd_extract as sx
    from oracle import sunrgbd_scene_synth as ss
    rng = np.random.default_rng(seed)
    out = []
    for f in range(F):
        cloud, cal, lines = ss.large_frame(seed * 10 + f, H, W, n_objects)
        dets = [(SUNRGBD_CLASSES.index(o.classname), float(np.float32(rng.uniform(0.1, 1.0))),
                 o.box2d + rng.uniform(-4, 4, 4))
                for o in (sx.SUNObject3d(ln) for ln in lines) if o.classname in SUNRGBD_CLASSES]
        c = (dets[0][2][:2] + dets[0][2][2:]) / 2
        dets[0] = (dets[0][0], dets[0][1], np.concatenate([c - 15, c + 15]))
        out.append((cloud, cal, dets))
    return out


def stage(frames, P, D, cloud_counts=None, det_counts=None):
    """Frames as synth_frames gives them -> the raw inputs of fcn_sunrgbd_frame_extract in capacities (P, D): (clouds,
    cloud_counts, calibs, boxes, det_class, det_prob, det_counts).  Rows past a capacity are cut; the counts default
    to the frames' own (a count may exceed its capacity or be negative)."""
    F = len(frames)
    clouds = np.zeros((F, P, 6), np.float32)
    boxes, det_class = np.zeros((F, D, 4)), np.zeros((F, D), np.int32)
    det_prob = np.zeros((F, D), np.float32)
    for f, (cloud, _, dets) in enumerate(frames):
        clouds[f, :min(len(cloud), P)] = cloud[:P]
        for j, (c, p, b) in enumerate(dets[:D]):
            det_class[f, j], det_prob[f, j], boxes[f, j] = c, p, b
    cc = np.array([len(x[0]) for x in frames] if cloud_counts is None else cloud_counts, np.int32)
    dc = np.array([len(x[2]) for x in frames] if det_counts is None else det_counts, np.int32)
    return clouds, cc, [x[1] for x in frames], boxes, det_class, det_prob, dc


class _Rows:
    """An rng whose choice(n, 2048, replace=False) returns the given (n, row) draws in order."""

    def __init__(self, rows):
        self.rows = list(rows)

    def choice(self, n, size, replace=True):
        want_n, row = self.rows.pop(0)
        assert (int(n), size, replace) == (want_n, CAP, False)
        return row.astype(np.int64)


def dummy_record(strides, max_depth):
    """The record of a dummy entry: angle 0, unit K and Rtilt, the fixed T."""
    r = np.zeros(1, dtype=np.dtype(_lib.TrainFrustum))[0]
    rot = np.pi / 2.0 + 0.0
    r["rot"], r["cs"], r["sn"] = rot, np.cos(rot), np.sin(rot)
    r["K"] = r["Rtilt"] = np.eye(3).reshape(9)
    r["T"][:len(strides)] = [len(np.arange(0, max_depth, s)) for s in strides]
    return r


def frame_tables(clouds, cloud_counts, calibs, boxes, det_class, det_prob, det_counts, P_out, class_mask, seed, call,
                 strides, max_depth):
    """The outputs of fcn_sunrgbd_frame_extract for F frames of capacities (P, D) = clouds.shape[1], boxes.shape[1]:
    clouds (F, P, 6) float32, cloud_counts (F,), calibs F dicts (Rtilt, K), boxes (F, D, 4) float64, det_class (F, D),
    det_prob (F, D) float32, det_counts (F,); seed and call: the cap draw's key and call counter.  -> dict of status,
    points (offsets[B], 6) float32, offsets (B + 1), det_index, valid, cls_index, rgb_prob, seg (B each), box2d
    (B, 4) float32, seg_class (F, 10), cap_choice (B, 2048), records (B) fcn_train_frustum and angle (B): the
    frustum angle of each kept entry (0 for a dummy); also det_points (B), each slot's in-box count n (-1: not a
    candidate) and kept (B), its kept points before the budget (-1: dropped)."""
    F, P = clouds.shape[:2]
    D = boxes.shape[1]
    B = F * D
    status = 0
    det_points, kept_n = np.full(B, -1, np.int64), np.full(B, -1, np.int64)
    cap_choice = np.zeros((B, CAP), np.int32)
    pts, angle = {}, {}
    flat_boxes, flat_cls, flat_prob = boxes.reshape(-1, 4), det_class.reshape(-1), det_prob.reshape(-1)
    for f in range(F):
        c, nd = int(cloud_counts[f]), int(det_counts[f])
        status |= (SCAN_POINTS if c > P else 0) | (DETS if nd > D else 0)
        cloud = clouds[f, :min(max(c, 0), P)]
        slots = []
        for j in range(min(max(nd, 0), D)):
            d = f * D + j
            cls, b = int(flat_cls[d]), flat_boxes[d]
            if not (0 <= cls < NC and np.all(np.isfinite(b))):
                status |= BAD_DET
            elif (class_mask >> cls) & 1:
                slots.append(d)
        if not slots:
            continue
        uv = ox.image_coords(cloud, calibs[f])
        for d in slots:
            det_points[d] = int(ox.cut(uv, flat_boxes[d]).sum())
        rows = []
        for d in slots:
            if det_points[d] > CAP:
                cap_choice[d] = choice_row(int(det_points[d]), CAP, seed, d, call)
                rows.append((int(det_points[d]), cap_choice[d]))
        # every candidate is tagged with its slot as its type, so the kept lists name their slots
        tags = [str(d) for d in slots]
        L, trace = ox.from_rgb_detections({f: cloud}, {f: calibs[f]}, [f] * len(slots), tags,
                                          [flat_boxes[d] for d in slots], [float(flat_prob[d]) for d in slots],
                                          type_whitelist=tags, rng=_Rows(rows))
        assert [t["n"] for t in trace] == [int(det_points[d]) for d in slots]
        for t, p, a in zip(L["type"], L["input"], L["frustum_angle"]):
            d = int(t)
            kept_n[d], pts[d], angle[d] = len(p), p, a
    seg_class = np.full((F, NC), -1, np.int32)
    entries = []                      # (slot, seg) of the kept frustums, in slot order
    for f in range(F):
        kp = kept_n[f * D:(f + 1) * D]
        if kp[kp >= 0].sum() > P_out:
            status |= OUT_POINTS
        c2 = budget(kp, P_out)
        rank, seg_class[f] = class_ranks(flat_cls[f * D:(f + 1) * D], c2 >= 0)
        entries += [(f * D + j, NC * f + rank[flat_cls[f * D + j]]) for j in range(D) if c2[j] >= 0]
    K = len(entries)
    slots = [d for d, _ in entries]
    rec = np.zeros(B, dtype=np.dtype(_lib.TrainFrustum))
    if K:
        rec[:K] = frustum_table("sunrgbd", strides, max_depth, False, SUNRGBD_CLASSES,
                                [SUNRGBD_CLASSES[flat_cls[d]] for d in slots],
                                frustum_angle_list=[angle[d] for d in slots],
                                box2d_list=[flat_boxes[d] for d in slots],
                                calib_K_list=[np.asarray(calibs[d // D]["K"], np.float64) for d in slots],
                                calib_R_list=[np.asarray(calibs[d // D]["Rtilt"], np.float64) for d in slots],
                                prob_list=[float(flat_prob[d]) for d in slots])
    rec[K:] = dummy_record(strides, max_depth)
    allp = [pts[d] for d in slots] + [np.zeros((1, 6), np.float32)] * (B - K)
    counts = [len(p) for p in allp]
    return {
        "status": status,
        "points": np.concatenate(allp).astype(np.float32),
        "offsets": np.concatenate([[0], np.cumsum(counts)]).astype(np.int32),
        "det_index": np.array(slots + [-1] * (B - K), np.int32),
        "valid": np.array([1] * K + [0] * (B - K), np.int32),
        "cls_index": np.array([flat_cls[d] for d in slots] + [0] * (B - K), np.int32),
        "rgb_prob": np.array([flat_prob[d] for d in slots] + [0.0] * (B - K), np.float32),
        "box2d": np.array([flat_boxes[d] for d in slots] + [[0.0, 0.0, 1.0, 1.0]] * (B - K),
                          np.float64).reshape(B, 4).astype(np.float32),
        "seg": np.array([s for _, s in entries] + [0] * (B - K), np.int32),
        "seg_class": seg_class,
        "cap_choice": cap_choice,
        "records": rec,
        "angle": np.array([angle[d] for d in slots] + [0.0] * (B - K), np.float64),
        "det_points": det_points,
        "kept": kept_n,
    }
