"""numpy restatement of fcn_frame_extract's tables (C ABI section (21), csrc/frame_extract.cu): the clamped frame
inputs, the status bits, the count pass (oracle/frustum_extract.extract on each clamped frame), each frame's P_out
budget, the class ranks and the B = F * D batch entries with their dummy tail."""
import numpy as np

from oracle.frustum_extract import extract

SCAN_POINTS, DETS, OUT_POINTS, BAD_DET = 1, 2, 4, 16          # FCN_FRAME_* bits of the C header
UNIT_P = np.array([1.0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0])


def synth_frames(rng, F, n_points, n_dets, classes=(0, 1, 2)):
    """F seeded KITTI-like frames: [(scan (n, 4) float32, calib, (h, w), [(class, prob, box2d), ...])]; detection j
    of a frame has class classes[(t0 + j) % len(classes)], a box inside the image and an object in its frustum."""
    from oracle import kitti_scan_synth as ks
    out = []
    for _ in range(F):
        calib = ks.kitti_calib(rng)
        hw = (int(rng.integers(370, 376)), int(rng.integers(1224, 1243)))
        dets, t0 = [], int(rng.integers(0, len(classes)))
        for j in range(n_dets):
            bw, bh = np.exp(rng.uniform(np.log(20), np.log(300))), np.exp(rng.uniform(np.log(10), np.log(200)))
            x0, y0 = rng.uniform(0, hw[1] - bw), rng.uniform(0, hw[0] - bh)
            dets.append((classes[(t0 + j) % len(classes)], float(np.float32(rng.uniform(0.05, 1.0))),
                         np.array([x0, y0, x0 + bw, y0 + bh]).round(2)))
        out.append((ks.kitti_scan(rng, calib, [d[2] for d in dets], n_points), calib, hw, dets))
    return out


def stage(frames, P, D, scan_counts=None, det_counts=None):
    """Frames as synth_frames gives them -> the raw inputs of fcn_frame_extract in capacities (P, D): (scans, scan_counts,
    calibs, image_hw, boxes, det_class, det_prob, det_counts).  Rows past a capacity are cut; the counts default to
    the frames' own (a count may exceed its capacity or be negative)."""
    F = len(frames)
    scans = np.zeros((F, P, 4), np.float32)
    boxes, det_class = np.zeros((F, D, 4)), np.zeros((F, D), np.int32)
    det_prob = np.zeros((F, D), np.float32)
    for f, (scan, _, _, dets) in enumerate(frames):
        scans[f, :min(len(scan), P)] = scan[:P]
        for j, (c, p, b) in enumerate(dets[:D]):
            det_class[f, j], det_prob[f, j], boxes[f, j] = c, p, b
    sc = np.array([len(x[0]) for x in frames] if scan_counts is None else scan_counts, np.int32)
    dc = np.array([len(x[3]) for x in frames] if det_counts is None else det_counts, np.int32)
    return (scans, sc, [x[1] for x in frames], np.array([x[2] for x in frames], np.int32).reshape(F, 2), boxes,
            det_class, det_prob, dc)


def budget(det_points, P_out):
    """One frame's slots after the count pass (det_points[j] = its points, -1 when dropped) -> the points of the
    slots that fit P_out, -1 for the others: a kept slot fits when the points of every kept slot before it in the
    frame, plus its own, are at most P_out (the longest prefix of the kept slots that fits)."""
    out, run = [], 0
    for c in det_points:
        if c < 0:
            out.append(-1)
            continue
        run += c
        out.append(c if run <= P_out else -1)
    return np.asarray(out, dtype=np.int64)


def class_ranks(classes, fits, num_classes=3):
    """One frame's slot classes and budget flags -> (rank of each class 0..num_classes - 1 or -1, seg_class
    (num_classes,)): classes by first appearance among the slots that fit."""
    rank, seg_class = [-1] * num_classes, [-1] * num_classes
    n = 0
    for c, ok in zip(classes, fits):
        if ok and rank[c] < 0:
            rank[c], seg_class[n] = n, c
            n += 1
    return rank, np.asarray(seg_class, dtype=np.int32)


def count_pass(scans, scan_counts, calibs, image_hw, boxes, det_class, det_counts, class_mask):
    """-> (status bits 1 | 2 | 16, slot table): slot f * D + j -> (points (n, 4) float32, clipped box2d, angle) for
    every slot the count pass keeps, from oracle/frustum_extract.extract on frame f's first min(scan_counts, P) points
    and first min(det_counts, D) detections."""
    F, P, _ = scans.shape
    D = boxes.shape[1]
    status, kept = 0, {}
    for f in range(F):
        c, nd = int(scan_counts[f]), int(det_counts[f])
        status |= (SCAN_POINTS if c > P else 0) | (DETS if nd > D else 0)
        n = min(max(c, 0), P)
        slots = []
        for j in range(min(max(nd, 0), D)):
            cls, b = int(det_class[f, j]), boxes[f, j]
            if not (0 <= cls < 3 and np.all(np.isfinite(b))):
                status |= BAD_DET
            elif (class_mask >> cls) & 1:
                slots.append(f * D + j)
        if not slots:
            continue
        # every candidate is tagged with its slot as its type, so the kept lists name their slots
        tags = [str(d) for d in slots]
        _, box2d, pts, types, angle, _, _ = extract(
            {f: scans[f, :n]}, {f: calibs[f]}, {f: tuple(image_hw[f])}, [f] * len(slots), tags, [0.0] * len(slots),
            [boxes.reshape(-1, 4)[d] for d in slots], type_whitelist=tags)
        for t, b, p, a in zip(types, box2d, pts, angle):
            kept[int(t)] = (p, np.asarray(b, np.float64), float(a))
    return status, kept


def frame_tables(scans, scan_counts, calibs, image_hw, boxes, det_class, det_prob, det_counts, P_out, class_mask=7):
    """The outputs of fcn_frame_extract for F frames of capacities (P, D) = scans.shape[1], boxes.shape[1]:
    scans (F, P, 4) float32, scan_counts (F,), calibs F dicts (P2, Tr_velo_to_cam, R0_rect), image_hw (F, 2),
    boxes (F, D, 4) float64, det_class (F, D), det_prob (F, D) float32, det_counts (F,).  -> dict of status,
    points (offsets[B], 4) float32, offsets (B + 1), frustum_angle, box2d, P, det_index, valid, cls_index, rgb_prob,
    seg (B each) and seg_class (F, 3); also det_points (B), the count pass's points of each slot (-1: dropped)."""
    F, D = boxes.shape[:2]
    B = F * D
    status, kept = count_pass(scans, scan_counts, calibs, image_hw, boxes, det_class, det_counts, class_mask)
    det_points = np.array([len(kept[d][0]) if d in kept else -1 for d in range(B)], dtype=np.int64)
    cls = det_class.reshape(-1)
    seg_class = np.full((F, 3), -1, np.int32)
    entries = []                      # (slot, seg) of the kept frustums, in slot order
    for f in range(F):
        dp = det_points[f * D:(f + 1) * D]
        if dp[dp >= 0].sum() > P_out:
            status |= OUT_POINTS
        c2 = budget(dp, P_out)
        rank, seg_class[f] = class_ranks(cls[f * D:(f + 1) * D], c2 >= 0)
        entries += [(f * D + j, 3 * f + rank[cls[f * D + j]]) for j in range(D) if c2[j] >= 0]
    K = len(entries)
    pts = [kept[d][0] for d, _ in entries] + [np.zeros((1, 4), np.float32)] * (B - K)
    counts = [len(p) for p in pts]
    prob = det_prob.reshape(-1)
    calib_P = [np.asarray(calibs[d // D]["P2"], np.float64).reshape(12) for d, _ in entries]
    return {
        "status": status,
        "points": np.concatenate(pts).astype(np.float32) if pts else np.zeros((0, 4), np.float32),
        "offsets": np.concatenate([[0], np.cumsum(counts)]).astype(np.int32),
        "frustum_angle": np.array([kept[d][2] for d, _ in entries] + [0.0] * (B - K), np.float64),
        "box2d": np.array([kept[d][1] for d, _ in entries] + [[0.0, 0.0, 1.0, 1.0]] * (B - K),
                          np.float64).reshape(B, 4),
        "P": np.array(calib_P + [UNIT_P] * (B - K), np.float64).reshape(B, 12),
        "det_index": np.array([d for d, _ in entries] + [-1] * (B - K), np.int32),
        "valid": np.array([1] * K + [0] * (B - K), np.int32),
        "cls_index": np.array([cls[d] for d, _ in entries] + [0] * (B - K), np.int32),
        "rgb_prob": np.array([prob[d] for d, _ in entries] + [0.0] * (B - K), np.float32),
        "seg": np.array([s for _, s in entries] + [0] * (B - K), np.int32),
        "seg_class": seg_class,
        "det_points": det_points,
    }
