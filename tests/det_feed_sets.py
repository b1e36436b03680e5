"""Detection sets fed through a DetectionCollector so that finalize() returns chosen rows: one frustum per row, T2 = 1,
rot_angle 0, no ref_center and rgb_prob 0, method 'top' (every row kept; KITTI scores are positive).  The decode then
passes box2d, the size, ry and the score through unchanged (score = p1 + 0 for KITTI, 0 + max size_prob for SUN-RGBD), tx and tz as
x * 1 + z * 0, and KITTI's ty as (ty - h / 2) + h / 2 in float32 (exact for the dyadic values of the tie sets)."""
import numpy as np
import torch


def collector_for(det_results, dataset, extra_frustums=(), method="top", device=None):
    """det_results {idx: {class: (n, 12) float32 rows}} -> (DetectionCollector with every row added, the frustums'
    (id, class) in dataset order).  `extra_frustums`: (id, class) pairs appended to the dataset and never added.
    Rows with a size below 0.01 are dropped by the decode, so such rows give zero-row lists."""
    from frustum_convnet_b200.detect import DetectionCollector
    ids, types, rows = [], [], []
    for idx, by_class in det_results.items():
        for ct, d in by_class.items():
            d = np.asarray(d, np.float32).reshape(-1, 12)
            if len(d) == 0:                       # a list that exists but holds nothing: one dropped row
                d = np.zeros((1, 12), np.float32)
            for r in d:
                ids.append(idx)
                types.append(ct)
                rows.append(r)
    F = len(rows)
    rows = np.asarray(rows, np.float32).reshape(F, 12)
    all_ids = ids + [i for i, _ in extra_frustums]
    all_types = types + [c for _, c in extra_frustums]
    box2d = np.concatenate([rows[:, :4], np.zeros((len(extra_frustums), 4), np.float32)]).astype(np.float64)
    col = DetectionCollector(all_ids, all_types, box2d, dataset=dataset, method=method, thresh=0.1,
                             capacity=max(F, 1), device=device)
    if F == 0:
        return col
    dev = col.device
    kitti = dataset == "KITTI"
    if kitti:
        size = rows[:, [9, 8, 7]]                                          # (l, w, h) from [h, w, l]
        y = rows[:, 5] - rows[:, 7] * np.float32(0.5)
    else:
        size = rows[:, [7, 8, 9]]
        y = rows[:, 5]
    cls_probs = np.zeros((F, 1, 2), np.float32)
    cls_probs[:, 0, 1] = rows[:, 11] if kitti else 1      # 'top' needs p1 above 0 to pick the position
    size_probs = (rows[:, 11] if not kitti else np.zeros(F, np.float32)).reshape(F, 1, 1).astype(np.float32)
    center = np.stack([rows[:, 4], y, rows[:, 6]], 1).reshape(F, 1, 3).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    outs = (t(cls_probs), t(center), t(rows[:, 10].reshape(F, 1)), t(size.reshape(F, 1, 3)), t(size_probs),
            t(size_probs))
    d = {"rot_angle": t(np.zeros((F, 1), np.float32)), "rgb_prob": t(np.zeros((F, 1), np.float32))}
    col.add(outs, d, first=0)
    return col


def kitti_rows(records):
    """(n, 14) float64 result records -> (n, 12) float32 rows [x1, y1, x2, y2, tx, ty, tz, h, w, l, ry, score]."""
    r = np.asarray(records, np.float64).reshape(-1, 14)
    return np.concatenate([r[:, 2:6], r[:, 9:12], r[:, 6:9], r[:, 12:14]], 1).astype(np.float32)


KITTI_NAMES = {0: "Car", 1: "Pedestrian", 2: "Cyclist", 3: "Van", 4: "Person_sitting", 5: "DontCare", 6: "Truck"}


def kitti_set(n_images, seed=0):
    """The synthetic KITTI set of scripts/bench_kitti_eval.py at n_images -> (gt records per image, det_results)."""
    from oracle import kitti_synth as ks
    labels, results = ks.make_set(seed, n_images, n_obj=8, det_rate=0.8)
    gts = [ks.parse_label_lines(l) for l in labels]
    dets = {}
    for i, lines in enumerate(results):
        rec = ks.parse_result_lines(lines)
        if len(rec) == 0:
            continue
        by = {}
        for code in dict.fromkeys(rec[:, 0].astype(int).tolist()):
            by[KITTI_NAMES[code]] = kitti_rows(rec[rec[:, 0] == code])
        dets[i] = by
    return gts, dets
