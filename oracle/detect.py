"""TEST INFRASTRUCTURE ONLY - numpy restatement of the reference's per-batch detection loop and its NMS pass.

KITTI: train/test_net_det.py:243-293 (loop) and :126-152 (write_detection_results_nms); SUN-RGBD:
train/test_net_det_sunrgbd.py:197-252 and :120-145; from_prediction_to_label_format of
datasets/provider_sample.py:375-387 / provider_sample_sunrgbd.py:374-385.  NMS is oracle/nms.py (ties in the score
order: larger list index first).  Pinned by tests/golden/detect_{kitti,sunrgbd}.npz, which
oracle/make_golden_detect.py captures from the reference's own ``test()``.

    det = collect(batches, id_list, type_list, box2d_list, dataset, method)   # det_results[image][class] = rows
    res = nms_results(det, thresh, method)                                     # what write_detection_results gets
A batch is (first, outputs, rot_angle, rgb_prob or None, ref_center or None) with the six model outputs as numpy."""
import numpy as np

from . import nms as onms


def rotate_pc_along_y(pc, rot_angle):
    cosval, sinval = np.cos(rot_angle), np.sin(rot_angle)
    rotmat = np.array([[cosval, -sinval], [sinval, cosval]])
    pc = pc.copy()
    pc[:, [0, 2]] = np.dot(pc[:, [0, 2]], np.transpose(rotmat))
    return pc


def label_format(center, angle, size, rot_angle, ref_center, dataset):
    """-> (tx, ty, tz, l, w, h, ry) as the reference's float32 numpy scalars."""
    l, w, h = size
    ry = angle + rot_angle
    tx, ty, tz = rotate_pc_along_y(np.expand_dims(center, 0), -rot_angle).squeeze()
    tx, ty, tz = tx + ref_center[0], ty + ref_center[1], tz + ref_center[2]
    if dataset == "KITTI":
        ty += h / 2.0
    return tx, ty, tz, l, w, h, ry


def foreground(p, dataset, method):
    """fg positions of one frustum, p = cls_probs[b] (T2, 2)."""
    if method == "nms":
        fg = (p[:, 0] < p[:, 1]).nonzero()[0] if dataset == "KITTI" else (p[:, 1] > 0.5).nonzero()[0]
        if fg.size == 0:
            fg = np.array([np.argmax(p[:, 1])])
        return fg
    return np.array([np.argmax(p[:, 1])])


def collect(batches, id_list, type_list, box2d_list, dataset="KITTI", method="nms", trace=None):
    """det_results[data_idx][class_type] = list of float32 rows in dataset order.  `trace` (a list) receives
    (frustum, t, kept) for every selected position."""
    det = {}
    for first, outs, rot, rgb, ref in batches:
        cls_probs, center, heading, size, _, size_probs = [np.asarray(o, dtype=np.float32) for o in outs]
        B = cls_probs.shape[0]
        rot = np.asarray(rot, dtype=np.float32).reshape(-1)
        rgb = np.ones_like(rot) if rgb is None else np.asarray(rgb, dtype=np.float32).reshape(-1)
        ref = np.zeros((B, 3), dtype=np.float32) if ref is None else np.asarray(ref, dtype=np.float32)
        for b in range(B):
            fg = foreground(cls_probs[b], dataset, method)
            if dataset == "KITTI":
                scores = cls_probs[b, fg, 1] + rgb[b]
            else:
                scores = rgb[b] + size_probs[b, fg].max(1)
            f = first + b
            data_idx, class_type, box2d = id_list[f], type_list[f], box2d_list[f]
            lists = det.setdefault(data_idx, {}).setdefault(class_type, [])
            for n, t in enumerate(fg):
                tx, ty, tz, l, w, h, ry = label_format(center[b, t], heading[b, t], size[b, t], rot[b], ref[b],
                                                       dataset)
                kept = not (h < 0.01 or w < 0.01 or l < 0.01)
                if trace is not None:
                    trace.append((f, int(t), kept))
                if not kept:
                    continue
                x1, y1, x2, y2 = box2d
                if dataset == "KITTI":
                    lists.append([x1, y1, x2, y2, tx, ty, tz, h, w, l, ry, scores[n]])
                else:
                    lists.append([x1, y1, x2, y2, tx, ty, tz, l, w, h, ry, scores[n]])
    return det


def nms_boxes(dets, dataset):
    """(n, 12) rows -> (n, 8) [cx, cy, cz, l, w, h, ry, score] as the reference hands them to cube_nms."""
    return dets[:, 4:][:, [0, 1, 2, 5, 4, 3, 6, 7]] if dataset == "KITTI" else dets[:, 4:]


def nms_results(det, thresh, dataset="KITTI", method="nms", top_k=300):
    """{data_idx: {class_type: float32 (n, 12)}}; with method 'nms' the keep lists of write_detection_results_nms
    (also returned per list as `keeps`), else the lists unchanged."""
    out, keeps = {}, {}
    for idx in det:
        for ct in det[idx]:
            dets = np.array(det[idx][ct], dtype=np.float32).reshape(-1, 12)
            if method == "nms" and len(dets) > 1:
                keep = onms.rotate_nms_3d_cc(nms_boxes(dets, dataset), thresh, top_k)
                dets = dets[keep]
            else:
                keep = list(range(len(dets)))
            out.setdefault(idx, {})[ct] = dets
            keeps[(idx, ct)] = keep
    return out, keeps


def sparse_pair_margin(boxes, thresh):
    """min |IoU_3D - thresh| over the pairs whose bounding cubes overlap (the only pairs the NMS tests), and the
    smallest |min overlap extent| of any pair (the cube test is that extent > 0): tests skip inputs where either
    decision is ambiguous in fp32."""
    from . import box_iou as ob
    b = np.asarray(boxes, dtype=np.float64)
    n = len(b)
    if n < 2:
        return np.inf, np.inf
    c = onms.boxes3d2corners(b)
    mn, mx = c.min(1), c.max(1)
    ext = np.minimum(mx[:, None], mx[None]) - np.maximum(mn[:, None], mn[None])      # (n, n, 3)
    iu = np.triu_indices(n, 1)
    e = ext[iu].min(1)                         # the cubes overlap iff this is > 0
    edge = float(np.abs(e).min())
    ov = e > 0
    m = np.inf
    for i, j in zip(iu[0][ov], iu[1][ov]):
        m = min(m, abs(ob.rbbox_iou_3d_pair(c[i:i + 1], c[j:j + 1])[0, 1] - thresh))
    return m, edge
