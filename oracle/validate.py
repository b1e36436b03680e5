"""ORACLE (test infrastructure) - numpy restatement of the validation pass (csrc/validate.cu,
frustum_convnet_b200/validate.py).

``batch_values`` restates the eval-with-labels branch of models/det_base.py:414-525 from the head logits, in
float32 where the reference computes in float32 (the IoU in float64, as the Boost call returns it);
``average_meters`` replays utils/utils.py:51-67 AverageMeter through TrainingStates in Python floats (float64)."""
from __future__ import annotations

from collections import OrderedDict

import numpy as np

from .box_iou import rbbox_iou_3d_pair

F32 = np.float32
LOSS_KEYS = ("total_loss", "cls_loss", "center_loss", "head_cls_loss", "head_res_loss", "size_cls_loss",
             "size_res_loss", "corners_loss")


def _softmax(x):
    m = x.max(-1, keepdims=True)
    e = np.exp(x - m)
    return e / e.sum(-1, keepdims=True)


def _huber(a, delta):
    a = np.abs(a)
    q = np.minimum(a, F32(delta))
    return (F32(0.5) * q * q + F32(delta) * (a - q)).mean(dtype=F32)


def _corners(c, h, s):
    l, w, hh = s[:, 0], s[:, 1], s[:, 2]
    half = F32(0.5)
    xs = np.stack([l, l, -l, -l, l, l, -l, -l], 1) * half
    ys = np.stack([hh, hh, hh, hh, -hh, -hh, -hh, -hh], 1) * half
    zs = np.stack([w, -w, -w, w, w, -w, -w, w], 1) * half
    cs, sn = np.cos(h)[:, None], np.sin(h)[:, None]
    return np.stack([cs * xs + sn * zs + c[:, 0:1], ys + c[:, 1:2], -sn * xs + cs * zs + c[:, 2:3]], 2).astype(F32)


def _angle_decode(res, cls, nb):
    apc = F32(2 * np.pi / nb)
    ang = cls.astype(F32) * apc + res[np.arange(len(cls)), cls] * (apc / F32(2))
    return np.where(ang > F32(np.pi), ang - F32(2 * np.pi), ang).astype(F32)


def batch_values(cls, reg, center_ref2, cls_label, size_class, box3d_center, box3d_heading, box3d_size, mean_size,
                 num_bins, weights=(1.0, 20.0, 20.0, 10.0), iou_thresh=0.7, with_iou=True, details=False):
    """The 14 values of one batch (loss keys, then cls_acc, head_acc, size_acc, IoU_2D, IoU_3D, IoU_thresh).
    cls (B,2,T2) and reg (B,out,T2) as the heads emit them; labels as the providers collate them.
    details=True also returns per-row quantities the tests use to find rows near a decision boundary."""
    cls, reg = np.asarray(cls, F32), np.asarray(reg, F32)
    B, _, T2 = cls.shape
    nb, ns = int(num_bins), len(mean_size)
    mean_size = np.asarray(mean_size, F32)
    cs = cls.transpose(0, 2, 1).reshape(-1, 2)
    out = reg.transpose(0, 2, 1).reshape(B * T2, -1)
    ref2 = np.asarray(center_ref2, F32).transpose(0, 2, 1).reshape(-1, 3)
    lab = np.asarray(cls_label).reshape(-1).astype(np.int64)
    p = _softmax(cs)
    fg = np.nonzero(lab == 1)[0]
    keep = np.nonzero(lab != -1)[0]
    nfg = len(fg)
    assert nfg != 0
    # focal loss (common.py:217-232)
    t = lab[keep]
    alpha = F32(0.75) * (t == 0).astype(F32) + F32(0.25) * (t >= 1).astype(F32)
    pt = p[keep, t]
    focal = -alpha * (F32(1) - pt) ** 2 * np.log(pt + F32(1e-14))
    cls_loss = F32(focal.sum(dtype=F32) / F32(nfg + 1e-14))
    bidx = fg // T2
    o = out[fg]
    ctr, hs, hr = o[:, 0:3], o[:, 3:3 + nb], o[:, 3 + nb:3 + 2 * nb]
    ss, sr = o[:, 3 + 2 * nb:3 + 2 * nb + ns], o[:, 3 + 2 * nb + ns:].reshape(-1, ns, 3)
    c_l = np.asarray(box3d_center, F32).reshape(B, 3)[bidx]
    h_l = np.asarray(box3d_heading, F32).reshape(B)[bidx]
    s_l = np.asarray(box3d_size, F32).reshape(B, 3)[bidx]
    sc = np.asarray(size_class).reshape(B).astype(np.int64)[bidx]
    r2 = ref2[fg]
    two_pi = F32(2 * np.pi)
    apc = F32(2 * np.pi / nb)
    g = np.mod(h_l, two_pi)
    shifted = np.mod(g + apc / F32(2), two_pi)
    hc = np.floor(shifted / apc).astype(np.int64)
    hres_lab = (shifted - (hc.astype(F32) * apc + apc / F32(2))) / (apc / F32(2))
    ex = mean_size[sc]
    s_res_lab = (s_l - ex) / ex
    center_loss = _huber(np.linalg.norm((c_l - r2) - ctr, axis=-1).astype(F32), 3.0)
    lsm_h = hs - hs.max(-1, keepdims=True)
    lsm_h = lsm_h - np.log(np.exp(lsm_h).sum(-1, keepdims=True))
    head_cls = F32(-lsm_h[np.arange(nfg), hc].mean(dtype=F32))
    head_res = _huber(hr[np.arange(nfg), hc] - hres_lab, 1.0)
    lsm_s = ss - ss.max(-1, keepdims=True)
    lsm_s = lsm_s - np.log(np.exp(lsm_s).sum(-1, keepdims=True))
    size_cls = F32(-lsm_s[np.arange(nfg), sc].mean(dtype=F32))
    s_sel = sr[np.arange(nfg), sc]
    size_res = _huber(np.linalg.norm(s_res_lab - s_sel, axis=-1).astype(F32), 1.0)
    cp = r2 + ctr
    c_pred = _corners(cp, _angle_decode(hr, hc, nb), s_sel * ex + ex)
    c_gt = _corners(c_l, h_l, s_l)
    c_flip = _corners(c_l, h_l + F32(np.pi), s_l)
    dist = np.minimum(np.linalg.norm(c_pred - c_gt, axis=-1).mean(-1, dtype=F32),
                      np.linalg.norm(c_pred - c_flip, axis=-1).mean(-1, dtype=F32))
    corners = _huber(dist.astype(F32), 1.0)
    w_box, w_h, w_s, w_c = (F32(w) for w in weights)
    total = cls_loss + w_box * (center_loss + head_cls + size_cls + w_h * head_res + w_s * size_res + w_c * corners)
    # accuracies: correct.sum() * float32(1.0 / n) (utils/utils.py:28-48)
    cls_acc = F32((np.argmax(p[keep], -1) == t).sum()) * F32(1.0 / len(keep))
    hp, sp = _softmax(hs), _softmax(ss)
    h_arg, s_arg = np.argmax(hp, -1), np.argmax(sp, -1)
    head_acc = F32((h_arg == hc).sum()) * F32(1.0 / nfg)
    size_acc = F32((s_arg == sc).sum()) * F32(1.0 / nfg)
    iou = np.full((nfg, 2), np.nan)
    if with_iou:
        ms = mean_size[s_arg]
        c_metric = _corners(cp, _angle_decode(hr, h_arg, nb), sr[np.arange(nfg), s_arg] * ms + ms)
        iou = rbbox_iou_3d_pair(c_metric, c_gt)
        ious = (F32(iou[:, 0].mean()), F32(iou[:, 1].mean()), F32((iou[:, 1] >= iou_thresh).mean()))
    else:
        ious = (F32(np.nan),) * 3
    vals = np.array([total, cls_loss, center_loss, head_cls, head_res, size_cls, size_res, corners,
                     cls_acc, head_acc, size_acc, *ious], dtype=F32)
    if not details:
        return vals

    def margin(pr):
        s = np.sort(pr, -1)
        return s[:, -1] - s[:, -2]
    return vals, dict(nfg=nfg, nkeep=len(keep), iou3d=iou[:, 1], cls_margin=margin(p[keep]), head_margin=margin(hp),
                      size_margin=margin(sp))


def average_meters(rows, batch_sizes, keys):
    """TrainingStates.update_states(values, batch_size) per row, then get_states(avg=True): -> (states, meters) with
    meters[key] = (sum, count), all Python floats (float64)."""
    sums = {k: 0 for k in keys}
    count = 1e-14
    for vals, n in zip(rows, batch_sizes):
        n = int(n)
        for k, v in zip(keys, vals):
            sums[k] += float(v) * n
        count += n
    states = OrderedDict((k, sums[k] / count) for k in keys)
    return states, OrderedDict((k, (float(sums[k]), float(count))) for k in keys)


# ----------------------------------------------------------------------------------- fixture epochs
# name -> workload, weight seed, batches (B, data seed, max_depth override, refine half-extent of the refs).  Small T
# keeps the fixtures small; every epoch ends with a partial batch; the refine epoch mixes two T pyramids.
VAL_CASES = {
    "kitti": ("car", 7, [(3, 301, 17.5, None), (3, 302, 17.5, None), (2, 303, 17.5, None)]),
    "sunrgbd": ("sunrgbd", 10, [(2, 311, 4.0, None), (2, 312, 4.0, None), (1, 313, 4.0, None)]),
    "refine": ("refine_car", 11, [(3, 321, None, None), (3, 322, None, 1.5), (2, 323, None, None)]),
}


def epoch_inputs(name):
    """The label-free inputs of each batch of fixture epoch `name` (numpy dicts, reference key names).  A refine batch
    with a half-extent gets its section centres rebuilt as synth does for 0.977: arange(-h, h, s) + s / 2."""
    from frustum_convnet_b200 import synth
    workload, _, batches = VAL_CASES[name]
    out = []
    for B, seed, md, half in batches:
        d = synth.make_frustums(workload, B, seed=seed, max_depth=md)
        if half is not None:
            for i, s in enumerate(synth._PRESETS[workload]["strides"]):
                zc = np.arange(-half, half, s) + s / 2.0
                c = np.zeros((B, 3, len(zc)), dtype=np.float64)
                c[:, 2, :] = zc[None, :]
                d["center_ref%d" % (i + 1)] = c.astype(np.float32)
        out.append(d)
    return out


def checksum(batches):
    return float(sum(np.asarray(v, dtype=np.float64).sum() for d in batches for v in d.values()))
