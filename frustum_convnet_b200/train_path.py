"""Training-mode / label-branch forward of the drop-in modules.

Scope note (SURVEY.md section 8 a6): the train branch of PointNetDet.forward
(/root/reference/models/det_base.py:414-525) "stays in PyTorch autograd".  Batch-statistics
BatchNorm makes the eval kernels (folded BN, duplicate-row skipping) inapplicable, so here the
grouping runs on libfrustum_b200 (``QueryDepthPoint``) and the differentiable arithmetic is
composed from torch CUDA ops on the modules' own parameters.  Loss definitions follow
det_base.py:280-332,414-476, models/model_util.py:9-19,48-72, models/common.py:80-94,217-232 and
models/box_transform.py:15-65.  The CPU Boost IoU metric (det_base.py:494-503,
ops/pybind11/box_ops.h) is row 8(f)-1: it is computed on the device by ``fcn_rbbox_iou_3d_pair``
(box_iou.py) by default; ``model.gpu_iou_metrics = False`` opts out (NaN placeholders).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from .config import get_cfg


# ------------------------------------------------------------------ feature path (autograd)
def pointnet_module_torch(mod, pc, feat, new_pc):
    B, T, K = pc.size(0), new_pc.shape[2], mod.nsample
    idx, num = mod.query_depth_point(pc, new_pc)
    flat = idx.view(B, 1, T * K)
    parts = []
    if mod.use_xyz:
        g = torch.gather(pc, 2, flat.expand(-1, 3, -1)).view(B, 3, T, K)
        parts.append(g - new_pc.unsqueeze(3))
    if mod.use_feature:
        parts.append(torch.gather(feat, 2, flat.expand(-1, feat.size(1), -1)).view(B, feat.size(1), T, K))
    x = parts[0].contiguous() if len(parts) == 1 else torch.cat(parts, 1)
    x = mod.conv3(mod.conv2(mod.conv1(x)))
    return x * (num > 0).view(B, 1, -1, 1).float()


def pointnet_feat_torch(mod, point_cloud, sample_pc, feat, one_hot_vec):
    outs = []
    for i, c in enumerate(sample_pc):
        f = getattr(mod, "pointnet%d" % (i + 1))(point_cloud, feat, c).max(-1)[0]
        if one_hot_vec is not None:
            assert mod.num_vec == one_hot_vec.shape[1]
            f = torch.cat([f, one_hot_vec.unsqueeze(-1).expand(-1, -1, f.shape[-1])], 1)
        outs.append(f)
    return tuple(outs)


def conv_feat_net_torch(mod, xs):
    S = len(xs)
    x = mod.block1_conv1(xs[0])
    branches = []
    for i in range(2, S + 1):
        x = getattr(mod, "block%d_conv1" % i)(x)
        x = getattr(mod, "block%d_conv2" % i)(x)
        x = getattr(mod, "block%d_merge" % i)(torch.cat([x, xs[i - 1]], 1))
        branches.append(x)
    ups = [getattr(mod, "block%d_deconv" % (i + 2))(b) for i, b in enumerate(branches)]
    L = ups[0].shape[-1]
    return torch.cat([u[:, :, :L] for u in ups], 1)


# ------------------------------------------------------------------ box coding / losses
def huber(err, delta):
    a = err.abs()
    q = torch.clamp(a, max=delta)
    return (0.5 * q * q + delta * (a - q)).mean()


def focal_loss_ignore(prob, target, alpha=0.25, gamma=2, ignore_idx=-1):
    keep = (target != ignore_idx).nonzero().view(-1)
    num_fg = (target > 0).sum()
    target, prob = target[keep], prob[keep, :]
    alpha_t = (1 - alpha) * (target == 0).float() + alpha * (target >= 1).float()
    p_t = prob[torch.arange(len(target), device=prob.device), target]
    loss = -alpha_t * (1 - p_t) ** gamma * torch.log(p_t + 1e-14)
    return loss.sum() / (num_fg + 1e-14)


def accuracy(output, target, ignore=None):
    if ignore is not None:
        keep = (target != ignore).nonzero().view(-1)
        output, target = output[keep], target[keep]
    pred = torch.argmax(output, -1)
    return (pred.view(-1) == target.view(-1)).float().sum() * (1.0 / target.view(-1).shape[0])


def angle_encode(gt, num_bins):
    two_pi = 2 * np.pi
    gt = gt % two_pi
    apc = two_pi / float(num_bins)
    shifted = (gt + apc / 2) % two_pi
    cls = torch.floor(shifted / apc).long()
    res = shifted - (cls.float() * apc + apc / 2)
    return cls, res / (apc / 2)


def angle_decode(res, cls, num_bins):
    apc = 2 * np.pi / float(num_bins)
    ang = cls.float() * apc + torch.gather(res, 1, cls.unsqueeze(1)).squeeze(1) * (apc / 2)
    return torch.where(ang > np.pi, ang - 2 * np.pi, ang)


def size_decode(off, mean_size, cls):
    sel = torch.gather(off, 1, cls.view(-1, 1, 1).expand(-1, -1, 3)).squeeze(1)
    ex = mean_size[cls]
    return sel * ex + ex


def box_corners(centers, headings, sizes):
    l, w, h = sizes[:, 0], sizes[:, 1], sizes[:, 2]
    xs = torch.stack([l, l, -l, -l, l, l, -l, -l], 1) / 2
    ys = torch.stack([h, h, h, h, -h, -h, -h, -h], 1) / 2
    zs = torch.stack([w, -w, -w, w, w, -w, -w, w], 1) / 2
    corners = torch.stack([xs, ys, zs], 1)
    c, s = torch.cos(headings), torch.sin(headings)
    one, zero = torch.ones_like(c), torch.zeros_like(c)
    R = torch.stack([torch.stack([c, zero, s], 1), torch.stack([zero, one, zero], 1),
                     torch.stack([-s, zero, c], 1)], 1)
    return (torch.bmm(R, corners) + centers.unsqueeze(2)).transpose(1, 2).contiguous()


def slice_output(out, num_bins, num_sizes):
    n = out.shape[0]
    c0 = 3 + num_bins
    c1 = c0 + num_bins
    c2 = c1 + num_sizes
    return (out[:, 0:3].contiguous(), out[:, 3:c0].contiguous(), out[:, c0:c1].contiguous(),
            out[:, c1:c2].contiguous(), out[:, c2:].contiguous().view(n, num_sizes, 3))


def _iou_metrics(c_metric, c_gt, thresh):
    """(mean IoU_2D, mean IoU_3D, fraction >= thresh) on the device (det_base.py:494-503)."""
    from .box_iou import rbbox_iou_3d_pair
    _, stats = rbbox_iou_3d_pair(c_metric, c_gt, iou_thresh=thresh)
    return stats


def pointnet_det_torch(model, data):
    pc = data.get("point_cloud")
    one_hot = data.get("one_hot")
    S = model.ARCH.num_scales
    centers = [data.get("center_ref%d" % (i + 1)) for i in range(S)]
    xyz = pc[:, :3, :].contiguous()
    extra = pc[:, [3], :].contiguous() if pc.shape[1] > 3 else None
    feats = model.feat_net(xyz, centers, extra, one_hot)
    x = model.conv_net(*feats)
    cls_scores, outputs = model.cls_out(x), model.reg_out(x)
    osz = outputs.shape[1]
    cls_scores = cls_scores.permute(0, 2, 1).contiguous().view(-1, 2)
    outputs = outputs.permute(0, 2, 1).contiguous().view(-1, osz)
    return losses_from_logits(model, cls_scores, outputs, centers[1], data)


def deterministic_mode(setting):
    """The training kernels' mode for a ``deterministic`` setting: True / False as given, None follows
    ``torch.are_deterministic_algorithms_enabled()`` (read at every step)."""
    return torch.are_deterministic_algorithms_enabled() if setting is None else bool(setting)


def pointnet_det_kernels(model, data):
    """Train branch on the hand-written kernels (csrc/train.cu): everything up to the head logits runs through
    ``TrainEngine`` behind an autograd.Function, the losses are the PyTorch ops below."""
    from .train_engine import LogitsFn, TrainEngine
    S = model.ARCH.num_scales
    pc = data["point_cloud"][:, :3, :].contiguous()
    centers = [data["center_ref%d" % (i + 1)].contiguous() for i in range(S)]
    det = deterministic_mode(getattr(model, "deterministic", None))
    key = (pc.shape[0], pc.shape[2], tuple(c.shape[2] for c in centers), det)
    cache = model.__dict__.setdefault("_train_engines", {})
    eng = cache.get(key)
    if eng is None:
        eng = cache[key] = TrainEngine(model, *key[:3], deterministic=det)
    params = tuple(model.parameters())
    cls, reg = LogitsFn.apply(eng, pc, data.get("one_hot"), S, *centers, *params)
    return losses_from_logits(model, cls, reg, centers[1], data)


def losses_from_logits(model, cls_scores, outputs, center_ref2, data):
    """det_base.py:376-525 from the head logits on: ``cls_scores`` (B*T2, 2), ``outputs`` (B*T2, out) rows in
    (frustum, position) order.  Eval decode without labels, else (losses, metrics)."""
    cfg = get_cfg()
    pc = data.get("point_cloud")
    cls_label, size_class = data.get("cls_label"), data.get("size_class")
    center_label, heading_label, size_label = (data.get("box3d_center"), data.get("box3d_heading"),
                                               data.get("box3d_size"))
    B = pc.shape[0]
    num_out = cls_scores.shape[0] // B
    mean_size = torch.from_numpy(model.mean_size_array).type_as(pc)
    ref2 = center_ref2.permute(0, 2, 1).contiguous().view(-1, 3)
    cls_probs = F.softmax(cls_scores, -1)
    nb, ns = model.num_bins, model.num_size_cluster

    if center_label is None:  # eval decode composed from torch ops (e.g. 4-channel inputs)
        assert not model.training, "Please provide labels for training."
        ctr, h_sc, h_res, s_sc, s_res = slice_output(outputs, nb, ns)
        h_pr, s_pr = F.softmax(h_sc, -1), F.softmax(s_sc, -1)
        h_lab, s_lab = torch.argmax(h_pr, -1), torch.argmax(s_pr, -1)
        return (cls_probs.view(B, -1, 2), (ctr + ref2).view(B, -1, 3),
                angle_decode(h_res, h_lab, nb).view(B, -1), size_decode(s_res, mean_size, s_lab).view(B, -1, 3),
                h_pr.view(B, -1, nb), s_pr.view(B, -1, ns))

    fg = (cls_label.view(-1) == 1).nonzero().view(-1)
    assert fg.numel() != 0
    outputs, ref2 = outputs[fg, :], ref2[fg]
    ctr, h_sc, h_res, s_sc, s_res = slice_output(outputs, nb, ns)
    h_pr, s_pr = F.softmax(h_sc, -1), F.softmax(s_sc, -1)
    cls_loss = focal_loss_ignore(cls_probs, cls_label.view(-1), ignore_idx=-1)

    center_label = center_label.unsqueeze(1).expand(-1, num_out, -1).contiguous().view(-1, 3)[fg]
    heading_label = heading_label.expand(-1, num_out).contiguous().view(-1)[fg]
    size_label = size_label.unsqueeze(1).expand(-1, num_out, -1).contiguous().view(-1, 3)[fg]
    size_class = size_class.expand(-1, num_out).contiguous().view(-1)[fg]

    center_gt = center_label - ref2
    h_cls, h_res_lab = angle_encode(heading_label, nb)
    ex = mean_size[size_class]
    s_res_lab = (size_label - ex) / ex

    center_loss = huber(torch.norm(center_gt - ctr, 2, dim=-1), 3.0)
    head_cls_loss = F.cross_entropy(h_sc, h_cls)
    head_res_loss = huber(torch.gather(h_res, 1, h_cls.view(-1, 1)).squeeze(1) - h_res_lab, 1.0)
    size_cls_loss = F.cross_entropy(s_sc, size_class)
    s_sel = torch.gather(s_res, 1, size_class.view(-1, 1, 1).expand(-1, 1, 3)).squeeze(1)
    size_res_loss = huber(torch.norm(s_res_lab - s_sel, 2, dim=-1), 1.0)

    center_preds = ref2 + ctr
    heading = angle_decode(h_res, h_cls, nb)
    size = size_decode(s_res, mean_size, size_class)
    c_gt = box_corners(center_label, heading_label, size_label)
    c_flip = box_corners(center_label, heading_label + np.pi, size_label)
    c_pred = box_corners(center_preds, heading, size)
    corner_dist = torch.min(torch.norm(c_pred - c_gt, 2, dim=-1).mean(-1),
                            torch.norm(c_pred - c_flip, 2, dim=-1).mean(-1))
    corners_loss = huber(corner_dist, 1.0)

    L = cfg.LOSS
    loss = cls_loss + L.BOX_LOSS_WEIGHT * (center_loss + head_cls_loss + size_cls_loss +
                                           L.HEAD_REG_WEIGHT * head_res_loss +
                                           L.SIZE_REG_WEIGHT * size_res_loss +
                                           L.CORNER_LOSS_WEIGHT * corners_loss)
    with torch.no_grad():
        cls_prec = accuracy(cls_probs, cls_label.view(-1), ignore=-1)
        head_prec = accuracy(h_pr, h_cls.view(-1))
        size_prec = accuracy(s_pr, size_class.view(-1))
        if getattr(model, "gpu_iou_metrics", True):
            # det_base.py:488-500 with the boxes kept on the device (fcn_rbbox_iou_3d_pair instead of the
            # CPU Boost call on `.cpu().numpy()` copies): PREDICTED class labels, as the reference
            h_lab, s_lab = torch.argmax(h_pr, -1), torch.argmax(s_pr, -1)
            c_metric = box_corners(center_preds, angle_decode(h_res, h_lab, nb), size_decode(s_res, mean_size, s_lab))
            iou2d, iou3d, iou3d_gt = (v.type_as(cls_prec) for v in _iou_metrics(c_metric, c_gt, cfg.IOU_THRESH))
        else:   # explicit opt-out (model.gpu_iou_metrics = False): NaN placeholders, no kernel launch
            iou2d = iou3d = iou3d_gt = torch.tensor(float("nan")).type_as(cls_prec)
    losses = {"total_loss": loss, "cls_loss": cls_loss, "center_loss": center_loss,
              "head_cls_loss": head_cls_loss, "head_res_loss": head_res_loss,
              "size_cls_loss": size_cls_loss, "size_res_loss": size_res_loss,
              "corners_loss": corners_loss}
    metrics = {"cls_acc": cls_prec, "head_acc": head_prec, "size_acc": size_prec,
               "IoU_2D": iou2d, "IoU_3D": iou3d, "IoU_" + str(cfg.IOU_THRESH): iou3d_gt}
    return losses, metrics


class FusedLoss:
    """Losses, metrics and d(total_loss)/d(logits) by the fused kernels of csrc/loss.cu (``fcn_det_loss``): three
    tiny launches instead of ~300 PyTorch ops + their autograd backward.  Its settings (``validate.set_loss_settings``)
    and the names of its 14 values (``keys``, ``validate.state_keys``) are read once, at construction.
    ``deterministic``: ``fcn_det_loss_deterministic``, whose 16 outputs are bit-reproducible."""

    def __init__(self, model, B, T2, out_size, device, deterministic=False):
        import ctypes as C

        from . import _lib
        from .validate import loss_weights, set_loss_settings, state_keys
        self._C, self._lib = C, _lib
        f32 = torch.float32
        N = B * T2
        self.dcls = torch.zeros((N, 2), dtype=f32, device=device)
        self.dreg = torch.zeros((N, out_size), dtype=f32, device=device)
        self.out = torch.zeros(16, dtype=f32, device=device)
        self.deterministic = bool(deterministic)
        n_scratch = int(_lib.load().fcn_det_loss_deterministic_scratch_floats(N)) if self.deterministic else 16
        if n_scratch <= 0:
            raise ValueError("FusedLoss: %d rows are outside the deterministic loss's range [1, 2^24]" % N)
        self.scratch = torch.zeros(n_scratch, dtype=f32, device=device)
        self.mean_size = torch.from_numpy(np.asarray(model.mean_size_array)).to(device=device, dtype=f32).contiguous()
        a = _lib.LossArgs()
        a.B, a.T2 = B, T2
        set_loss_settings(a, model, loss_weights())
        assert out_size == 3 + 2 * a.NH + 4 * a.NS
        a.mean_size, a.dcls, a.dreg = self.mean_size.data_ptr(), self.dcls.data_ptr(), self.dreg.data_ptr()
        a.out, a.scratch = self.out.data_ptr(), self.scratch.data_ptr()
        self.args = a
        self.keys = state_keys()

    def run(self, cls, reg, center_ref2, data):
        """-> (losses, metrics, dcls, dreg); 0-dim views of one result block, overwritten by the next call."""
        a = self.args
        keep = [cls.contiguous(), reg.contiguous(), center_ref2.contiguous(), data["cls_label"].contiguous(),
                data["size_class"].contiguous(), data["box3d_center"].contiguous(),
                data["box3d_heading"].contiguous(), data["box3d_size"].contiguous()]
        assert keep[3].dtype == torch.int64 and keep[4].dtype == torch.int64
        (a.cls, a.reg, a.center_ref2, a.cls_label, a.size_class, a.box3d_center, a.box3d_heading,
         a.box3d_size) = [t.data_ptr() for t in keep]
        self._keep = keep
        self._lib.call("fcn_det_loss_deterministic" if self.deterministic else "fcn_det_loss", self._C.byref(a),
                       torch.cuda.current_stream().cuda_stream)
        o = self.out                                   # the eight losses, then the six metrics
        losses = {k: o[i] for i, k in enumerate(self.keys[:8])}
        metrics = {k: o[i] for i, k in enumerate(self.keys[8:], 8)}
        return losses, metrics, self.dcls, self.dreg
