"""Device-side training batches - what the reference's ``ProviderDataset.__getitem__`` + collate hand to the training
step, computed on the GPU from a dataset that stays resident in HBM (C ABI section 11, csrc/train_inputs.cu).

    tb = TrainBatchBuilder.from_dataset(ds, "refine", strides=cfg.DATA.STRIDE, npoints=cfg.DATA.NUM_SAMPLES)
    for idx in torch.utils.data.BatchSampler(RandomSampler(ds), cfg.TRAIN.BATCH_SIZE, drop_last=True):
        data = tb.build(idx, tb.draw(idx))          # dict of CUDA tensors, overwritten by the next build()
        train_step.step(data)

kind="det"     datasets/provider_sample.py, train branch (:133-270), default_collate
kind="refine"  datasets/provider_sample_refine.py, train branch (:174-316) or, with labels=False, the
               from_rgb_detection branch (:228-248); collate_fn (:388-419) edge-pads center_ref* / cls_label to the
               batch's largest T per scale.
kind="sunrgbd" datasets/provider_sample_sunrgbd.py, train branch (:116-263; random_flip = random_shift = False is the
               val split) or, with labels=False, the from_rgb_detection branch (:165-186); default_collate.  Exactly
               5 strides (the reference unpacks s1..s5), 10 classes, max depth 8 (cfgs/det_sample_sunrgbd.yaml).

``draw(index)`` replays the np.random calls the reference's ``__getitem__`` makes, item after item (choice, then
random() when flipping, then randn() when shifting, then for SUN-RGBD the height shift's random()), so a seeded run
draws what a ``num_workers=0`` loader over the same indices would.  Nothing random runs on the device.  Only cfg.DATA.RTC = True, WITH_EXTRA_FEAT = False (every reference
cfg) is supported.

To capture the kernel in a CUDA graph, capture ``launch()``; before each replay ``upload(index, draws)`` the next batch
(same B) into the builder's fixed device buffers, then read ``outputs()``."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

KITTI_CLASSES = ("Car", "Pedestrian", "Cyclist")
SUNRGBD_CLASSES = ("bathtub", "bed", "bookshelf", "chair", "desk", "dresser", "night_stand", "sofa", "table", "toilet")
_KINDS = {"det": _lib.TRAIN_DET, "refine": _lib.TRAIN_REFINE, "sunrgbd": _lib.TRAIN_SUNRGBD}
_MAX_DEPTH = {"det": 70.0, "refine": 70.0, "sunrgbd": 8.0}      # cfg.DATA.MAX_DEPTH of the reference cfgs
_F32, _I64 = torch.float32, torch.int64


def rotate_pc_along_y(pc, rot_angle):
    """datasets/data_utils.py:7-21, the same numpy expression (float64 rotation through np.dot)."""
    cosval, sinval = np.cos(rot_angle), np.sin(rot_angle)
    rotmat = np.array([[cosval, -sinval], [sinval, cosval]])
    pc = pc.copy()
    pc[:, [0, 2]] = np.dot(pc[:, [0, 2]], np.transpose(rotmat))
    return pc


def compute_box_3d(center, dimension, angle):
    """datasets/data_utils.py:44-70."""
    cx, cy, cz = center
    l, w, h = dimension
    c, s = np.cos(angle), np.sin(angle)
    R = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    x_corners = [l / 2, l / 2, -l / 2, -l / 2, l / 2, l / 2, -l / 2, -l / 2]
    y_corners = [h / 2, h / 2, h / 2, h / 2, -h / 2, -h / 2, -h / 2, -h / 2]
    z_corners = [w / 2, -w / 2, -w / 2, w / 2, w / 2, -w / 2, -w / 2, w / 2]
    corners_3d = np.dot(R, np.vstack([x_corners, y_corners, z_corners]))
    corners_3d[0, :] = corners_3d[0, :] + cx
    corners_3d[1, :] = corners_3d[1, :] + cy
    corners_3d[2, :] = corners_3d[2, :] + cz
    return np.transpose(corners_3d, (1, 0))


def refine_ref_line(pred_box3d, pred_box3d_size, pred_box3d_angle, strides):
    """The per-frustum constants of provider_sample_refine.py generate_ref (:336-385) for the centre-view predicted box
    (:217-226): -> (front-face mean c1 (3), c2 - c1 (3), arange start z1, [arange step per scale], [T per scale])."""
    center = (pred_box3d[0, :] + pred_box3d[6, :]) / 2
    c_rot = rotate_pc_along_y((center - center)[np.newaxis, :], pred_box3d_angle).squeeze(0)
    box = compute_box_3d(c_rot, pred_box3d_size, pred_box3d_angle - pred_box3d_angle)
    cz = ((box[0, :] + box[6, :]) / 2)[2]
    z1, z2 = np.min(box[:, 2], 0), np.max(box[:, 2], 0)
    c1, c2 = np.mean(box[box[:, 2] < cz], 0), np.mean(box[box[:, 2] > cz], 0)
    steps = [(z1 + s) - z1 for s in strides]                       # numpy's arange fills start + i * this
    Ts = [len(np.arange(z1, z2, s)) for s in strides]
    return c1, c2 - c1, z1, steps, Ts


def draw_items(counts, index, npoints, random_flip, random_shift, rng=np.random, height=False):
    """The np.random calls of ProviderDataset.__getitem__ for the items `index` (frustum point counts `counts`), in the
    reference's order -> dict(choice (B, npoints), flip_u (B), shift_n (B)); disabled draws read 0.  height=True (the
    SUN-RGBD provider) adds height_u (B): the random() it draws after randn() when shifting (:231)."""
    B = len(index)
    choice = np.empty((B, npoints), dtype=np.int64)
    flip_u, shift_n, height_u = np.zeros(B), np.zeros(B), np.zeros(B)
    for b, i in enumerate(index):
        n = int(counts[i])
        choice[b] = rng.choice(n, npoints, n < npoints)                              # :166 / :207
        if random_flip:
            flip_u[b] = rng.random()                                                 # :227 / :270
        if random_shift:
            shift_n[b] = rng.randn()                                                 # :241 / :284
            if height:
                height_u[b] = rng.random()
    out = {"choice": choice, "flip_u": flip_u, "shift_n": shift_n}
    if height:
        out["height_u"] = height_u
    return out


def frustum_table(kind, strides, max_depth, labels, classes, type_list, label_list=None, box3d_list=None,
                  heading_list=None, size_list=None, frustum_angle_list=None, box2d_list=None, calib_list=None,
                  prob_list=None, pred_box3d_list=None, pred_box3d_size_list=None, pred_box3d_angle_list=None,
                  calib_K_list=None, calib_R_list=None):
    """The per-frustum constants (fcn_train_frustum records) of the provider's lists, computed once in float64 with
    the reference's own numpy expressions."""
    classes = list(classes)
    F, S = len(type_list), len(strides)
    fr = np.zeros(F, dtype=np.dtype(_lib.TrainFrustum))
    det_T = [len(np.arange(0, max_depth, s)) for s in strides]
    for i in range(F):
        r = fr[i]
        r["cls_index"] = classes.index(type_list[i])
        if kind == "det":
            rot = np.pi / 2.0 + frustum_angle_list[i]                           # provider_sample.py:329-332
            r["rot"], r["cs"], r["sn"] = rot, np.cos(rot), np.sin(rot)
            r["box2d"] = np.asarray(box2d_list[i], dtype=np.float64).reshape(4)
            r["P"] = np.asarray(calib_list[i]["P2"], dtype=np.float64).reshape(12)
            b3 = box3d_list[i]
            r["center"] = rotate_pc_along_y(np.expand_dims((b3[0, :] + b3[6, :]) / 2.0, 0), rot).squeeze()
            r["heading"] = heading_list[i] - rot
            r["T"][:S] = det_T
        elif kind == "sunrgbd":
            rot = np.pi / 2.0 + frustum_angle_list[i]                           # provider_sample_sunrgbd.py:328-331
            r["rot"], r["cs"], r["sn"] = rot, np.cos(rot), np.sin(rot)
            box = box2d_list[i]
            r["cx"], r["cy"] = (box[0] + box[2]) / 2., (box[1] + box[3]) / 2.  # :294, in box2d's dtype (float32)
            r["K"] = np.asarray(calib_K_list[i], dtype=np.float64).reshape(9)
            r["Rtilt"] = np.asarray(calib_R_list[i], dtype=np.float64).reshape(9)
            if labels:
                b3 = box3d_list[i]
                r["center"] = rotate_pc_along_y(np.expand_dims((b3[0, :] + b3[6, :]) / 2.0, 0), rot).squeeze()
                r["heading"] = heading_list[i] - rot
            else:
                r["rgb_prob"] = prob_list[i]
            r["T"][:S] = det_T
        else:
            pb = pred_box3d_list[i]
            pa = pred_box3d_angle_list[i]
            pc = (pb[0, :] + pb[6, :]) / 2
            r["rot"], r["cs"], r["sn"], r["ref_center"] = pa, np.cos(pa), np.sin(pa), pc
            c1, delta, z1, steps, Ts = refine_ref_line(pb, pred_box3d_size_list[i], pa, strides)
            if min(Ts) < 1 or delta[2] == 0:
                raise ValueError("frustum %d: degenerate predicted box (size %s)" % (i, pred_box3d_size_list[i]))
            r["line0"], r["line_delta"], r["z_start"] = c1, delta, z1
            r["z_step"][:S], r["T"][:S] = steps, Ts
            if labels:                                                     # provider_sample_refine.py:141-147
                b3 = box3d_list[i]
                c = rotate_pc_along_y(((b3[0, :] + b3[6, :]) / 2 - pc)[np.newaxis, :], pa).squeeze(0)
                r["center"], r["heading"] = c, heading_list[i] - pa
            else:
                r["rgb_prob"] = prob_list[i]
        if labels:
            l, w, h = size_list[i]
            r["size"] = size_list[i]
            r["dist"] = np.sqrt(np.sum(l ** 2 + w ** 2))
    return fr


class TrainBatchBuilder:
    def __init__(self, kind, strides, npoints, max_depth=None, num_classes=None, random_flip=True, random_shift=True,
                 labels=True, one_hot=True, rtc=True, with_extra_feat=False, device="cuda"):
        """max_depth / num_classes default to the kind's reference cfg (70 / 3 for KITTI, 8 / 10 for SUN-RGBD)."""
        if kind not in _KINDS:
            raise ValueError("kind must be 'det', 'refine' or 'sunrgbd', got %r" % (kind,))
        if kind == "sunrgbd" and len(strides) != 5:
            raise ValueError("the SUN-RGBD provider takes exactly 5 strides (s1, ..., s5 = cfg.DATA.STRIDE), got %d"
                             % len(strides))
        if not rtc or with_extra_feat:
            raise ValueError("only cfg.DATA.RTC = True and WITH_EXTRA_FEAT = False are supported (every reference cfg)")
        if kind == "det" and not labels:
            raise ValueError("the detection provider's from_rgb_detection branch is input_builder.FrustumBatchBuilder")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("TrainBatchBuilder builds on a CUDA device; there is no CPU path")
        self.kind, self.labels = kind, bool(labels)
        self.strides = [float(s) for s in strides]
        if not 2 <= len(self.strides) <= _lib.MAX_SCALES:
            raise ValueError("need 2..%d strides" % _lib.MAX_SCALES)
        if num_classes is None:
            num_classes = len(SUNRGBD_CLASSES if kind == "sunrgbd" else KITTI_CLASSES)
        self.N, self.V = int(npoints), int(num_classes)
        self.max_depth = float(_MAX_DEPTH[kind] if max_depth is None else max_depth)
        self.random_flip = bool(random_flip) and self.labels
        self.random_shift = bool(random_shift) and self.labels
        self.one_hot = bool(one_hot)
        self._has_seg = kind == "det" or (kind == "sunrgbd" and self.labels)
        self.num_frustums = 0
        self.B_cap = 0
        self._B = 0

    # ------------------------------------------------------------------ dataset (once)
    @classmethod
    def from_dataset(cls, ds, kind, strides, npoints=None, max_depth=None, classes=None, **kw):
        """Reads the lists off a reference ``ProviderDataset`` instance by attribute name (the reference itself need
        not be importable).  npoints / random_flip / random_shift / one_hot / labels default to the instance's;
        classes to its category_info, else the dataset's class list (the SUN-RGBD provider has no category_info)."""
        kw.setdefault("random_flip", getattr(ds, "random_flip", False))
        kw.setdefault("random_shift", getattr(ds, "random_shift", False))
        kw.setdefault("one_hot", getattr(ds, "one_hot", True))
        kw.setdefault("labels", not getattr(ds, "from_rgb_detection", False))
        if classes is None:
            classes = ds.category_info.CLASSES if hasattr(ds, "category_info") else \
                (SUNRGBD_CLASSES if kind == "sunrgbd" else KITTI_CLASSES)
        classes = list(classes)
        kw.setdefault("num_classes", len(classes))
        tb = cls(kind, strides, ds.npoints if npoints is None else npoints, max_depth=max_depth, **kw)
        names = ("label_list", "box3d_list", "heading_list", "size_list", "frustum_angle_list", "box2d_list",
                 "calib_list", "prob_list", "pred_box3d_list", "pred_box3d_size_list", "pred_box3d_angle_list",
                 "calib_K_list", "calib_R_list")
        tb.set_dataset(ds.input_list, ds.type_list, classes, **{n: getattr(ds, n, None) for n in names})
        return tb

    def set_dataset(self, input_list, type_list, classes=None, label_list=None, box3d_list=None,
                    heading_list=None, size_list=None, frustum_angle_list=None, box2d_list=None, calib_list=None,
                    prob_list=None, pred_box3d_list=None, pred_box3d_size_list=None, pred_box3d_angle_list=None,
                    calib_K_list=None, calib_R_list=None):
        """Copies the provider's lists to the device once; per-frustum constants are computed here in float64 with the
        reference's own numpy expressions.  classes defaults to the kind's dataset (KITTI, or SUN-RGBD's 10)."""
        if classes is None:
            classes = SUNRGBD_CLASSES if self.kind == "sunrgbd" else KITTI_CLASSES
        F = len(input_list)
        if F == 0:
            raise ValueError("empty dataset")
        counts = np.asarray([int(np.shape(p)[0]) for p in input_list], dtype=np.int64)
        if (counts < 1).any():
            raise ValueError("frustum %d has no points" % int(np.argmax(counts < 1)))
        dtypes = {np.asarray(p).dtype for p in input_list}
        if not dtypes <= {np.dtype(np.float32), np.dtype(np.float64)} or len(dtypes) != 1:
            raise ValueError("input_list must be all float32 or all float64, got %s" % sorted(map(str, dtypes)))
        self.points_f64 = dtypes == {np.dtype(np.float64)}
        need = {"det": ["label_list", "box3d_list", "heading_list", "size_list", "frustum_angle_list", "box2d_list",
                        "calib_list"],
                "refine": ["pred_box3d_list", "pred_box3d_size_list", "pred_box3d_angle_list"] +
                          (["box3d_list", "heading_list", "size_list"] if self.labels else ["prob_list"]),
                "sunrgbd": ["frustum_angle_list", "box2d_list", "calib_K_list", "calib_R_list"] +
                           (["label_list", "box3d_list", "heading_list", "size_list"] if self.labels else
                            ["prob_list"])}[self.kind]
        lists = dict(label_list=label_list, box3d_list=box3d_list, heading_list=heading_list, size_list=size_list,
                     frustum_angle_list=frustum_angle_list, box2d_list=box2d_list, calib_list=calib_list,
                     prob_list=prob_list, pred_box3d_list=pred_box3d_list, pred_box3d_size_list=pred_box3d_size_list,
                     pred_box3d_angle_list=pred_box3d_angle_list, calib_K_list=calib_K_list,
                     calib_R_list=calib_R_list)
        for n in need:
            if lists[n] is None or len(lists[n]) != F:
                raise ValueError("kind=%r needs %s with one entry per frustum" % (self.kind, n))
        fr = frustum_table(self.kind, self.strides, self.max_depth, self.labels, classes, type_list, **lists)
        pts = np.concatenate([np.asarray(p)[:, :3] for p in input_list]).astype(np.float64 if self.points_f64 else
                                                                                  np.float32)
        self._install(fr, counts, torch.from_numpy(np.ascontiguousarray(pts)).to(self.device), label_list)

    @classmethod
    def from_frustums(cls, fr, kind, strides, npoints, classes=None, **kw):
        """The dataset of a refine_extract.RefineFrustums (kind="refine"), a gt_extract.GtFrustums (kind="det") or a
        sunrgbd_extract.SunrgbdFrustums (kind="sunrgbd"): its points stay on the device (the x, y, z columns are
        copied there; uint8 labels are cast to the int32 seg labels there), the per-frustum constants come from its
        host lists.  The same batches as set_dataset on fr's lists.  labels defaults to whether fr has ground truth;
        classes to the kind's dataset."""
        from .gt_extract import GtFrustums
        from .sunrgbd_extract import SunrgbdFrustums
        if isinstance(fr, SunrgbdFrustums):
            if kind != "sunrgbd":
                raise ValueError("from_frustums builds the SUN-RGBD provider's batches (kind='sunrgbd') from "
                                 "SunrgbdFrustums, got %r" % kind)
            return cls._from_sunrgbd(fr, strides, npoints, classes, **kw)
        gt = isinstance(fr, GtFrustums)
        if gt and kind != "det":
            raise ValueError("from_frustums builds the detection provider's batches (kind='det') from GtFrustums, "
                             "got %r" % kind)
        if not gt and kind != "refine":
            raise ValueError("from_frustums builds the refinement provider's batches (kind='refine'), got %r" % kind)
        kw.setdefault("labels", fr.has_labels)
        tb = cls(kind, strides, npoints, **kw)
        if tb.labels and not fr.has_labels:
            raise ValueError("labels=True needs frustums with ground truth (from_ground_truth or "
                             "from_matched_detections)")
        if len(fr) == 0:
            raise ValueError("empty dataset")
        if fr.points.device.type != "cuda" or (tb.device.index is not None and fr.points.device != tb.device):
            raise RuntimeError("the frustums live on %s, the builder on %s" % (fr.points.device, tb.device))
        counts = np.asarray(fr.counts, dtype=np.int64)
        fr.wait()                          # the points and labels were written on the extraction's stream
        tb.points_f64 = False
        d_seg = fr.label.to(torch.int32) if gt else None
        rec = getattr(fr, "frustum_records", None)
        if rec is not None and fr.record_strides == tb.strides and fr.record_labels == tb.labels and \
                fr.record_classes is not None and (classes is None or tuple(classes) == fr.record_classes):
            # the extractor's device records (refine_extract.CollectedRefineFrustums): one read for T and the flags
            S = len(tb.strides)
            words = fr.record_words.cpu().numpy()
            if words[:, S].any():
                i = int(np.argmax(words[:, S]))
                raise ValueError("frustum %d: degenerate predicted box (size %s)" % (i, fr.pred_box3d_size_list[i]))
            tb._install_device(words[:, :S].astype(np.int64), rec, counts, fr.points[:, :3].contiguous(), None, d_seg)
            return tb
        names = ("box3d_list", "heading_list", "size_list") + (
            ("frustum_angle_list", "box2d_list", "calib_list") if gt else
            ("prob_list", "pred_box3d_list", "pred_box3d_size_list", "pred_box3d_angle_list"))
        table = frustum_table(kind, tb.strides, tb.max_depth, tb.labels,
                              KITTI_CLASSES if classes is None else classes, fr.type_list,
                              **{n: getattr(fr, n) for n in names})
        tb._install(table, counts, fr.points[:, :3].contiguous(), None, d_seg)
        return tb

    @classmethod
    def _from_sunrgbd(cls, fr, strides, npoints, classes, **kw):
        kw.setdefault("labels", fr.has_labels)
        tb = cls("sunrgbd", strides, npoints, **kw)
        if tb.labels and not fr.has_labels:
            raise ValueError("labels=True needs frustums with ground truth (from_ground_truth)")
        if len(fr) == 0:
            raise ValueError("empty dataset")
        if fr.points.device.type != "cuda" or (tb.device.index is not None and fr.points.device != tb.device):
            raise RuntimeError("the frustums live on %s, the builder on %s" % (fr.points.device, tb.device))
        fr.wait()                          # the points and labels were written on the extraction's stream
        names = ("frustum_angle_list", "box2d_list", "calib_K_list", "calib_R_list") + (
            ("box3d_list", "heading_list", "size_list") if tb.labels else ("prob_list",))
        table = frustum_table("sunrgbd", tb.strides, tb.max_depth, tb.labels,
                              SUNRGBD_CLASSES if classes is None else classes, fr.type_list,
                              **{n: getattr(fr, n) for n in names})
        tb.points_f64 = False
        tb._install(table, np.asarray(fr.counts, dtype=np.int64), fr.points[:, :3].contiguous(), None,
                    fr.label.to(torch.int32) if tb.labels else None)
        return tb

    def _install(self, fr, counts, d_points, label_list, d_seg=None):
        self._install_device(fr["T"][:, :len(self.strides)].astype(np.int64),
                             torch.from_numpy(fr.view(np.uint8)).to(self.device), counts, d_points, label_list, d_seg)

    def _install_device(self, T_of, d_frustums, counts, d_points, label_list, d_seg=None):
        """T_of (F, S) host sections per scale, d_frustums the fcn_train_frustum records already on the device."""
        self.T_of = T_of
        self.counts = counts
        dev = self.device
        self.d_points = d_points
        self.d_offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)).to(dev)
        self.d_frustums = d_frustums
        self.d_seg = d_seg
        if self._has_seg and d_seg is None:
            seg = np.concatenate([np.asarray(s).astype(np.int64) for s in label_list])  # provider_sample.py:206
            if len(seg) != len(d_points) or (np.abs(seg) >= 2 ** 31).any():
                raise ValueError("label_list must hold one int32-range label per point")
            self.d_seg = torch.from_numpy(seg.astype(np.int32)).to(dev)
        self.num_frustums = len(counts)
        self.B_cap = 0                     # output buffers follow the dataset (T capacity)

    # ------------------------------------------------------------------ per step
    def draw(self, index, rng=np.random):
        """The reference's np.random calls for these items, in its order -> dict(choice, flip_u, shift_n).
        ``rng``: the np.random module (the reference's global stream) or a np.random.RandomState."""
        return draw_items(self.counts, self._index(index), self.N, self.random_flip, self.random_shift, rng,
                          height=self.kind == "sunrgbd")

    def _index(self, index):
        if isinstance(index, torch.Tensor):
            if index.device.type != "cpu":
                raise TypeError("index must be on the host (it is validated and sizes the collate there)")
            index = index.numpy()
        index = np.asarray(index).reshape(-1)
        if self.num_frustums == 0:
            raise RuntimeError("set_dataset() first")
        if len(index) == 0 or not np.issubdtype(index.dtype, np.integer):
            raise ValueError("index must be a non-empty integer array")
        if index.min() < 0 or index.max() >= self.num_frustums:
            raise IndexError("index out of range [0, %d)" % self.num_frustums)
        return index.astype(np.int64)

    def _alloc(self, B):
        dev, S = self.device, len(self.strides)
        self.B_cap = B
        self.T_cap = self.T_of.max(0)
        self._flat = {"point_cloud": torch.empty(B * 3 * self.N, dtype=_F32, device=dev),
                      "rot_angle": torch.empty(B, dtype=_F32, device=dev)}
        for s in range(S):
            self._flat["center_ref%d" % (s + 1)] = torch.empty(B * 3 * int(self.T_cap[s]), dtype=_F32, device=dev)
        if self.one_hot:
            self._flat["one_hot"] = torch.empty(B * self.V, dtype=_F32, device=dev)
        if self.labels:
            self._flat["cls_label"] = torch.empty(B * int(self.T_cap[1]), dtype=_I64, device=dev)
            for k in ("box3d_center", "box3d_size"):
                self._flat[k] = torch.empty(B * 3, dtype=_F32, device=dev)
            self._flat["box3d_heading"] = torch.empty(B, dtype=_F32, device=dev)
            self._flat["size_class"] = torch.empty(B, dtype=_I64, device=dev)
        if self._has_seg:
            self._flat["seg_label"] = torch.empty(B * self.N, dtype=_I64, device=dev)
        if self.kind == "refine":
            self._flat["ref_center"] = torch.empty(B * 3, dtype=_F32, device=dev)
        if not self.labels:
            self._flat["rgb_prob"] = torch.empty(B, dtype=_F32, device=dev)
        # draws: one packed host staging buffer -> one H2D copy per step into fixed device buffers
        # [flip_u f64 | shift_n f64 | height_u f64 | index i32 | choice i32]
        self._nbytes = 24 * B + 4 * B + 4 * B * self.N
        self._host = np.zeros(self._nbytes, dtype=np.uint8)
        self._dev = torch.empty(self._nbytes, dtype=torch.uint8, device=dev)
        base = self._dev.data_ptr()
        a = _lib.TrainInputArgs()
        a.kind = _KINDS[self.kind]
        a.labels, a.rtc, a.extra_feat = int(self.labels), 1, 0
        a.random_flip, a.random_shift = int(self.random_flip), int(self.random_shift)
        a.B, a.N, a.num_scales, a.num_classes, a.num_frustums = B, self.N, S, self.V, self.num_frustums
        a.points_f64 = int(self.points_f64)
        for s in range(S):
            a.stride[s] = self.strides[s]
            a.centers[s] = self._flat["center_ref%d" % (s + 1)].data_ptr()
        a.max_depth = self.max_depth
        a.points, a.point_offsets, a.frustums = self.d_points.data_ptr(), self.d_offsets.data_ptr(), \
            self.d_frustums.data_ptr()
        a.seg = None if self.d_seg is None else self.d_seg.data_ptr()
        a.flip_u, a.shift_n, a.height_u = base, base + 8 * B, base + 16 * B
        a.index, a.choice = base + 24 * B, base + 28 * B
        for k in ("point_cloud", "cls_label", "seg_label", "box3d_center", "box3d_heading", "box3d_size", "size_class",
                  "rot_angle", "one_hot", "ref_center", "rgb_prob"):
            setattr(a, k, self._flat[k].data_ptr() if k in self._flat else None)
        self.args = a

    def upload(self, index, draws):
        """Validates the batch on the host and copies index + draws to the builder's device buffers (one copy)."""
        index = self._index(index)
        B = len(index)
        choice = np.asarray(draws["choice"])
        if choice.shape != (B, self.N):
            raise ValueError("choice must be (%d, %d), got %s" % (B, self.N, choice.shape))
        if choice.min() < 0 or (choice >= self.counts[index][:, None]).any():
            raise IndexError("choice holds an index past its frustum's point count")
        if self.B_cap != B:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("upload() of a new batch size while a CUDA graph is being captured")
            self._alloc(B)
        h = self._host
        h[:8 * B].view(np.float64)[:] = np.asarray(draws.get("flip_u", np.zeros(B)), dtype=np.float64).reshape(B)
        h[8 * B: 16 * B].view(np.float64)[:] = np.asarray(draws.get("shift_n", np.zeros(B)),
                                                          dtype=np.float64).reshape(B)
        h[16 * B: 24 * B].view(np.float64)[:] = np.asarray(draws.get("height_u", np.zeros(B)),
                                                           dtype=np.float64).reshape(B)
        h[24 * B: 28 * B].view(np.int32)[:] = index
        h[28 * B:].view(np.int32)[:] = choice.reshape(-1)
        self._dev.copy_(torch.from_numpy(h), non_blocking=True)
        self._B, self._pad = B, self.T_of[index].max(0)
        return B

    def launch(self):
        """The kernel alone on the current stream (what a CUDA graph captures)."""
        with torch.cuda.device(self.device):
            _lib.call("fcn_build_train_inputs", C.byref(self.args), torch.cuda.current_stream(self.device).cuda_stream)

    def outputs(self):
        """Views of the builder's buffers for the last uploaded batch, with the reference collate's shapes."""
        B, N, P = self._B, self.N, [int(p) for p in self._pad]
        f = self._flat
        out = {"point_cloud": f["point_cloud"].view(B, 3, N), "rot_angle": f["rot_angle"].view(B, 1)}
        for s, p in enumerate(P):
            out["center_ref%d" % (s + 1)] = f["center_ref%d" % (s + 1)][: B * 3 * p].view(B, 3, p)
        if self.labels:
            out["cls_label"] = f["cls_label"][: B * P[1]].view(B, P[1])
            out["box3d_center"] = f["box3d_center"].view(B, 3)
            out["box3d_heading"] = f["box3d_heading"].view(B, 1)
            out["box3d_size"] = f["box3d_size"].view(B, 3)
            out["size_class"] = f["size_class"].view(B, 1)
        if "seg_label" in f:
            out["seg_label"] = f["seg_label"].view(B, N)
        if "ref_center" in f:
            out["ref_center"] = f["ref_center"].view(B, 3)
        if "rgb_prob" in f:
            out["rgb_prob"] = f["rgb_prob"].view(B, 1)
        if self.one_hot:
            out["one_hot"] = f["one_hot"].view(B, self.V)
        return out

    def build(self, index, draws):
        """index (B,) dataset indices (host), draws = draw(index) -> dict of CUDA tensors (overwritten by the next
        call), the keys, shapes and dtypes of the reference collate's batch."""
        self.upload(index, draws)
        self.launch()
        return self.outputs()
