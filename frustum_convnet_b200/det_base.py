"""Drop-in for /root/reference/models/det_base.py (KITTI, 4 scales) on the H100 hot path.

Exports the same classes with the same constructor / forward signatures and the same
parameter & buffer names, so reference checkpoints load unchanged and the reference's drivers
can select this file through ``cfg.MODEL.FILE`` (train/train_net_det.py:293-304,
utils/utils.py:12-25):

  QueryDepthPoint(dis_z, nsample)                                   ops/.../query_depth_point.py:47-54
  PointNetModule(Infea, mlp, dist, nsample, use_xyz, use_feature)   det_base.py:35-103
  PointNetFeat(input_channel=3, num_vec=0)                          det_base.py:107-159
  ConvFeatNet(i_c=128, num_vec=3)                                   det_base.py:163-224
  PointNetDet(input_channel=3, num_vec=0, num_classes=2)            det_base.py:228-525

In eval mode every forward runs the hand-written sm_90a kernels of libfrustum_b200.so through
``FrustumEngine`` (BN folded into a private weight pack; the state dict is never modified).
In training mode (batch-statistics BN, autograd) the grouping still runs on the library
(``QueryDepthPoint``) while conv/BN/loss arithmetic is composed from torch CUDA ops — see
``frustum_convnet_b200/train_path.py``; hand-written backward kernels are listed as next in
DESIGN.md.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.nn as nn

# The reference selects the model file with ``cfg.MODEL.FILE`` and loads it as a TOP-LEVEL module
# (utils/utils.py:12-25: ``sys.path.append(folder); importlib.import_module(file[:-3])``), so this file
# must import without a parent package: absolute imports + a bootstrap that makes the package reachable.
_PKG_PARENT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if _PKG_PARENT not in sys.path:
    sys.path.insert(0, _PKG_PARENT)

from frustum_convnet_b200.config import ARCH_KITTI, DATASET_INFO, ArchSpec, get_cfg  # noqa: E402
from frustum_convnet_b200.engine import FrustumEngine  # noqa: E402
from frustum_convnet_b200.query_depth_point import QueryDepthPoint  # noqa: E402

__all__ = ["QueryDepthPoint", "PointNetModule", "PointNetFeat", "ConvFeatNet", "PointNetDet"]


def _block2d(ci, co):
    return nn.Sequential(nn.Conv2d(ci, co, 1, bias=False), nn.BatchNorm2d(co), nn.ReLU(True))


def _block1d(ci, co, k, s=1, p=0):
    return nn.Sequential(nn.Conv1d(ci, co, k, s, p, bias=False), nn.BatchNorm1d(co), nn.ReLU(True))


def _upblock1d(ci, co, k, s):
    return nn.Sequential(nn.ConvTranspose1d(ci, co, k, s, 0, bias=False), nn.BatchNorm1d(co), nn.ReLU(True))


def _init_kaiming(module):
    for m in module.modules():
        if isinstance(m, (nn.Conv1d, nn.Conv2d, nn.ConvTranspose1d)):
            nn.init.kaiming_normal_(m.weight.data, mode="fan_in")
            if m.bias is not None:
                m.bias.data.zero_()
        elif isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d)):
            m.weight.data.fill_(1)
            m.bias.data.zero_()


def default_precision() -> int:
    """Eval arithmetic of a drop-in module whose ``precision`` attribute was not set: ``FCN_PRECISION``
    (1 = TF32 wgmma tensor cores — the benchmarked configuration and what cuDNN itself computes for these
    convolutions by default; 0 = fp32 FMA everywhere)."""
    return int(os.environ.get("FCN_PRECISION", "1"))


def default_cuda_graph() -> bool:
    """``FCN_CUDA_GRAPH`` (default 1): replay one CUDA graph per input shape in PointNetDet.forward."""
    return os.environ.get("FCN_CUDA_GRAPH", "1") != "0"


class _EngineOwner(nn.Module):
    """Mixin: lazily (re)builds the kernel-ready weight pack when weights/device/mode change.

    Staleness rules (ADVICE r1): mode switches, device moves and every ``load_state_dict`` — also one issued
    on a parent/wrapper module, which reaches this module only through ``_load_from_state_dict`` — mark the
    pack dirty; in-place updates that go through autograd-visible tensors (optimizer steps, ``p.copy_()``)
    bump ``Tensor._version`` and are caught by a version scan on EVERY call (a cached tensor list makes
    the scan ~10 us).  Edits through ``.data`` (``p.data.copy_()``) bypass the version counter by
    construction: call ``refresh()`` after them."""

    _engine = None
    _engine_key = None
    _engine_dirty = True
    _tensor_cache = None
    _frozen = False
    precision = None  # None: default_precision(); 0: fp32 CUDA cores, 1: TF32 tensor cores for the dense layers

    def __init__(self):
        super().__init__()
        self.register_load_state_dict_post_hook(_mark_dirty_hook)

    def _engine_spec(self):  # -> (arch, num_vec, dataset, dists, num_bins, prefix)
        raise NotImplementedError

    def _tensors(self):
        if self._tensor_cache is None:
            self._tensor_cache = list(self.parameters()) + list(self.buffers())
        return self._tensor_cache

    def _param_version(self):
        return tuple([t._version for t in self._tensors()])

    def train(self, mode=True):
        self._engine_dirty = True
        return super().train(mode)

    def _apply(self, fn, *args, **kwargs):
        self._engine_dirty = True
        self._tensor_cache = None
        return super()._apply(fn, *args, **kwargs)

    def _load_from_state_dict(self, *args, **kwargs):
        self._engine_dirty = True
        return super()._load_from_state_dict(*args, **kwargs)

    def refresh(self):
        """Force a rebuild of the kernel-ready weight pack at the next eval forward."""
        self._engine_dirty = True
        self._tensor_cache = None

    def resolved_precision(self) -> int:
        return default_precision() if self.precision is None else int(self.precision)

    def freeze(self, frozen: bool = True):
        """Serving mode: the weights will not change behind the module's back, so the per-call version scan
        (~10 us of host time) is skipped; mode switches, device moves, load_state_dict and refresh() still rebuild."""
        self._frozen = bool(frozen)
        return self

    def engine(self) -> FrustumEngine:
        prec = self.resolved_precision()
        if self._engine is not None and not self._engine_dirty:
            if self._frozen and self._engine_key[1] == prec:
                return self._engine
            ver = self._param_version()
            if self._engine_key[1] == prec and self._engine_key[2] == ver:
                return self._engine
        if getattr(self, "_is_replica", False) or next(self.parameters(), None) is None:
            # nn.DataParallel replicas carry no parameters and share the source module's attributes
            # (test_net_det.py:404, train_net_det.py:308): the hot path is one process per GPU instead
            raise RuntimeError("frustum_convnet_b200 modules cannot run as nn.DataParallel replicas; launch one "
                               "process per GPU (torchrun) — see INTEGRATION.md, multi-GPU")
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("the frustum hot path runs on CUDA only (no CPU fallback); "
                               "move the module to an H100 with .cuda()")
        self._tensor_cache = None
        key = (dev, prec, self._param_version())
        if self._engine is None or self._engine_key != key or self._engine_dirty:
            arch, num_vec, dataset, dists, num_bins, prefix = self._engine_spec()
            sd = {prefix + k: v for k, v in self.state_dict().items()}
            self._engine = FrustumEngine(arch, num_vec, dataset, dists, num_bins, sd, dev, prec)
            self._engine_key = key
        self._engine_dirty = False
        return self._engine


def _mark_dirty_hook(module, incompatible_keys):
    module._engine_dirty = True


class PointNetModule(_EngineOwner):
    """Single-scale grouping + shared MLP; returns the masked, un-pooled (B, mlp[2], T, nsample)."""

    def __init__(self, Infea, mlp, dist, nsample, use_xyz=True, use_feature=True):
        super().__init__()
        self.dist, self.nsample, self.use_xyz = dist, nsample, use_xyz
        self.use_feature = Infea > 0
        self.mlp = tuple(mlp)
        self.query_depth_point = QueryDepthPoint(dist, nsample)
        cin = Infea + 3 if use_xyz else Infea
        self.conv1 = _block2d(cin, mlp[0])
        self.conv2 = _block2d(mlp[0], mlp[1])
        self.conv3 = _block2d(mlp[1], mlp[2])
        _init_kaiming(self)

    def _engine_spec(self):
        arch = ArchSpec("single", (self.nsample,), (self.mlp,), 0, 0)
        return arch, 0, "KITTI", (self.dist,), 12, "feat_net.pointnet1."

    def forward(self, pc, feat, new_pc=None):
        if self.training or self.use_feature or not self.use_xyz:
            from frustum_convnet_b200.train_path import pointnet_module_torch
            return pointnet_module_torch(self, pc, feat, new_pc)
        return self.engine().pointnet_module(0, pc.contiguous(), new_pc.contiguous())


class PointNetFeat(_EngineOwner):
    ARCH = ARCH_KITTI

    def __init__(self, input_channel=3, num_vec=0):
        super().__init__()
        self.num_vec = num_vec
        u = get_cfg().DATA.HEIGHT_HALF
        arch = self.ARCH
        assert len(u) == arch.num_scales
        self.dists = tuple(float(x) for x in u)
        for i in range(arch.num_scales):
            setattr(self, "pointnet%d" % (i + 1),
                    PointNetModule(input_channel - 3, list(arch.mlps[i]), u[i], arch.nsample[i],
                                   use_xyz=True, use_feature=True))

    def _engine_spec(self):
        return self.ARCH, self.num_vec, "KITTI", self.dists, 12, "feat_net."

    def forward(self, point_cloud, sample_pc, feat=None, one_hot_vec=None):
        if self.training or feat is not None or (one_hot_vec is None) != (self.num_vec == 0):
            from frustum_convnet_b200.train_path import pointnet_feat_torch
            return pointnet_feat_torch(self, point_cloud, sample_pc, feat, one_hot_vec)
        if one_hot_vec is not None:
            assert self.num_vec == one_hot_vec.shape[1]
        return self.engine().pointnet_feat(point_cloud.contiguous(), [c.contiguous() for c in sample_pc],
                                           None if one_hot_vec is None else one_hot_vec.contiguous())


class ConvFeatNet(_EngineOwner):
    ARCH = ARCH_KITTI

    def __init__(self, i_c=128, num_vec=3):
        super().__init__()
        self.num_vec = num_vec
        self.block1_conv1 = _block1d(i_c + num_vec, 128, 3, 1, 1)
        self.block2_conv1 = _block1d(128, 128, 3, 2, 1)
        self.block2_conv2 = _block1d(128, 128, 3, 1, 1)
        self.block2_merge = _block1d(128 + 128 + num_vec, 128, 1, 1)
        self.block3_conv1 = _block1d(128, 256, 3, 2, 1)
        self.block3_conv2 = _block1d(256, 256, 3, 1, 1)
        self.block3_merge = _block1d(256 + 256 + num_vec, 256, 1, 1)
        self.block4_conv1 = _block1d(256, 512, 3, 2, 1)
        self.block4_conv2 = _block1d(512, 512, 3, 1, 1)
        self.block4_merge = _block1d(512 + 512 + num_vec, 512, 1, 1)
        self.block2_deconv = _upblock1d(128, 256, 1, 1)
        self.block3_deconv = _upblock1d(256, 256, 2, 2)
        self.block4_deconv = _upblock1d(512, 256, 4, 4)
        _init_kaiming(self)

    def _engine_spec(self):
        return self.ARCH, self.num_vec, "KITTI", (0.0,) * self.ARCH.num_scales, 12, "conv_net."

    def forward(self, *xs):
        if self.training:
            from frustum_convnet_b200.train_path import conv_feat_net_torch
            return conv_feat_net_torch(self, xs)
        return self.engine().conv_feat_net([x.contiguous() for x in xs])


class PointNetDet(_EngineOwner):
    ARCH = ARCH_KITTI
    FEAT_CLS = PointNetFeat
    FCN_CLS = ConvFeatNet

    def __init__(self, input_channel=3, num_vec=0, num_classes=2):
        super().__init__()
        cfg = get_cfg()
        dataset_name = cfg.DATA.DATASET_NAME
        assert dataset_name in DATASET_INFO
        self.dataset_name = dataset_name
        self.category_info = DATASET_INFO[dataset_name]
        self.num_size_cluster = len(self.category_info.CLASSES)
        self.mean_size_array = self.category_info.MEAN_SIZE_ARRAY
        self.num_vec = num_vec
        self.feat_net = self.FEAT_CLS(input_channel, num_vec)
        self.conv_net = self.FCN_CLS(128, num_vec)
        self.num_classes = num_classes
        self.num_bins = cfg.DATA.NUM_HEADING_BIN
        output_size = 3 + self.num_bins * 2 + self.num_size_cluster * 4
        self.reg_out = nn.Conv1d(self.ARCH.reg_in, output_size, 1)
        self.cls_out = nn.Conv1d(self.ARCH.reg_in, 2, 1)
        self.relu = nn.ReLU(True)
        nn.init.kaiming_uniform_(self.cls_out.weight, mode="fan_in")
        nn.init.kaiming_uniform_(self.reg_out.weight, mode="fan_in")
        self.cls_out.bias.data.zero_()
        self.reg_out.bias.data.zero_()
        self.use_cuda_graph = default_cuda_graph()   # replay one CUDA graph per input shape (FCN_CUDA_GRAPH)
        self.copy_outputs = True      # False: return views of the engine's output block (zero-copy)
        self.train_kernels = os.environ.get("FCN_TRAIN_KERNELS", "1") != "0"   # train(): csrc/train.cu, else autograd
        # train() kernels in their bit-reproducible mode: True / False, or None = torch.are_deterministic_algorithms_enabled()
        self.deterministic = None

    def _engine_spec(self):
        return self.ARCH, self.num_vec, self.dataset_name, self.feat_net.dists, self.num_bins, ""

    def forward(self, data_dicts):
        point_cloud = data_dicts.get("point_cloud")
        one_hot_vec = data_dicts.get("one_hot")
        S = self.ARCH.num_scales
        centers = [data_dicts.get("center_ref%d" % (i + 1)) for i in range(S)]
        has_labels = data_dicts.get("box3d_center") is not None
        if has_labels or self.training or point_cloud.shape[1] > 3:
            assert has_labels or not self.training, "Please provide labels for training."
            from frustum_convnet_b200.train_path import pointnet_det_kernels, pointnet_det_torch
            # train() mode with labels on a CUDA xyz cloud: hand-written training kernels (csrc/train.cu);
            # everything else (label inputs in eval mode, extra point features, train_kernels = False): torch ops
            if self.training and has_labels and self.train_kernels and point_cloud.is_cuda and point_cloud.shape[1] == 3:
                return pointnet_det_kernels(self, data_dicts)
            return pointnet_det_torch(self, data_dicts)
        # repeated calls with the SAME dict object and the same tensors (serving loops cycle through a pool of
        # pre-built batches): the shape / dtype / contiguity checks were done on first sight
        cache = self.__dict__.setdefault("_seen_inputs", {})
        ent = cache.get(id(data_dicts))
        if ent is not None and ent[0] is point_cloud and ent[5] is one_hot_vec and \
                all(a is b for a, b in zip(ent[3], centers)):
            xyz, cs, oh = ent[1], ent[2], ent[4]
            trusted = True
        else:
            xyz = point_cloud[:, :3, :].contiguous()
            cs = [c.contiguous() for c in centers]
            oh = None if one_hot_vec is None else one_hot_vec.contiguous()
            trusted = False
            if len(cache) > 4096:
                cache.clear()
            cache[id(data_dicts)] = (point_cloud, xyz, cs, tuple(centers), oh, one_hot_vec)
        out = self.engine().forward(xyz, cs, oh, use_graph=self.use_cuda_graph, copy_out=self.copy_outputs,
                                    trusted=trusted)
        return tuple(out)
