"""Device-side input builder - what the reference's ``ProviderDataset.__getitem__`` + ``collate`` hand to the model
(datasets/provider_sample.py:133-203,291-327), computed on the GPU from resident raw frustum points.

    fb = FrustumBatchBuilder(strides=cfg.DATA.STRIDE, max_depth=cfg.DATA.MAX_DEPTH, npoints=cfg.DATA.NUM_SAMPLES)
    fb.set_frustums(points_list, frustum_angles, box2d, P2, cls_index)        # once: raw data -> HBM
    data = fb.build(choice)          # per step: (B, N) int32 resampling indices -> dict for PointNetDet.forward

``choice`` stays the caller's ``np.random.choice(n, npoints, n < npoints)`` draw (provider_sample.py:164-166): the
RNG stream is part of the reference's behaviour and is not re-implemented on the device."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._host import on_device


class FrustumBatchBuilder:
    def __init__(self, strides, max_depth, npoints, num_classes=3, device="cuda"):
        self.strides = [float(s) for s in strides]
        self.max_depth = float(max_depth)
        self.T = [len(np.arange(0, self.max_depth, s)) for s in self.strides]
        self.N, self.V = int(npoints), int(num_classes)
        self.device = torch.device(device)
        self.B = 0

    def set_frustums(self, points_list, frustum_angles, box2d, P2, cls_index=None):
        dev = self.device
        counts = [int(p.shape[0]) for p in points_list]
        assert min(counts) >= 1
        self.B = len(counts)
        self.points = torch.from_numpy(np.concatenate([np.asarray(p, dtype=np.float32)[:, :3] for p in points_list])).to(dev)
        self.offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)).to(dev)
        self.angle = torch.from_numpy(np.asarray(frustum_angles, dtype=np.float64).reshape(-1)).to(dev)
        self.box2d = torch.from_numpy(np.asarray(box2d, dtype=np.float64).reshape(self.B, 4)).to(dev)
        self.P = torch.from_numpy(np.asarray(P2, dtype=np.float64).reshape(self.B, 12)).to(dev)
        self.cls = None if cls_index is None else torch.from_numpy(np.asarray(cls_index, dtype=np.int32)).to(dev)
        self._bind()

    def set_frustums_device(self, points, offsets, frustum_angle, box2d, P, cls_index=None):
        """set_frustums from CUDA tensors already on this builder's device (FrustumExtractor's output), with no host
        round trip: points (M, 4 or 3) float32, offsets (B + 1) int32, frustum_angle (B) float64, box2d (B, 4) and
        P (B, 12) float64; cls_index (B) int32 (CUDA tensor or host values) or None.  Every frustum must hold at least
        one point (the extractor drops empty ones; this is not checked here, as that would need the host)."""
        dev = self.device
        for name, t, dt, cols in (("points", points, torch.float32, (3, 4)), ("offsets", offsets, torch.int32, None),
                                  ("frustum_angle", frustum_angle, torch.float64, None),
                                  ("box2d", box2d, torch.float64, (4,)), ("P", P, torch.float64, (12,))):
            if not on_device(t, dev):
                raise RuntimeError("set_frustums_device: %s must be a CUDA tensor on %s" % (name, dev))
            if t.dtype != dt or t.dim() != (1 if cols is None else 2) or (cols is not None and t.shape[1] not in cols):
                raise ValueError("set_frustums_device: %s has dtype %s and shape %s" % (name, t.dtype, tuple(t.shape)))
        self.B = int(offsets.shape[0]) - 1
        if self.B < 1 or frustum_angle.shape[0] != self.B or box2d.shape[0] != self.B or P.shape[0] != self.B:
            raise ValueError("set_frustums_device: offsets, frustum_angle, box2d and P disagree on the frustum count")
        self.points = points[:, :3].contiguous()
        self.offsets, self.angle = offsets.contiguous(), frustum_angle.contiguous()
        self.box2d, self.P = box2d.contiguous(), P.contiguous()
        if isinstance(cls_index, torch.Tensor):
            if not on_device(cls_index, dev):
                raise RuntimeError("set_frustums_device: cls_index must be a CUDA tensor on %s or host values" % dev)
            self.cls = cls_index.to(torch.int32).contiguous()
        else:
            self.cls = None if cls_index is None else torch.from_numpy(np.asarray(cls_index, dtype=np.int32)).to(dev)
        if self.cls is not None and self.cls.numel() != self.B:
            raise ValueError("set_frustums_device: cls_index must have one entry per frustum")
        self._bind()

    def _bind(self):
        dev = self.device
        f32 = torch.float32
        self.out = {"point_cloud": torch.empty((self.B, 3, self.N), dtype=f32, device=dev),
                    "rot_angle": torch.empty((self.B, 1), dtype=f32, device=dev)}
        for s, T in enumerate(self.T):
            self.out["center_ref%d" % (s + 1)] = torch.empty((self.B, 3, T), dtype=f32, device=dev)
        if self.cls is not None:
            self.out["one_hot"] = torch.empty((self.B, self.V), dtype=f32, device=dev)
        a = _lib.InputArgs()
        a.B, a.N, a.num_scales, a.num_classes = self.B, self.N, len(self.T), self.V
        for s, T in enumerate(self.T):
            a.T[s], a.stride[s] = T, self.strides[s]
            a.centers[s] = self.out["center_ref%d" % (s + 1)].data_ptr()
        a.points, a.point_offsets = self.points.data_ptr(), self.offsets.data_ptr()
        a.frustum_angle, a.box2d, a.P = self.angle.data_ptr(), self.box2d.data_ptr(), self.P.data_ptr()
        a.cls_index = None if self.cls is None else self.cls.data_ptr()
        a.point_cloud, a.rot_angle = self.out["point_cloud"].data_ptr(), self.out["rot_angle"].data_ptr()
        a.one_hot = self.out["one_hot"].data_ptr() if self.cls is not None else None
        self.args = a

    def build(self, choice):
        """choice: (B, N) int32 indices (numpy, CPU or CUDA tensor) -> dict of CUDA tensors (overwritten by the next call)."""
        if not isinstance(choice, torch.Tensor):
            choice = torch.from_numpy(np.ascontiguousarray(choice, dtype=np.int32))
        ch = choice.to(device=self.device, dtype=torch.int32, non_blocking=True).contiguous()
        assert tuple(ch.shape) == (self.B, self.N)
        self.args.choice = ch.data_ptr()
        with torch.cuda.device(self.device):
            _lib.call("fcn_build_inputs", C.byref(self.args), torch.cuda.current_stream(self.device).cuda_stream)
        self._keep = ch
        return self.out
