"""SUN-RGBD point clouds from depth images on the device: the SUNRGBD toolbox's read3dPoints as the reference's port
restates it (sunrgbd/read_3d_points.py), C ABI section (24).  This is the point-cloud part of the reference's MATLAB
dump (sunrgbd/matlab/extract_rgbd_data.m, which saves pc/%06d.mat), so the offline extractor and the frame detector
start from the camera's images.

    import cv2
    depth = cv2.imread(depth_png, cv2.IMREAD_UNCHANGED)           # (h, w) uint16, the toolbox's bit-rotated depth
    rgb = cv2.imread(image_jpg)[:, :, ::-1]                        # cv2 gives BGR; the cloud's colours are RGB
    points = depth_clouds([depth], [rgb], [calib], [idx])          # {idx: CUDA (n, 6) float32}
    det = SunrgbdFrustumExtractor().from_rgb_detections(points, {idx: calib}, *read_det_file(path))

Per pixel (v, u) with raw depth r0 != 0: r = r0 rotated right by 3 bits, d = min(float32(r) / 1000, 8) metres,
x3 = ((u - cx) * d) / fx and y3 = ((v - cy) * d) / fy in float64, the point Rtilt @ (x3, d, -y3) in float64 rounded
to float32, and the colour float32(rgb) / 255.  Points are the valid pixels in row-major order.  Decoding the PNG and
JPEG stays with the caller.  No CPU fallback: CPU tensors and devices raise."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from ._host import check_tensors, cuda_device, workspace
from .sunrgbd_extract import calib_mats


class DepthCloudStage:
    """fcn_sunrgbd_depth_cloud for fixed capacities: F frames of at most H x W pixels into (F, P, 6) clouds on one
    device, with the workspace allocated once, so a call allocates nothing and can be captured in a CUDA graph."""

    def __init__(self, frames, height, width, points, device):
        self.F, self.H, self.W, self.P = int(frames), int(height), int(width), int(points)
        self.device = device
        a = _lib.SunrgbdDepthArgs()
        a.num_frames, a.height, a.width, a.point_capacity = self.F, self.H, self.W, self.P
        with torch.cuda.device(device):
            self._ws, a.workspace_bytes = workspace("fcn_sunrgbd_depth_cloud_workspace_bytes", device, C.byref(a))
        a.workspace = self._ws.data_ptr()
        self._a = a

    def check(self, who, depth, rgb, image_hw, calibs):
        F, H, W = self.F, self.H, self.W
        specs = [("depth", depth, (F, H, W), torch.uint16), ("image_hw", image_hw, (F, 2), torch.int32),
                 ("calibs", calibs, (F, 18), torch.float64)]
        if rgb is not None:
            specs.append(("rgb", rgb, (F, H, W, 3), torch.uint8))
        check_tensors(who, self.device, specs)

    def run(self, depth, rgb, image_hw, calibs, clouds, counts, status, stream):
        """Launch on `stream` (a cudaStream_t): clouds (F, P, 6) float32 and counts (F,) int32 written, status bits
        OR-ed into status (int32, one element)."""
        a = self._a
        a.depth, a.rgb = depth.data_ptr(), None if rgb is None else rgb.data_ptr()
        a.image_hw, a.calibs = image_hw.data_ptr(), calibs.data_ptr()
        a.status, a.clouds, a.counts = status.data_ptr(), clouds.data_ptr(), counts.data_ptr()
        _lib.call("fcn_sunrgbd_depth_cloud", C.byref(a), stream)


def pack_calib(calib):
    """A calib dict (or object) with 'Rtilt' and 'K' -> (18,) float64: Rtilt, then K, row-major."""
    return np.concatenate([np.asarray(m, np.float64).reshape(9) for m in calib_mats(calib)])


@torch.no_grad()
def depth_clouds(depths, rgbs, calibs, ids, device=None, chunk=16):
    """depths: (h, w) uint16 depth images (the toolbox's PNGs as read, e.g. cv2.IMREAD_UNCHANGED); rgbs: (h, w, 3)
    uint8 images in RGB order, or None (for the list or an image: colour columns 0); calibs: dicts (or objects) with
    'Rtilt' and 'K', 3 x 3; ids: the frame ids.  -> {id: CUDA (n, 6) float32}, what the reference's read_3d_points
    returns (rounded to float32), for SunrgbdFrustumExtractor.from_ground_truth / from_rgb_detections.

    One device call per `chunk` frames, with capacity P = H * W (the chunk's largest image), so no frame overflows;
    the counts are read back once per chunk."""
    n = len(ids)
    rgbs = [None] * n if rgbs is None else list(rgbs)
    if len(depths) != n or len(rgbs) != n or len(calibs) != n:
        raise ValueError("depth_clouds: depths, rgbs, calibs and ids must have the same length")
    dev = cuda_device(device, "depth_clouds")
    out = {}
    for c0 in range(0, n, int(chunk)):
        part = range(c0, min(c0 + int(chunk), n))
        imgs = [np.asarray(depths[i]) for i in part]
        for i, d in zip(part, imgs):
            if d.ndim != 2 or d.dtype != np.uint16 or min(d.shape) < 1:
                raise ValueError("depth_clouds: depth image of frame %r must be a non-empty (h, w) uint16 array"
                                 % (ids[i],))
            if rgbs[i] is not None and np.asarray(rgbs[i]).shape != d.shape + (3,):
                raise ValueError("depth_clouds: rgb image of frame %r must be (h, w, 3) like its depth" % (ids[i],))
        F = len(imgs)
        H, W = max(d.shape[0] for d in imgs), max(d.shape[1] for d in imgs)
        any_rgb = any(rgbs[i] is not None for i in part)
        h_depth, h_hw = np.zeros((F, H, W), np.uint16), np.zeros((F, 2), np.int32)
        h_rgb = np.zeros((F, H, W, 3), np.uint8) if any_rgb else None
        h_cal = np.stack([pack_calib(calibs[i]) for i in part])
        for f, (i, d) in enumerate(zip(part, imgs)):
            h, w = d.shape
            h_depth[f, :h, :w], h_hw[f] = d, (h, w)
            if rgbs[i] is not None:
                h_rgb[f, :h, :w] = np.asarray(rgbs[i], np.uint8)
        st = DepthCloudStage(F, H, W, H * W, dev)
        with torch.cuda.device(dev):
            to = lambda a: torch.from_numpy(a).to(dev)
            depth = torch.from_numpy(h_depth.view(np.int16)).to(dev).view(torch.uint16)
            rgb = None if h_rgb is None else to(h_rgb)
            clouds = torch.empty((F, H * W, 6), dtype=torch.float32, device=dev)
            counts = torch.empty(F, dtype=torch.int32, device=dev)
            status = torch.zeros(1, dtype=torch.int32, device=dev)
            st.run(depth, rgb, to(h_hw), to(h_cal), clouds, counts, status,
                   torch.cuda.current_stream(dev).cuda_stream)
            for f, k in enumerate(counts.tolist()):
                out[ids[part[f]]] = clouds[f, :k].clone()
    return out
