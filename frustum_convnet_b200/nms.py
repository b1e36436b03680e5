"""Rotated 3-D NMS on the device - drop-in for the reference's ``cube_nms`` (= ``rotate_nms_3d_cc``,
ops/pybind11/rbbox_iou.py:294-311, imported by train/test_net_det.py:44 and called at :140).

    keep = cube_nms(dets_for_nms, threshold)                   # one list, like the reference (CUDA tensor in)
    keep, counts = rotate_nms_3d_batched(dets, offsets, thr)   # every image x class list of a batch in ONE launch

`dets`: (n, 8) rows [cx, cy, cz, l, w, h, ry, score].  No CPU fallback: CPU tensors raise."""
from __future__ import annotations

import torch

from . import _lib


def rotate_nms_3d_batched(dets: torch.Tensor, seg_offsets: torch.Tensor, thresh: float, top_k: int = 300):
    """-> (keep (S, top_k) int32 global row indices in descending-score order, counts (S,) int32).  Every list
    holds at most ``fcn_rotate_nms_3d_max_dets()`` (512) rows; a longer one raises RuntimeError."""
    if not dets.is_cuda:
        raise RuntimeError("rotate_nms_3d: CUDA tensors required (there is no CPU fallback)")
    assert dets.dim() == 2 and dets.shape[1] == 8, "dets must be (n, 8): cx, cy, cz, l, w, h, ry, score"
    d = dets.detach().to(torch.float32).contiguous()
    lens = torch.diff(seg_offsets.detach().to("cpu", torch.int64))
    cap = int(_lib.load().fcn_rotate_nms_3d_max_dets())
    if lens.numel() and int(lens.max()) > cap:
        # the kernel ranks and suppresses one list in shared memory; a longer list would be cut to its first rows
        raise RuntimeError("rotate_nms_3d: a list of %d detections exceeds the %d one launch handles per list"
                           % (int(lens.max()), cap))
    off = seg_offsets.to(device=d.device, dtype=torch.int32).contiguous()
    S = off.numel() - 1
    keep = torch.full((max(S, 0), top_k), -1, dtype=torch.int32, device=d.device)
    cnt = torch.zeros(max(S, 0), dtype=torch.int32, device=d.device)
    if S > 0:
        with torch.cuda.device(d.device):
            _lib.call("fcn_rotate_nms_3d", S, d.data_ptr(), off.data_ptr(), float(thresh), int(top_k), keep.data_ptr(),
                      cnt.data_ptr(), int(top_k), torch.cuda.current_stream(d.device).cuda_stream)
    return keep, cnt


def rotate_nms_3d_cc(dets: torch.Tensor, thresh: float, top_k: int = 300):
    """Same contract as the reference function of that name: indices to keep (descending score)."""
    n = dets.shape[0]
    if n == 0:
        return []
    off = torch.tensor([0, n], dtype=torch.int32, device=dets.device)
    keep, cnt = rotate_nms_3d_batched(dets, off, thresh, top_k)
    return keep[0, : int(cnt[0])].tolist()


cube_nms = rotate_nms_3d_cc
