"""Host side of the two-phase device entries (detect, kitti_eval, sunrgbd_eval, frustum_extract, refine_extract,
gt_extract): check the device, build the host CSR offsets, upload the packed inputs in one copy, query and allocate
the workspace.  Every entry of those modules takes its inputs the same way, so the rules live here once."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

ALIGN = 256          # every part of a packed upload starts at a multiple of this, as every workspace piece does


def cuda_device(device, who):
    """torch.device of `device` (None: the current CUDA device); anything but a CUDA device raises RuntimeError
    naming `who`."""
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("%s: a CUDA device is required (there is no CPU fallback)" % who)
    return dev


def on_device(t, dev):
    """t is a CUDA tensor on dev ('cuda' without an index: the current device)."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        return False
    return t.device.index == (dev.index if dev.index is not None else torch.cuda.current_device())


def check_tensors(who, dev, specs):
    """specs: (name, tensor, shape, dtype) tuples; raises ValueError naming `who` and the first tensor that is not a
    contiguous CUDA tensor of that shape and dtype on dev."""
    for name, t, shape, dt in specs:
        if not on_device(t, dev) or tuple(t.shape) != shape or t.dtype != dt or not t.is_contiguous():
            raise ValueError("%s: %s must be a contiguous %s CUDA tensor of shape %s on %s"
                             % (who, name, dt, shape, dev))


def csr_offsets(counts):
    """Per-group record counts -> int32 CSR offsets [0, n0, n0 + n1, ...] (len(counts) + 1 entries)."""
    off = np.zeros(len(counts) + 1, dtype=np.int32)
    np.cumsum(counts, out=off[1:])
    return off


def pack(parts):
    """Parts (bytes or numpy arrays) -> (one uint8 host buffer holding each part's bytes at a multiple of ALIGN,
    the start of each part)."""
    views = [np.frombuffer(p, dtype=np.uint8) if isinstance(p, bytes) else
             np.ascontiguousarray(p).reshape(-1).view(np.uint8) for p in parts]
    starts, end = [], 0
    for v in views:
        starts.append(end)
        end += -(-v.size // ALIGN) * ALIGN
    buf = np.empty(end, dtype=np.uint8)       # not np.zeros: a calloc of a reused block zeroes every byte again
    for v, s, e in zip(views, starts, starts[1:] + [end]):
        buf[s:s + v.size] = v
        buf[s + v.size:e] = 0
    return buf, starts


def upload(parts, dev):
    """pack(parts) copied to dev in one host-to-device copy -> (the device buffer, which must outlive the calls that
    read it, and each part's device address)."""
    buf, starts = pack(parts)
    t = torch.from_numpy(buf).to(dev)
    return t, [t.data_ptr() + s for s in starts]


def workspace(size_fn, dev, *args):
    """fcn_*_workspace_bytes(*args) -> (a uint8 workspace of max(n, 1) bytes on dev, n).  A negative size raises
    RuntimeError with the library's message."""
    n = int(getattr(_lib.load(), size_fn)(*args))
    if n < 0:
        _lib.check(-1, size_fn)
    return torch.empty(max(n, 1), dtype=torch.uint8, device=dev), n
