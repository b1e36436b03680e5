"""The validation pass of train/train_net_det.py ``validate()`` (:162-203) on the device: eval-mode losses and metrics
of every batch from the fused forward's head logits, averaged over the epoch without a host sync per batch.

    val = Validator(model)                       # model.eval(); reuse the object across epochs
    for data_dicts in val_loader:
        val.add({k: v.cuda() for k, v in data_dicts.items()})   # forward graph + two launches, no host sync
    states = val.finalize()                      # == TrainingStates.get_states(avg=True) of the reference loop
    val.reset()

`TrainStates` keeps the reference train() loop's per-step TrainingStates the same way (``TrainStep.states``).

A sharded pass (one process per GPU, each rank adding its chunk of every batch) constructs
``Validator(model, group=dist.group.WORLD)``: `finalize` is then collective and every rank returns the same averages,
those of each batch's values averaged over the ranks, as the reference logs them under DataParallel.

`add` stages the batch into the forward plan of its (B, N, T) shape, replays the plan's forward graph and runs
``fcn_val_batch`` (csrc/validate.cu) on the plan's pitched head logits; the batch's 14 values are appended to a
device table.  `finalize` replays the reference's float64 AverageMeter over that table (``fcn_val_finalize``) and
reads the result once.  Weights are taken from ``model.engine()`` on every `add`, so optimizer steps between epochs
are picked up.  ``PointNetDet.forward`` itself is unchanged.  No CPU fallback: CPU tensors raise."""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from .config import get_cfg


def state_keys():
    """The 14 names of the reference's TrainingStates in its order (det_base.py:505-523), IoU_<cfg.IOU_THRESH> last."""
    return ("total_loss", "cls_loss", "center_loss", "head_cls_loss", "head_res_loss", "size_cls_loss", "size_res_loss",
            "corners_loss", "cls_acc", "head_acc", "size_acc", "IoU_2D", "IoU_3D", "IoU_" + str(get_cfg().IOU_THRESH))


def loss_weights():
    """The cfg's (w_box, w_head_reg, w_size_reg, w_corner, iou_thresh), read now."""
    cfg = get_cfg()
    L = cfg.LOSS
    return (float(L.BOX_LOSS_WEIGHT), float(L.HEAD_REG_WEIGHT), float(L.SIZE_REG_WEIGHT),
            float(L.CORNER_LOSS_WEIGHT), float(cfg.IOU_THRESH))


def set_loss_settings(a, model, weights):
    """NH, NS, with_iou of `model` (read now) and `weights` (`loss_weights()`) into a LossArgs or a ValBatchArgs."""
    a.NH, a.NS = model.num_bins, model.num_size_cluster
    a.with_iou = 1 if getattr(model, "gpu_iou_metrics", True) else 0
    a.w_box, a.w_head_reg, a.w_size_reg, a.w_corner, a.iou_thresh = weights


class _PlanLabels:
    """Label buffers and the fcn_val_batch arguments of one forward plan (kept on the plan, so they live and die
    with its workspace)."""

    def __init__(self, plan):
        eng, B, T2 = plan.eng, plan.B, plan.T[1]
        dev, f32, i64 = eng.device, torch.float32, torch.int64
        self.cls_label = torch.zeros((B, T2), dtype=i64, device=dev)
        self.size_class = torch.zeros(B, dtype=i64, device=dev)
        self.center = torch.zeros((B, 3), dtype=f32, device=dev)
        self.heading = torch.zeros(B, dtype=f32, device=dev)
        self.size = torch.zeros((B, 3), dtype=f32, device=dev)
        n = int(_lib.load().fcn_val_partials_floats(B, T2))
        self.partials = torch.zeros(max(n, 1), dtype=f32, device=dev)
        logits, pitch, ld, ref2 = plan.head_logits()
        a = _lib.ValBatchArgs()
        a.B, a.T2 = B, T2
        a.logit_pitch, a.ld_logit = pitch, ld
        a.logits, a.center_ref2, a.mean_size = logits.data_ptr(), ref2.data_ptr(), eng.mean_size.data_ptr()
        a.cls_label, a.size_class = self.cls_label.data_ptr(), self.size_class.data_ptr()
        a.box3d_center, a.box3d_heading, a.box3d_size = (self.center.data_ptr(), self.heading.data_ptr(),
                                                          self.size.data_ptr())
        a.partials = self.partials.data_ptr()
        self.args = a

    def stage(self, data, B, T2):
        self.cls_label.copy_(data["cls_label"].reshape(B, T2), non_blocking=True)
        self.size_class.copy_(data["size_class"].reshape(B), non_blocking=True)
        self.center.copy_(data["box3d_center"].reshape(B, 3), non_blocking=True)
        self.heading.copy_(data["box3d_heading"].reshape(B), non_blocking=True)
        self.size.copy_(data["box3d_size"].reshape(B, 3), non_blocking=True)


class _MeterTable:
    """A device table of `capacity` ``FCN_VAL_ROW`` rows, its 4-int state and their float64 AverageMeter replay; a
    subclass appends the rows and names them by ``_NAMES`` = (class, row, rows, reference loop, capacity call)."""

    def __init__(self, device, capacity=None):
        self.device = torch.device(device)
        self.capacity = int(capacity) if capacity is not None else 4096
        if self.capacity < 1:
            raise ValueError("capacity must be >= 1")
        self.keys = state_keys()
        self.table = torch.zeros((self.capacity, _lib.VAL_ROW), dtype=torch.float32, device=self.device)
        self.state = torch.zeros(4, dtype=torch.int32, device=self.device)
        self._result = torch.zeros(C.sizeof(_lib.ValResult), dtype=torch.uint8, device=self.device)
        self.last_result = None

    def _join(self):
        """-> the stream the reads are ordered on, after every append so far."""
        return torch.cuda.current_stream(self.device)

    def _check(self, status, first_no_fg, added):
        name, row, rows, loop, call = self._NAMES
        if status & _lib.VAL_NO_FG:
            raise RuntimeError("%s: %s %d of the epoch has no foreground row (cls_label == 1); the reference %s "
                               "rejects it (assert fg_idx.numel() != 0)" % (name, row, first_no_fg, loop))
        if status & _lib.VAL_OVERFLOW:
            raise RuntimeError("%s: %d %s were added but the capacity is %d; construct %s or more"
                               % (name, added, rows, self.capacity, call % added))

    def _rows(self, full):
        with torch.cuda.device(self.device):
            self._join()
            n = min(int(self.state[0].item()), self.capacity)
            t = self.table[:n].cpu().numpy()
        return np.ascontiguousarray(t if full else t[:, :_lib.VAL_VALUES])

    def _over_ranks(self, group, ordered):
        """(table, state) as the reference's DataParallel loop logs them: each row's values averaged over the
        ranks of `group`, B / nfg / nkeep summed (the full batch), the status bits of every rank and the earliest
        row without a foreground row on any rank.  ordered=True sums the rows in rank order (one all_gather of the
        table and ``fcn_rank_fold``), so the bits do not depend on the transport; False takes one all_reduce.  The
        flags are reduced by one integer MAX all_reduce, which is exact.  Collective; runs on the current stream."""
        import torch.distributed as dist
        world = dist.get_world_size(group)
        if ordered:
            n = self.table.numel()
            rows = torch.empty(world * n, dtype=self.table.dtype, device=self.device)
            dist.all_gather_into_tensor(rows, self.table.view(-1), group=group)
            table = torch.empty_like(self.table)
            _lib.call("fcn_rank_fold", rows.data_ptr(), n, world, n, table.data_ptr(),
                      torch.cuda.current_stream(self.device).cuda_stream)
        else:
            table = self.table.clone()
            dist.all_reduce(table, group=group)
        table[:, :_lib.VAL_VALUES] /= world
        s = self.state
        no_fg = (s[1] & _lib.VAL_NO_FG) != 0
        flags = torch.stack([s[1] & _lib.VAL_NO_FG, s[1] & _lib.VAL_OVERFLOW,
                             torch.where(no_fg, -s[2], torch.full_like(s[2], -(2 ** 31 - 1)))])
        dist.all_reduce(flags, op=dist.ReduceOp.MAX, group=group)   # OR of the bits, earliest row without foreground
        state = torch.stack([s[0], flags[0] | flags[1], -flags[2], s[3]])
        return table, state

    def _replay(self, table, state):
        """fcn_val_finalize over `table` and `state`, one host read and the status check -> the 14 averages."""
        with torch.cuda.device(self.device):
            _lib.call("fcn_val_finalize", table.data_ptr(), self.capacity, state.data_ptr(), self._result.data_ptr(),
                      self._join().cuda_stream)
            r = _lib.ValResult.from_buffer_copy(self._result.cpu().numpy().tobytes())
        self.last_result = r
        self._check(r.status, r.first_no_fg, r.added)
        return OrderedDict((k, float(r.avg[i])) for i, k in enumerate(self.keys))


class Validator(_MeterTable):
    """Eval-mode losses and metrics of one epoch on the device (see the module docstring); `capacity` = batches one
    epoch may add (default 4096).  Without `group`: one process, one device.  With `group` (a torch.distributed
    process group, NCCL or gloo; every rank adds its chunk of every batch): `add` is unchanged and `finalize` is
    collective, returning on every rank the same averages of the rank-ordered mean of each batch's values."""

    LABEL_KEYS = ("cls_label", "size_class", "box3d_center", "box3d_heading", "box3d_size")
    _NAMES = ("Validator", "batch", "batches", "validate()", "Validator(model, capacity=%d)")

    def __init__(self, model, capacity=None, group=None):
        self.model = model
        self.group = group
        p = next(model.parameters(), None)
        if p is None or p.device.type != "cuda":
            raise RuntimeError("Validator: the model must live on a CUDA device (there is no CPU fallback)")
        super().__init__(p.device, capacity)
        self._weights = loss_weights()
        self._streams = {}
        self._reset_event, self._reset_waited = None, set()
        self._engine, self._pinned = None, {}

    def reset(self):
        """Start a new epoch.  The counter is zeroed on the current stream; the next `add` on any other stream waits
        for it."""
        with torch.cuda.device(self.device):
            self.state.zero_()
            self._reset_event = torch.cuda.Event()
            self._reset_event.record()
        self._reset_waited = {torch.cuda.current_stream(self.device).cuda_stream}
        self._streams = {}

    def add(self, data):
        """One reference-style batch with labels (CUDA tensors): stage it into the forward plan of its shape, replay
        the plan's forward graph, then compute and append the batch's losses and metrics.  No host sync (except the
        first time a shape is seen on a stream, when its forward plan and graph are built), so the caller may capture
        `add` itself after one un-captured `add` per shape on the capture stream.  Such a graph stays valid while the
        model's weight pack does: the Validator keeps every plan it used alive (also past the engine's plan limit)
        until a weight change rebuilds the engine, whose old workspaces are then released."""
        m = self.model
        if m.training:
            raise RuntimeError("Validator.add: call model.eval() first (the reference validate() runs in eval mode)")
        pc = data["point_cloud"]
        if pc.dim() != 3 or pc.shape[1] != 3:
            raise ValueError("Validator.add: point_cloud must be (B, 3, N); inputs with extra channels are not supported")
        missing = [k for k in self.LABEL_KEYS if data.get(k) is None]
        if missing:
            raise ValueError("Validator.add: labels missing: %s" % ", ".join(missing))
        for k in ("point_cloud",) + self.LABEL_KEYS:
            if not data[k].is_cuda:
                raise RuntimeError("Validator.add: %s must be a CUDA tensor (there is no CPU fallback)" % k)
        eng = m.engine()
        S = eng.arch.num_scales
        centers = [data["center_ref%d" % (i + 1)].contiguous() for i in range(S)]
        one_hot = data.get("one_hot") if eng.num_vec > 0 else None
        if one_hot is not None:
            one_hot = one_hot.contiguous()
        pc = pc.contiguous()
        B, N = int(pc.shape[0]), int(pc.shape[2])
        plan = eng.plan(B, N, [int(c.shape[2]) for c in centers])
        if eng is not self._engine:                  # a rebuilt engine: its plans replace the old ones
            self._engine, self._pinned = eng, {}
        self._pinned[id(plan)] = plan
        lab = plan.__dict__.get("_val_labels")
        if lab is None:
            lab = plan._val_labels = _PlanLabels(plan)
        stream = torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device):
            if stream.cuda_stream not in self._reset_waited and not torch.cuda.is_current_stream_capturing():
                if self._reset_event is not None:
                    stream.wait_event(self._reset_event)
                self._reset_waited.add(stream.cuda_stream)
            lab.stage(data, B, plan.T[1])
            plan.forward_staged(pc, centers, one_hot)
            a = lab.args
            set_loss_settings(a, m, self._weights)
            a.capacity, a.state, a.table = self.capacity, self.state.data_ptr(), self.table.data_ptr()
            _lib.call("fcn_val_batch", C.byref(a), stream.cuda_stream)
        self._streams[stream.cuda_stream] = stream

    def _join(self):
        cur = torch.cuda.current_stream(self.device)
        for st in self._streams.values():
            if st.cuda_stream != cur.cuda_stream:
                cur.wait_stream(st)
        return cur

    def finalize(self):
        """-> OrderedDict of the 14 epoch averages in the order of the reference's
        ``TrainingStates.get_states(avg=True)``; one host read.  Raises if a batch had no foreground row or the
        table overflowed.  With `group` every rank of it must call it: the batch counters of all ranks are gathered
        and read once, each batch's row is summed over the ranks in rank order, its 14 values divided by the number
        of ranks, and B / nfg / nkeep kept summed.  Every verdict is taken from the gathered values, so every rank
        raises the same error: ValueError if the ranks added different numbers of batches, RuntimeError if a batch
        had no foreground row on some rank or a rank's table overflowed."""
        if self.group is None:
            return self._replay(self.table, self.state)
        import torch.distributed as dist
        world = dist.get_world_size(self.group)
        with torch.cuda.device(self.device):
            self._join()
            states = torch.empty(world * 4, dtype=torch.int32, device=self.device)
            dist.all_gather_into_tensor(states, self.state, group=self.group)
            added = states.view(world, 4)[:, 0].cpu().tolist()
            if len(set(added)) > 1:
                raise ValueError("Validator: the ranks of the group added different numbers of batches (%s); every "
                                 "rank must add its chunk of every batch"
                                 % ", ".join("rank %d: %d" % (r, a) for r, a in enumerate(added)))
            table, state = self._over_ranks(self.group, ordered=True)
        return self._replay(table, state)

    def meters(self):
        """(sum, count) of each AverageMeter after the last `finalize`, keyed like its result."""
        r = self.last_result
        if r is None:
            raise RuntimeError("Validator.meters: call finalize() first")
        return OrderedDict((k, (float(r.sum[i]), float(r.count))) for i, k in enumerate(self.keys))

    def per_batch(self, full=False):
        """(n, 14) float32 values of the batches added so far (the `val` of each meter, for logging); full=True
        returns the whole rows (n, 18) with B, nfg and nkeep in columns 14-16."""
        return self._rows(full)


class TrainStates(_MeterTable):
    """The training loop's TrainingStates (train/train_net_det.py:131-134) on the device: every optimizer step of
    ``TrainStep.step`` appends its 14 losses and metrics and its batch size to a device table
    (``fcn_train_states_append``, no host sync), and the epoch's averages are the same float64 AverageMeter replay as
    `Validator.finalize` (``fcn_val_finalize``).  Appends, `reset` and the reads are ordered on the current stream.

        ts.states.reset()                          # start of an epoch
        for i, data in enumerate(loader):
            ts.step(data)
            if (i + 1) % cfg.disp == 0:
                print(ts.states.last())            # training_states.get_states(avg=False); one sync
        epoch = ts.states.finalize()               # training_states.get_states(avg=True)

    `capacity` = steps one epoch may add (default 4096); `deterministic`: a callable read at `finalize`, True when
    the owning TrainStep runs in deterministic mode (then the mean over ranks is summed in rank order)."""

    _NAMES = ("TrainStates", "step", "steps", "train()", "TrainStep(..., states_capacity=%d)")

    def __init__(self, device, capacity=None, deterministic=None):
        super().__init__(device, capacity)
        self._deterministic = deterministic

    def reset(self):
        """Start a new epoch (stream-ordered: the counter is zeroed on the current stream)."""
        with torch.cuda.device(self.device):
            self.state.zero_()

    def append(self, block, B):
        """One step: `block` holds 16 device floats laid out as fcn_det_loss's result (the 14 values, #foreground,
        #non-ignored rows); B is the step's batch size."""
        if not (block.is_cuda and block.dtype == torch.float32 and block.numel() == 16 and block.is_contiguous()):
            raise ValueError("TrainStates.append: block must be 16 contiguous float32 values on the device")
        _lib.call("fcn_train_states_append", block.data_ptr(), int(B), self.table.data_ptr(), self.capacity,
                  self.state.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)

    def last(self):
        """-> OrderedDict of the last step's 14 values (``get_states(avg=False)``); one host read, meant for every
        `cfg.disp` steps rather than every step."""
        with torch.cuda.device(self.device):
            idx = (self.state[:1].long() - 1).clamp_(0, self.capacity - 1)
            raw = torch.cat([self.table.index_select(0, idx).view(-1), self.state.view(torch.float32)]).cpu().numpy()
        row, state = raw[:_lib.VAL_ROW], raw[_lib.VAL_ROW:].view(np.int32)
        if state[0] == 0:
            raise RuntimeError("TrainStates.last: no step since the last reset()")
        self._check(int(state[1]), int(state[2]), int(state[0]))
        return OrderedDict((k, float(row[i])) for i, k in enumerate(self.keys))

    def per_step(self, full=False):
        """(n, 14) float32 values of the steps added so far; full=True returns the whole rows (n, 18) with B, nfg and
        nkeep in columns 14-16."""
        return self._rows(full)

    def finalize(self):
        """-> OrderedDict of the 14 epoch averages (``get_states(avg=True)``); one host read.  With torch.distributed
        initialised and world > 1 every rank must call it (ranks step in lockstep, so row i is the same step on every
        rank); in deterministic mode the rows are summed over the ranks in rank order, so every rank returns the same
        bits.  Raises, naming the step, if a step had no foreground row, and if more steps were added than
        `capacity`, naming the capacity needed."""
        import torch.distributed as dist
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        with torch.cuda.device(self.device):
            if world > 1:
                ordered = bool(self._deterministic()) if self._deterministic is not None else False
                table, state = self._over_ranks(None, ordered)
            else:
                table, state = self.table, self.state
        return self._replay(table, state)
