"""Per-image 3-D detections on the device: the step between the forward and the result files of
train/test_net_det.py:243-305 (test_net_det_sunrgbd.py:197-266), with no per-batch host copy.

    col = DetectionCollector(test_dataset.id_list, test_dataset.type_list, test_dataset.box2d_list,
                             dataset=cfg.DATA.DATASET_NAME, method=cfg.TEST.METHOD, thresh=cfg.TEST.THRESH)
    for i, data_dicts in enumerate(test_loader):
        outputs = model(data_dicts_var)
        col.add(outputs, data_dicts_var, first=load_batch_size * i)   # one launch, no host sync, capturable
    nms_results = col.finalize()      # == the dict test() hands to write_detection_results

`add` appends the foreground rows of a batch to device records (csrc/detect.cu, ``fcn_det_candidates``);
`finalize` orders them as the reference's lists, runs rotated 3-D NMS on every image x class list of any length and
returns {data_idx: {class_type: float32 (n, 12)}} in the reference's dict order, zero-row lists included (as
(0, 12) arrays).  The collector belongs to one device.  No CPU fallback: CPU tensors raise.

With one process per GPU, ``DetectionCollector(..., group=pg)`` collects a sharded pass: every rank adds the frustums
of its own chunk of each batch (``first`` stays the dataset index), and ``finalize_device()`` / ``finalize()`` on every
rank of the group return what one collector that received every rank's adds would return."""
from __future__ import annotations

import ctypes as C
import hashlib

import numpy as np
import torch

from . import _lib
from ._host import cuda_device, workspace

_DATASETS = {"KITTI": 0, "SUNRGBD": 1}
_METHODS = {"nms": _lib.DET_NMS}   # every other cfg.TEST.METHOD behaves as 'top' (test_net_det.py:256-263)
_SETUP_FIELDS = ("id_list", "type_list", "box2d_list", "dataset", "method", "thresh", "top_k", "num_frustums")


def setup_digests(id_list, type_list, box2d_list, dataset, method, thresh, top_k):
    """One digest per argument that defines the segment table and the finalize, in _SETUP_FIELDS order."""
    h = lambda b: hashlib.sha256(b).hexdigest()
    text = lambda xs: h("\x1f".join(str(x) for x in xs).encode())
    return (text(id_list), text(type_list), h(np.ascontiguousarray(box2d_list, dtype=np.float32).tobytes()),
            str(dataset), "nms" if method == "nms" else "top", repr(float(thresh)), repr(int(top_k)),
            repr(len(id_list)))


def check_same_setup(group, digests):
    """Collective over `group`: raises the same ValueError on every rank unless every rank passed the same
    setup_digests."""
    import torch.distributed as dist
    everyone = [None] * dist.get_world_size(group)
    dist.all_gather_object(everyone, tuple(digests), group=group)
    for r, theirs in enumerate(everyone):
        differ = [name for name, a, b in zip(_SETUP_FIELDS, everyone[0], theirs) if a != b]
        if differ:
            raise ValueError("DetectionCollector: rank %d of the group was constructed with a different %s than rank "
                             "0; every rank must describe the same dataset and finalize" % (r, ", ".join(differ)))


def shard_merge_plan(counts, capacities, added):
    """The host decisions of a sharded finalize, made alike on every rank from the gathered block: counts and
    capacities (world,) of every rank's records, added (world, num_frustums) bool.  -> the frustums added on any rank
    (num_frustums,) bool.  Raises ValueError naming the first frustum added on two ranks, and RuntimeError naming the
    first rank whose rows overflowed its capacity."""
    added = np.asarray(added, dtype=bool)
    twice = np.flatnonzero(added.sum(axis=0) > 1)
    if len(twice):
        f = int(twice[0])
        ranks = np.flatnonzero(added[:, f])
        raise ValueError("DetectionCollector: frustum %d was added on ranks %d and %d; the shards of a pass must not "
                         "overlap" % (f, ranks[0], ranks[1]))
    for r, (n, cap) in enumerate(zip(np.asarray(counts).tolist(), np.asarray(capacities).tolist())):
        if n > cap:
            raise RuntimeError("DetectionCollector: record capacity exceeded on rank %d: %d rows were produced, the "
                               "capacity is %d (needs capacity >= %d)" % (r, n, cap, n))
    return added.any(axis=0)


class DetectionCollector:
    def __init__(self, id_list, type_list, box2d_list, dataset="KITTI", method="nms", thresh=0.1, top_k=300,
                 capacity=None, device=None, group=None):
        """group: a torch.distributed process group for a sharded pass (None: this process's adds alone).  With a
        group, construction is collective and raises the same ValueError on every rank if the ranks' id_list,
        type_list, box2d_list, dataset, method, thresh or top_k differ."""
        self.group = group
        if group is not None:
            with torch.cuda.device(cuda_device(device, "DetectionCollector")):
                check_same_setup(group, setup_digests(id_list, type_list, box2d_list, dataset, method, thresh, top_k))
        if dataset not in _DATASETS:
            raise ValueError("dataset must be one of %s" % sorted(_DATASETS))
        n = len(id_list)
        if len(type_list) != n or len(box2d_list) != n:
            raise ValueError("id_list, type_list and box2d_list must have the same length")
        self.dataset, self.method = dataset, ("nms" if method == "nms" else "top")
        self.thresh, self.top_k = float(thresh), int(top_k)
        self.num_frustums = n
        self.device = cuda_device(device, "DetectionCollector")
        # segment table in the reference's dict order: images by first appearance, classes by first appearance
        # within the image (test_net_det.py:278-282)
        seg_of, self.segments = {}, []
        table = np.empty(n, dtype=np.int32)
        for f in range(n):
            key = (id_list[f], type_list[f])
            s = seg_of.get(key)
            if s is None:
                s = seg_of[key] = len(self.segments)
                self.segments.append(key)
            table[f] = s
        self._seg_host = table
        self.capacity = int(capacity) if capacity is not None else max(65536, 16 * n)
        dev = self.device
        self.seg_of_frustum = torch.from_numpy(table).to(dev)
        self.box2d = torch.from_numpy(np.asarray(box2d_list, dtype=np.float32).reshape(n, 4)).to(dev)
        self.counter = torch.zeros(1, dtype=torch.int32, device=dev)
        self.records = torch.empty((max(self.capacity, 1), 12), dtype=torch.int32, device=dev)   # fcn_det_record
        self.added = np.zeros(n, dtype=bool)
        self._streams = {}

    def reset(self):
        """Start a new pass (stream-ordered on the current stream)."""
        self.counter.zero_()
        self.added[:] = False
        self._streams = {}

    def add(self, outputs, data_dicts, first):
        """Append the rows of one batch: `outputs` = the model's six-tuple, `data_dicts` supplies rot_angle and the
        optional rgb_prob / ref_center, frustum b of the batch is dataset entry first + b.  One launch on the
        current stream; no host sync, so it may be captured in a CUDA graph (a captured add marks its frustums when
        it is captured, and every replay appends its rows again)."""
        cls_probs, center, heading, size, _, size_probs = outputs
        for t in (cls_probs, center, heading, size, size_probs):
            if not t.is_cuda:
                raise RuntimeError("DetectionCollector.add: CUDA tensors required (there is no CPU fallback)")
        B, T2 = int(cls_probs.shape[0]), int(cls_probs.shape[1])
        first = int(first)
        if first < 0 or first + B > self.num_frustums:
            raise ValueError("frustums [%d, %d) are outside the dataset of %d" % (first, first + B, self.num_frustums))
        f32 = lambda t: t.detach().to(device=self.device, dtype=torch.float32).contiguous()
        keep_alive = [f32(cls_probs), f32(center), f32(heading).reshape(B, T2), f32(size), f32(size_probs)]
        rot = data_dicts["rot_angle"]
        if not rot.is_cuda:
            raise RuntimeError("DetectionCollector.add: rot_angle must be a CUDA tensor")
        keep_alive.append(f32(rot).reshape(B))
        opt = []
        for k, shape in (("rgb_prob", (B,)), ("ref_center", (B, 3))):
            v = data_dicts.get(k)
            if v is not None:
                if not v.is_cuda:
                    raise RuntimeError("DetectionCollector.add: %s must be a CUDA tensor" % k)
                v = f32(v).reshape(shape)
                keep_alive.append(v)
            opt.append(v)
        cp, ce, he, sz, sp, ra = keep_alive[:6]
        a = _lib.DetCandidateArgs()
        a.B, a.T2, a.NS = B, T2, int(sp.shape[-1])
        a.dataset, a.method = _DATASETS[self.dataset], _METHODS.get(self.method, _lib.DET_TOP)
        a.first, a.num_frustums, a.capacity = first, self.num_frustums, self.capacity
        a.cls_probs, a.center, a.heading, a.size, a.size_probs = (t.data_ptr() for t in (cp, ce, he, sz, sp))
        a.rot_angle = ra.data_ptr()
        a.rgb_prob = opt[0].data_ptr() if opt[0] is not None else None
        a.ref_center = opt[1].data_ptr() if opt[1] is not None else None
        a.seg_of_frustum, a.counter, a.records = (self.seg_of_frustum.data_ptr(), self.counter.data_ptr(),
                                                  self.records.data_ptr())
        stream = torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device):
            _lib.call("fcn_det_candidates", C.byref(a), stream.cuda_stream)
        self._streams[stream.cuda_stream] = stream
        self.added[first:first + B] = True

    def finalize_device(self):
        """-> CollectedDetections: the kept rows stay on the device; one host sync to size the NMS bit matrix and one
        read of the per-segment offsets and keep counts (O(segments), no row crosses to the host).

        With a group this is collective (every rank of the group must call it) and every rank gets the same result:
        the union of every rank's records, finalized as one collector's.  Raises the same error on every rank if a
        frustum was added on two ranks or a rank overflowed its capacity."""
        dev = self.device
        cur = torch.cuda.current_stream(dev)
        for st in self._streams.values():
            if st.cuda_stream != cur.cuda_stream:
                cur.wait_stream(st)
        if self.group is None:
            counter, records, capacity, added = self.counter, self.records, self.capacity, self.added
        else:
            with torch.cuda.device(dev):
                counter, records, capacity, added = self._merge_ranks()
        S = len(self.segments)
        with torch.cuda.device(dev):
            ws, nbytes = workspace("fcn_det_workspace_bytes", dev, capacity, S)
            info = torch.zeros(4, dtype=torch.int64, device=dev)
            off = torch.zeros(S + 1, dtype=torch.int32, device=dev)
            kc = torch.zeros(max(S, 1), dtype=torch.int32, device=dev)
            rows = torch.empty((max(capacity, 1), 12), dtype=torch.float32, device=dev)
            a = _lib.DetFinalizeArgs()
            a.num_segments, a.num_frustums, a.capacity = S, self.num_frustums, capacity
            a.method, a.dataset = _METHODS.get(self.method, _lib.DET_TOP), _DATASETS[self.dataset]
            a.top_k, a.thresh = self.top_k, self.thresh
            a.counter, a.records, a.box2d = counter.data_ptr(), records.data_ptr(), self.box2d.data_ptr()
            a.workspace, a.workspace_bytes, a.info = ws.data_ptr(), nbytes, info.data_ptr()
            a.seg_offsets, a.keep_count, a.rows = off.data_ptr(), kc.data_ptr(), rows.data_ptr()
            _lib.call("fcn_det_prepare", C.byref(a), cur.cuda_stream)
            n_counted, mask_words = (int(v) for v in info[:2].tolist())          # the one host sync
            a.n_counted = n_counted
            mask = torch.empty(max(mask_words, 1), dtype=torch.int32, device=dev)
            a.mask, a.mask_words = mask.data_ptr(), mask_words
            _lib.call("fcn_det_select", C.byref(a), cur.cuda_stream)
            offkc = torch.cat([off, kc[:S]]).cpu().numpy()                      # O(S) metadata, one copy
        off_h, kc_h = offkc[:S + 1].copy(), offkc[S + 1:].copy()
        self.last_counts = {"rows": n_counted, "kept": int(kc_h.sum()) if S else 0}
        # dict order of the frustums that were added, in dataset order
        segs = self._seg_host[added]
        _, first_pos = np.unique(segs, return_index=True)
        order = segs[np.sort(first_pos)]
        return CollectedDetections(self.dataset, rows, off, kc, off_h, kc_h, list(self.segments), order, cur)

    def _merge_ranks(self):
        """-> (counter, records, capacity, added) of the union of every rank's records, on the current stream.  One
        all_gather of each rank's counter, capacity and added flags, one host read of that block, then one all_gather
        of the records.  Every decision is taken from the gathered block, so every rank takes it alike and none raises
        while another waits in a collective.  The union is in rank order; fcn_det_prepare orders records by
        (segment, frustum, t) whoever appended them, so it finalizes as one collector's records would."""
        import torch.distributed as dist
        dev, group, n = self.device, self.group, self.num_frustums
        world = dist.get_world_size(group)
        head = np.array([0, self.capacity], dtype=np.int32).view(np.uint8)
        meta = torch.from_numpy(np.concatenate([head, self.added.view(np.uint8)])).pin_memory().to(
            dev, non_blocking=True)
        meta[:4].view(torch.int32).copy_(self.counter)
        block = torch.empty((world, 8 + n), dtype=torch.uint8, device=dev)
        dist.all_gather(list(block.unbind(0)), meta, group=group)
        block = block.cpu().numpy()                                                # the one extra host sync
        head = block[:, :8].copy().view(np.int32)
        counts = head[:, 0].astype(np.int64)
        added = shard_merge_plan(counts, head[:, 1], block[:, 8:].astype(bool))
        total, most = int(counts.sum()), int(counts.max())
        if most == 0:
            records = torch.empty((1, 12), dtype=torch.int32, device=dev)
        else:
            send = self.records[:most]
            if len(send) < most:                           # another rank produced more rows than this one's capacity
                send = torch.cat([send, send.new_zeros((most - len(send), 12))])
            recv = torch.empty((world, most, 12), dtype=torch.int32, device=dev)
            dist.all_gather(list(recv.unbind(0)), send, group=group)
            records = torch.cat([recv[r, :c] for r, c in enumerate(counts.tolist())])
        counter = torch.full((1,), total, dtype=torch.int32, device=dev)
        return counter, records, total, added

    def finalize(self):
        """-> {data_idx: {class_type: float32 (n, 12)}}; one host sync to size the NMS bit matrix, one copy back."""
        return self.finalize_device().to_dict()


class CollectedDetections:
    """The result of DetectionCollector.finalize_device(), left on the device for the evaluators'
    ``evaluate_collected``.

    rows (n_rows, 12) float32 (device): kept row k of segment s at seg_offsets[s] + k, k < keep_count[s], in the
    reference's list order; seg_offsets / keep_count: the same offsets and counts on the device; host_seg_offsets
    (S + 1) / host_keep_count (S): their host copies; segments: the (data_idx, class_type) key of each segment;
    order: the segments of the added frustums in the reference's dict order (images by first appearance, classes by
    first appearance within the image).  `stream`: the stream the rows were written on."""

    def __init__(self, dataset, rows, seg_offsets, keep_count, host_seg_offsets, host_keep_count, segments, order,
                 stream):
        self.dataset = dataset
        self.num_rows = int(host_seg_offsets[-1])
        self.rows = rows
        self.seg_offsets, self.keep_count = seg_offsets, keep_count
        self.host_seg_offsets = np.ascontiguousarray(host_seg_offsets, dtype=np.int32)
        self.host_keep_count = np.ascontiguousarray(host_keep_count, dtype=np.int32)
        self.segments, self.order, self.stream = segments, np.asarray(order, dtype=np.int64), stream
        self.device = rows.device

    @property
    def num_segments(self):
        return len(self.segments)

    def image_order(self):
        """The images of the dict in its order, and for each segment of `order` the rank of its image there."""
        images, rank, seg_rank = [], {}, np.empty(len(self.order), dtype=np.int64)
        for j, s in enumerate(self.order.tolist()):
            idx = self.segments[s][0]
            r = rank.get(idx)
            if r is None:
                r = rank[idx] = len(images)
                images.append(idx)
            seg_rank[j] = r
        return images, seg_rank

    def to_dict(self):
        """-> {data_idx: {class_type: float32 (n, 12)}}, what DetectionCollector.finalize() returns (one copy of the
        rows to the host)."""
        rows_h = self.rows[:self.num_rows].cpu().numpy()
        off_h, kc_h = self.host_seg_offsets, self.host_keep_count
        res = {}
        for s in self.order:
            idx, ct = self.segments[s]
            res.setdefault(idx, {})[ct] = rows_h[off_h[s]: off_h[s] + kc_h[s]].copy()
        return res

    def feed_args(self, seg_dst, seg_value, num_out, plan_ptrs):
        """fcn_det_eval_feed_args for a gather plan: seg_dst / seg_value (S) int32 host arrays (kept alive by the
        caller), plan_ptrs = their device addresses."""
        a = _lib.DetEvalFeedArgs()
        a.num_segments, a.num_rows, a.num_out = self.num_segments, self.num_rows, int(num_out)
        a.rows, a.seg_offsets, a.keep_count = self.rows.data_ptr(), self.seg_offsets.data_ptr(), \
            self.keep_count.data_ptr()
        a.seg_dst, a.seg_value = plan_ptrs
        a.host_seg_offsets, a.host_keep_count = self.host_seg_offsets.ctypes.data, self.host_keep_count.ctypes.data
        a.host_seg_dst = seg_dst.ctypes.data
        return a
