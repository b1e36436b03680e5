"""A numpy restatement of fcn_frame_store_append (C ABI section (25)) and a generator of frame-call tables shaped like
a FrameDetections result, for tests/test_frame_store_cpu.py and tests/test_gpu_frame_store.py."""
import numpy as np

STORE_ROWS, STORE_SEGMENTS = 1, 2


class Store:
    """The device store's buffers on the host: rows (row_capacity, 12) float32, image (segments) int64, cls, frame
    and keep (segments) int32, offset (segments + 1) int32 and the cursor (segments, rows, calls, status,
    frame_status)."""

    def __init__(self, rows, segments):
        self.rows = np.zeros((rows, 12), np.float32)
        self.image = np.zeros(segments, np.int64)
        self.cls, self.frame, self.keep = (np.zeros(segments, np.int32) for _ in range(3))
        self.offset = np.zeros(segments + 1, np.int32)
        self.cursor = np.zeros(5, np.int32)

    def append(self, rows, seg_offsets, keep_count, seg_class, status, ids):
        """One call: rows (R, 12) float32, seg_offsets (S + 1), keep_count (S), seg_class (F, C), status, ids (F).
        -> True when the call was stored."""
        F, C = seg_class.shape
        R = len(rows)
        segs = []
        for s in range(C * F):
            f = s // C
            if seg_class.flat[s] < 0 or ids[f] < 0:
                continue
            off = min(max(int(seg_offsets[s]), 0), R)
            segs.append((f, s, off, min(max(int(keep_count[s]), 0), R - off)))
        used, at, calls = (int(v) for v in self.cursor[:3])
        seg_fit = len(segs) <= len(self.image) - used
        row_fit = sum(k for *_, k in segs) <= len(self.rows) - at
        if not (seg_fit and row_fit):
            self.cursor[3] |= (0 if seg_fit else STORE_SEGMENTS) | (0 if row_fit else STORE_ROWS)
            return False
        for j, (f, s, off, keep) in enumerate(segs):
            d = used + j
            self.image[d], self.cls[d] = ids[f], seg_class.flat[s]
            self.frame[d] = np.uint32((calls * F + f) & 0xFFFFFFFF).view(np.int32)
            self.offset[d], self.keep[d] = at, keep
            self.rows[at:at + keep] = rows[off:off + keep]
            at += keep
        self.offset[used + len(segs)] = at
        self.cursor[0], self.cursor[1], self.cursor[2] = used + len(segs), at, calls + 1
        self.cursor[4] |= status
        return True

    def to_dict(self, classes):
        """{image id: {class name: rows}} of the stored segments, in append order."""
        res = {}
        for d in range(int(self.cursor[0])):
            o = self.offset[d]
            res.setdefault(int(self.image[d]), {})[classes[self.cls[d]]] = self.rows[o:o + self.keep[d]].copy()
        return res


def call_tables(rng, F, C, R, p_frame=0.8, max_keep=6, extra=3):
    """A frame call's tables as a frame stage leaves them: frame f's present classes are a random prefix of a
    permutation (segment C f + r holds the r-th, -1 past them), each segment's counted rows lie at seg_offsets[s]
    in segment order with up to `extra` counted rows past its keep_count, and rows are cut at R.
    -> (rows (R, 12) float32, seg_offsets (S + 1), keep_count (S), seg_class (F, C)) int32."""
    S = C * F
    seg_class = np.full((F, C), -1, np.int32)
    counted, keep = np.zeros(S, np.int64), np.zeros(S, np.int32)
    for f in range(F):
        if rng.random() < p_frame:
            n = int(rng.integers(1, C + 1))
            seg_class[f, :n] = rng.permutation(C)[:n]
            k = rng.integers(0, max_keep + 1, n)
            keep[f * C:f * C + n] = k
            counted[f * C:f * C + n] = k + rng.integers(0, extra + 1, n)
    off = np.zeros(S + 1, np.int64)
    np.cumsum(counted, out=off[1:])
    off = np.minimum(off, R)
    keep = np.minimum(keep, np.diff(off)).astype(np.int32)
    rows = rng.standard_normal((R, 12)).astype(np.float32)
    rows.view(np.uint32)[rng.random((R, 12)) < 0.05] = 0x7FC00001          # NaN payloads travel bit for bit
    return rows, off.astype(np.int32), keep, seg_class


def call_dict(rows, seg_offsets, keep_count, seg_class, ids, classes):
    """FrameDetections.to_dict(ids) of a call's tables without the slots of negative id."""
    F, C = seg_class.shape
    res = {}
    for s in range(C * F):
        f = s // C
        if seg_class.flat[s] < 0 or ids[f] < 0:
            continue
        o = seg_offsets[s]
        res.setdefault(int(ids[f]), {})[classes[seg_class.flat[s]]] = rows[o:o + keep_count[s]].copy()
    return res
