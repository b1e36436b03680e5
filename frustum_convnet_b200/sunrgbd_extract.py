"""SUN-RGBD frustums on the device: extract_frustum_data and extract_frustum_data_from_rgb_detection of the reference's
sunrgbd/prepare_data.py (--gen_train, --gen_val, --gen_val_rgb_detection) without their pickles, for a whole set of
frames in one call.

    sx = SunrgbdFrustumExtractor()
    train = sx.from_ground_truth(points, calibs, train_ids, "mysunrgbd/training/label", perturb=True, augment=5)
    val   = sx.from_ground_truth(points, calibs, val_ids, "mysunrgbd/training/label")
    det   = sx.from_rgb_detections(points, calibs, *read_det_file("rgb_det_val.txt"))
    tb = TrainBatchBuilder.from_frustums(train, "sunrgbd", strides=cfg.DATA.STRIDE, npoints=cfg.DATA.NUM_SAMPLES)

``points[idx]`` is the frame's (n, 6) float32 cloud (x, y, z, r, g, b in upright depth coordinates; numpy or a CUDA
tensor), ``calibs[idx]`` a dict (or object) with 'Rtilt' and 'K', 3 x 3 float64 (read_calib).

  from_ground_truth    extract_frustum_data (:132-267): every label object of a whitelisted class, in line order,
                       `augment` times; with perturb, its 2-D box shifted and scaled by random_shift_box2d
                       (sunrgbd_utils.py:208-221: four rng.random() draws, no clip, no retry).  A box with a zero extent
                       is skipped after its draws (the reference's Qhull raises).  Labels: the points in its 3-D box.
                       A job is dropped when fewer than 5 of its kept points are labelled.
  from_rgb_detections  extract_frustum_data_from_rgb_detection (:270-381) on read_det_file's four lists: the
                       valid_ids filter, then the whitelist; a job is dropped when it keeps fewer than 5 points.
Every job cuts u < xmax, u >= xmin, v < ymax, v >= ymin out of the whole cloud (no image-bounds test), and keeps at
most 2048 points: np.random.choice(n, 2048, replace=False) from `rng` when it has more, in the reference's order.  How
far that draw moves the generator depends on n, and in the perturbed set the next box is drawn after it, so the host
learns each count from the device before it draws (replay: counted in rounds).  Every per-job constant (perturbation,
frustum_angle, corners, size, heading, float32 box2d) is computed here with the reference's own numpy expressions;
nothing random runs on the device.  "In the 3-D box" is the float64 half-space test of csrc/box_contains.cuh where the
reference triangulates the corners with scipy's Delaunay: the two agree except for points within rounding (~1e-9 m) of
a face.  No CPU fallback: CPU tensors and devices raise."""
from __future__ import annotations

import ctypes as C
import os
import pickle

import numpy as np
import torch

from . import _lib
from ._host import csr_offsets, cuda_device, upload
from .frustum_extract import LabelledFrustums, _scan, empty_outputs, frame_order, run_extract

TYPE_WHITELIST = ("bed", "table", "sofa", "chair", "toilet", "desk", "dresser", "night_stand", "bookshelf",
                  "bathtub")                         # prepare_data.py:405-408 (--num_classes 10)
SHIFT_RATIO = 0.1
CAP = _lib.SUNRGBD_MAX_POINTS                        # prepare_data.py:220
MIN_POINTS = 5                                       # :226, :352
MAX_WINDOW = 1024
GT_KEYS = (("id", "id_list"), ("box2d", "box2d_list"), ("box3d", "box3d_list"), ("box3d_size", "size_list"),
           ("box3d_heading", "heading_list"), ("type", "type_list"), ("input", None), ("frustum_angle",
           "frustum_angle_list"), ("label", None), ("calib_K", "calib_K_list"), ("calib_R", "calib_R_list"))
DET_KEYS = (("id", "id_list"), ("type", "type_list"), ("box2d", "box2d_list"), ("box2d_prob", "prob_list"),
            ("input", None), ("frustum_angle", "frustum_angle_list"), ("calib_K", "calib_K_list"),
            ("calib_R", "calib_R_list"))             # the pickled dicts (:249-262, :366-376)


# ------------------------------------------------------------------------------ readers (sunrgbd_utils.py)
class SUNObject3d:
    """sunrgbd_utils.SUNObject3d (:16-40): one label line."""

    def __init__(self, line, where=""):
        data = line.split(" ")
        data[1:] = [float(x) for x in data[1:]]
        self.line = where
        self.classname = data[0]
        self.xmin = data[1]
        self.ymin = data[2]
        self.xmax = data[1] + data[3]
        self.ymax = data[2] + data[4]
        self.box2d = np.array([self.xmin, self.ymin, self.xmax, self.ymax])
        self.centroid = np.array([data[5], data[6], data[7]])
        self.w = data[8]
        self.l = data[9]
        self.h = data[10]
        self.orientation = np.zeros((3,))
        self.orientation[0] = data[15]
        self.orientation[1] = data[16]
        self.heading_angle = -1 * np.arctan2(self.orientation[1], self.orientation[0])


def read_label(path):
    """read_sunrgbd_label: one SUNObject3d per line ('path:line' names each)."""
    with open(path) as f:
        return [SUNObject3d(ln.rstrip(), "%s:%d" % (path, k + 1)) for k, ln in enumerate(f)]


def read_calib(path):
    """SUNRGBD_Calibration's file reader (:74-80): line 1 Rtilt, line 2 K, 9 values each in column-major order."""
    with open(path) as f:
        lines = [ln.rstrip() for ln in f]
    Rtilt = np.reshape(np.array([float(x) for x in lines[0].split(" ")]), (3, 3), order="F")
    K = np.reshape(np.array([float(x) for x in lines[1].split(" ")]), (3, 3), order="F")
    return {"Rtilt": Rtilt, "K": K}


def read_det_file(path):
    """prepare_data.read_det_file (:88-102): 'data_idx type prob xmin ymin xmax ymax' lines ->
    (id_list, type_list, box2d_list, prob_list)."""
    id_list, type_list, prob_list, box2d_list = [], [], [], []
    with open(path) as f:
        for line in f:
            t = line.rstrip().split(" ")
            id_list.append(int(t[0]))
            type_list.append(t[1])
            prob_list.append(float(t[2]))
            box2d_list.append(np.array([float(t[i]) for i in range(3, 7)]))
    return id_list, type_list, box2d_list, prob_list


def objects_of(gt, image_ids):
    """A label directory (%06d.txt files) or {idx: [SUNObject3d]} -> {idx: [SUNObject3d]} for image_ids."""
    if isinstance(gt, (str, os.PathLike)):
        return {int(i): read_label(os.path.join(gt, "%06d.txt" % int(i))) for i in image_ids}
    return gt


def calib_mats(calib):
    """(Rtilt, K) of a calib dict or SUNRGBD_Calibration-like object, checked: 3 x 3 and finite."""
    out = []
    for name in ("Rtilt", "K"):
        m = calib[name] if isinstance(calib, dict) else getattr(calib, name)
        m = np.asarray(m)
        if m.shape != (3, 3) or not np.isfinite(m.astype(np.float64)).all():
            raise ValueError("calib %s must be a finite 3 x 3 matrix, got shape %s" % (name, m.shape))
        out.append(m)
    return out


# ------------------------------------------------------------------------------ per-job constants (host, float64)
def random_shift_box2d(box2d, rng=np.random, shift_ratio=SHIFT_RATIO):
    """sunrgbd_utils.random_shift_box2d (:208-221) with the generator as an argument."""
    r = shift_ratio
    xmin, ymin, xmax, ymax = box2d
    h = ymax - ymin
    w = xmax - xmin
    cx = (xmin + xmax) / 2.0
    cy = (ymin + ymax) / 2.0
    cx2 = cx + w * r * (rng.random() * 2 - 1)
    cy2 = cy + h * r * (rng.random() * 2 - 1)
    h2 = h * (1 + rng.random() * 2 * r - r)
    w2 = w * (1 + rng.random() * 2 * r - r)
    return np.array([cx2 - w2 / 2.0, cy2 - h2 / 2.0, cx2 + w2 / 2.0, cy2 + h2 / 2.0])


def flip_axis_to_camera(pc):
    pc2 = np.copy(pc)
    pc2[:, [0, 1, 2]] = pc2[:, [0, 2, 1]]
    pc2[:, 1] *= -1
    return pc2


def flip_axis_to_depth(pc):
    pc2 = np.copy(pc)
    pc2[:, [0, 1, 2]] = pc2[:, [0, 2, 1]]
    pc2[:, 2] *= -1
    return pc2


def project_upright_depth_to_image(pc, Rtilt, K):
    """sunrgbd_utils.py:109-123 -> (n, 2) float64 u, v."""
    pc2 = flip_axis_to_camera(np.transpose(np.dot(np.transpose(Rtilt), np.transpose(pc[:, 0:3]))))
    uv = np.dot(pc2, np.transpose(K))
    uv[:, 0] /= uv[:, 2]
    uv[:, 1] /= uv[:, 2]
    return uv[:, 0:2]


def frustum_angle(box, Rtilt, K):
    """-arctan2 of project_image_to_upright_camera of the box centre at depth 20 (prepare_data.py:196-204,
    sunrgbd_utils.py:131-145)."""
    xmin, ymin, xmax, ymax = box
    uvdepth = np.zeros((1, 3))
    uvdepth[0, 0:2] = np.array([(xmin + xmax) / 2.0, (ymin + ymax) / 2.0])
    uvdepth[0, 2] = 20
    f_u, f_v, c_u, c_v = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    x = ((uvdepth[:, 0] - c_u) * uvdepth[:, 2]) / f_u
    y = ((uvdepth[:, 1] - c_v) * uvdepth[:, 2]) / f_v
    cam = np.zeros((1, 3))
    cam[:, 0], cam[:, 1], cam[:, 2] = x, y, uvdepth[:, 2]
    upright = flip_axis_to_camera(np.transpose(np.dot(Rtilt, np.transpose(flip_axis_to_depth(cam)))))
    return -1 * np.arctan2(upright[0, 2], upright[0, 0])


def box3d_corners(obj):
    """compute_box_3d's (8, 3) corners (sunrgbd_utils.py:237-268) flipped to upright camera coordinates
    (prepare_data.py:207-208)."""
    t = -1 * obj.heading_angle
    c, s = np.cos(t), np.sin(t)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    l, w, h = obj.l, obj.w, obj.h
    x_corners = [-l, l, l, -l, -l, l, l, -l]
    y_corners = [w, w, -w, -w, w, w, -w, -w]
    z_corners = [h, h, h, h, -h, -h, -h, -h]
    corners_3d = np.dot(R, np.vstack([x_corners, y_corners, z_corners]))
    corners_3d[0, :] += obj.centroid[0]
    corners_3d[1, :] += obj.centroid[1]
    corners_3d[2, :] += obj.centroid[2]
    return flip_axis_to_camera(np.transpose(corners_3d))


def box_record(obj):
    """The label box as an fcn_refine_box: centre (cx, -cz, cy) and half extents (l, h, w) along the box's local x
    (heading), camera y (up, flipped) and local y; cs, sn = cos, sin of heading_angle.  The corners
    rotz(-heading) (a, b, c) + centroid, flipped to (x, -z, y), invert to a = cs dx - sn dz and b = sn dx + cs dz
    for dx = x - cx, dz = z_cam - cy.  Negative extents describe the same corners as their absolute values."""
    rec = np.zeros(1, dtype=np.dtype(_lib.RefineBox))[0]
    cx, cy, cz = (float(v) for v in obj.centroid)
    rec["center"] = (cx, -cz, cy)
    rec["half"] = (abs(obj.l), abs(obj.h), abs(obj.w))
    rec["cs"], rec["sn"] = np.cos(obj.heading_angle), np.sin(obj.heading_angle)
    return rec


def _check_obj(obj):
    v = np.concatenate([obj.box2d, obj.centroid, [obj.l, obj.w, obj.h, obj.heading_angle]])
    if not np.isfinite(v).all():
        raise ValueError("%s: the label box must be finite" % (obj.line or obj.classname))


def zero_extent(obj):
    """The reference's Qhull raises on a box with a zero extent; the job is skipped (prepare_data.py:209-213)."""
    return obj.l == 0 or obj.w == 0 or obj.h == 0


# ------------------------------------------------------------------------------ the draws (host)
def replay(slots, perturb, rng, count, window=MAX_WINDOW):
    """The reference's generator stream over the jobs `slots` (dicts with 'box' (4,) float64 and 'skip'), in order:
    for each, its cutting box (four random() draws when perturb), then, unless skipped, np.random.choice(n, 2048,
    replace=False) when its in-box count n exceeds 2048.

    count(begin, end, cuts) counts the live (not skipped) jobs [begin, end) (numbered among the live jobs) cut by
    `cuts` and returns their n.  Unperturbed: one count of every job, then the draws.  Perturbed: in rounds; a round
    draws the boxes of up to `window` jobs from a saved state as if none needed a choice, counts them and accepts the
    jobs up to and including the first with n > 2048; for that job it restores the state, draws the accepted boxes
    again (the same values) and then the choice.  The window doubles (up to `window`) after a fully accepted round
    and drops to 1 after a rejection.
    -> (cuts (S, 4) float64, n (S,) int64 (-1 for skipped), {slot: choice}, rounds)."""
    S = len(slots)
    live = np.array([not s["skip"] for s in slots], dtype=bool)
    lid = np.cumsum(live) - 1                       # the live number of each live slot
    n = np.full(S, -1, np.int64)
    choices, rounds = {}, 0
    if not perturb:
        cuts = np.array([s["box"] for s in slots], dtype=np.float64).reshape(S, 4)
        if live.any():
            n[live] = count(0, int(live.sum()), cuts[live])
            rounds = 1
        for k in np.flatnonzero(live & (n > CAP)).tolist():
            choices[k] = rng.choice(int(n[k]), CAP, replace=False)
        return cuts, n, choices, rounds
    cuts = np.zeros((S, 4), np.float64)
    start, w = 0, 1
    while start < S:
        state = rng.get_state()
        end = min(S, start + w)
        win = np.array([random_shift_box2d(slots[k]["box"], rng) for k in range(start, end)]).reshape(-1, 4)
        cuts[start:end] = win
        ks = [k for k in range(start, end) if live[k]]
        if ks:
            n[ks] = count(int(lid[ks[0]]), int(lid[ks[-1]]) + 1, win[np.array(ks) - start])
            rounds += 1
        first = next((k for k in ks if n[k] > CAP), None)
        if first is None:
            start, w = end, min(2 * w, window)
            continue
        rng.set_state(state)
        for k in range(start, first + 1):
            random_shift_box2d(slots[k]["box"], rng)
        choices[first] = rng.choice(int(n[first]), CAP, replace=False)
        n[first + 1:end] = -1
        start, w = first + 1, 1
    return cuts, n, choices, rounds


# ------------------------------------------------------------------------------ result
class SunrgbdFrustums(LabelledFrustums):
    """One extraction (LabelledFrustums): points (M, 6) float32 (x, -z, y, r, g, b: upright camera coordinates and
    colour), label (M) uint8 (None for detections).  The lists are the provider's (provider_sample_sunrgbd.py:89-109);
    rounds is the number of count rounds the draws took."""

    def __init__(self, points, offsets, label, counts, job_index, lists, stream=None, rounds=0):
        super().__init__(points, offsets, label, counts, job_index, stream)
        self.has_labels = label is not None
        for n, v in lists.items():
            setattr(self, n, v)
        self.rounds = rounds

    def label_list(self):
        """The per-frustum (n,) bool labels (True inside the 3-D box), copied to the host."""
        if not self.has_labels:
            raise ValueError("frustums from detections have no labels")
        self.wait()
        return self._split(self.label.cpu().numpy().astype(bool))

    def to_pickle(self, path):
        """The reference's dict (its keys, bool labels, protocol -1): provider_sample_sunrgbd.ProviderDataset reads it
        unchanged."""
        keys = GT_KEYS if self.has_labels else DET_KEYS
        values = {"input": self.input_list()}
        if self.has_labels:
            values["label"] = self.label_list()
        d = {k: values[k] if n is None else list(getattr(self, n)) for k, n in keys}
        with open(path, "wb") as fp:
            pickle.dump(d, fp, -1)


def _job_lists(jobs, labelled):
    L = {n: [] for n in ("id_list", "type_list", "box2d_list", "frustum_angle_list", "calib_K_list", "calib_R_list")}
    if labelled:
        L.update(box3d_list=[], size_list=[], heading_list=[])
    else:
        L["prob_list"] = []
    for jb in jobs:
        Rtilt, K = jb["calib"]
        cut = jb["cut"]
        L["id_list"].append(jb["frame"])
        L["type_list"].append(jb["type"])
        L["frustum_angle_list"].append(frustum_angle(cut, Rtilt, K))
        L["calib_K_list"].append(K)
        L["calib_R_list"].append(Rtilt)
        if labelled:
            obj = jb["obj"]
            xmin, ymin, xmax, ymax = cut
            L["box2d_list"].append(np.array([xmin, ymin, xmax, ymax], dtype=np.float32))
            L["box3d_list"].append(box3d_corners(obj))
            L["heading_list"].append(obj.heading_angle)
            L["size_list"].append(np.array([2 * obj.l, 2 * obj.w, 2 * obj.h]))
        else:
            L["box2d_list"].append(jb["box"])
            L["prob_list"].append(jb["prob"])
    return L


class SunrgbdFrustumExtractor:
    def __init__(self, type_whitelist=TYPE_WHITELIST, device=None):
        self.type_whitelist = frozenset(type_whitelist)
        self.device = cuda_device(device, "SunrgbdFrustumExtractor")

    def from_ground_truth(self, points, calibs, image_ids, gt, perturb=False, augment=1, rng=np.random,
                          stream=None, timer=None, window=MAX_WINDOW):
        """gt: a label directory or {idx: [SUNObject3d]}.  rng: the np.random module or a RandomState; it carries
        across calls.  `timer(name)` (optional, benchmarks) is called with "start", "project", then "round_start"
        and "round_end" around each count round, "count", "select", "write_start" and "write"."""
        gt = objects_of(gt, image_ids)
        slots = []
        for idx in image_ids:
            idx = int(idx)
            if idx not in gt:
                raise ValueError("no label objects for frame %d" % idx)
            for obj in gt[idx]:
                if obj.classname not in self.type_whitelist:
                    continue
                _check_obj(obj)
                skip = zero_extent(obj)
                for _ in range(int(augment)):
                    slots.append(dict(frame=idx, box=obj.box2d, obj=obj, type=obj.classname, skip=skip))
        return self._run(points, calibs, slots, True, perturb, rng, stream, timer, window)

    def from_rgb_detections(self, points, calibs, id_list, type_list, box2d_list, prob_list, valid_ids=None,
                            rng=np.random, stream=None, timer=None):
        """read_det_file's four lists (in its order: ids, types, boxes, probabilities)."""
        n = len(id_list)
        if len(type_list) != n or len(prob_list) != n or len(box2d_list) != n:
            raise ValueError("id_list, type_list, box2d_list and prob_list must have the same length")
        slots = []
        for i in range(n):
            idx = id_list[i]
            if valid_ids is not None and idx not in valid_ids:
                continue
            if type_list[i] not in self.type_whitelist:
                continue
            box = np.asarray(box2d_list[i])
            if box.shape != (4,) or not np.isfinite(box.astype(np.float64)).all():
                raise ValueError("detection line %d: the 2-D box must be 4 finite values" % i)
            slots.append(dict(frame=int(idx), box=box, type=type_list[i], prob=prob_list[i], skip=False))
        return self._run(points, calibs, slots, False, False, rng, stream, timer, MAX_WINDOW)

    # ------------------------------------------------------------------ device calls
    def _run(self, points, calibs, slots, labelled, perturb, rng, stream, timer, window):
        dev = self.device
        mark = timer if timer is not None else (lambda name: None)
        for s in slots:
            if not np.isfinite(np.asarray(s["box"], dtype=np.float64)).all():
                raise ValueError("%s: the 2-D box must be finite" % (s["obj"].line if "obj" in s else "a box"))
        jobs = [s for s in slots if not s["skip"]]
        frame_ids, fpos = frame_order(jb["frame"] for jb in jobs)
        for k in frame_ids:
            if k not in points or k not in calibs:
                raise ValueError("frame %d has no point cloud or no calibration" % k)
        mats = {k: calib_mats(calibs[k]) for k in frame_ids}
        J, F = len(jobs), len(frame_ids)
        stream = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.device(dev), torch.cuda.stream(stream):
            sc = [_scan(points[k], dev, "SunrgbdFrustumExtractor", 6) for k in frame_ids]
            so = csr_offsets([s.shape[0] for s in sc])
            if J == 0:                                  # nothing to count: only the skipped jobs' box draws
                replay(slots, perturb, rng, None)
                return SunrgbdFrustums(*empty_outputs(dev, 6, labelled), np.zeros(0, np.int64), np.zeros(0, np.int64),
                                       _job_lists([], labelled), stream)
            frames = np.zeros(F, dtype=np.dtype(_lib.SunrgbdFrame))
            for k in frame_ids:
                frames[fpos[k]]["Rtilt"] = np.asarray(mats[k][0], np.float64).reshape(9)
                frames[fpos[k]]["K"] = np.asarray(mats[k][1], np.float64).reshape(9)
            rec = np.zeros(J, dtype=np.dtype(_lib.GtJob))
            rec["frame"] = [fpos[jb["frame"]] for jb in jobs]
            rec["label"] = np.arange(J) if labelled else -1
            if not perturb:
                rec["box"] = np.array([np.asarray(jb["box"], np.float64) for jb in jobs]).reshape(J, 4)
            boxes = np.array([box_record(jb["obj"]) for jb in jobs] if labelled else np.zeros(0),
                             dtype=np.dtype(_lib.RefineBox))
            inp, (d_frames, d_jobs, d_boxes, d_so) = upload([frames, rec, boxes, so], dev)
            a = _lib.SunrgbdExtractArgs()
            a.num_frames, a.num_points, a.num_jobs = F, int(so[-1]), J
            a.num_labels, a.labelled = (J if labelled else 0), int(labelled)
            a.scan_offsets, a.frames, a.jobs = d_so, d_frames, d_jobs
            a.label_boxes = d_boxes if labelled else None
            jb_bytes = C.sizeof(_lib.GtJob)
            jobs_dev = inp[d_jobs - inp.data_ptr():d_jobs - inp.data_ptr() + J * jb_bytes]
            live = np.flatnonzero([not s["skip"] for s in slots])
            cuts = rounds = sel = None

            def count(words):
                nonlocal cuts, rounds, sel          # sel: the choice tables, alive until the write is enqueued
                _lib.call("fcn_sunrgbd_extract_project", C.byref(a), stream.cuda_stream)
                mark("project")

                def count_round(begin, end, win):
                    if perturb:
                        rec["box"][begin:end] = win
                        jobs_dev[begin * jb_bytes:end * jb_bytes].copy_(torch.from_numpy(rec[begin:end].view(np.uint8)))
                    a.job_begin, a.job_end = begin, end
                    mark("round_start")
                    _lib.call("fcn_sunrgbd_extract_count", C.byref(a), stream.cuda_stream)
                    mark("round_end")
                    return words[begin:end].cpu().numpy()

                cuts, n, choices, rounds = replay(slots, perturb, rng, count_round, window)
                mark("count")
                job_choice = np.full(J, -1, np.int32)
                ranks = np.zeros((len(choices), CAP), np.int32)
                order = np.zeros((len(choices), CAP), np.int32)
                for c, k in enumerate(sorted(choices)):       # job order
                    ch = np.asarray(choices[k])
                    order[c] = np.argsort(ch, kind="stable")
                    ranks[c] = ch[order[c]]
                    job_choice[np.searchsorted(live, k)] = c
                sel, (d_choice, d_ranks, d_slots) = upload([job_choice, ranks, order], dev)
                a.num_choices, a.job_choice, a.choice_ranks, a.choice_slots = len(choices), d_choice, d_ranks, d_slots
                _lib.call("fcn_sunrgbd_extract_select", C.byref(a), stream.cuda_stream)
                mark("select")

            words, kept, out = run_extract(
                "sunrgbd_extract", a, sc, so, J, ("job_points", "job_labelled"),
                lambda K, M, words: {"labels": torch.empty(M, dtype=torch.uint8, device=dev) if labelled else None},
                dev, stream, timer, "jobs reference no frame or label box, or disagree with their draws", count=count,
                cols=6)
        kept_slots = live[kept]
        for k in kept_slots.tolist():
            slots[k]["cut"] = cuts[k]
            slots[k]["calib"] = mats[slots[k]["frame"]]
        lists = _job_lists([slots[k] for k in kept_slots.tolist()], labelled)
        return SunrgbdFrustums(out["points"], out["offsets"], out["labels"], words[kept].astype(np.int64),
                               kept_slots.astype(np.int64), lists, stream, rounds)
