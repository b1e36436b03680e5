"""CPU: the refinement stage fed from the collector's device rows (csrc/refine_jobs.cu) restated in numpy and checked
against the dict path's host code: the gather plan (refine_extract.collected_plan) against job_table's job order, the
job kernel (quantization, box array, checks, 2-D drop rule, box record) against job_table / box_record, and the table
kernel (corners, angles, the refine records) against _result / train_inputs.frustum_table; then the ctypes layouts of
the new argument structs and the exports."""
import ctypes as C
from fractions import Fraction
from types import SimpleNamespace

import numpy as np
import pytest

from frustum_convnet_b200 import _lib
from frustum_convnet_b200 import refine_extract as rx
from frustum_convnet_b200.kitti_eval import detection_records
from frustum_convnet_b200.train_inputs import KITTI_CLASSES, frustum_table

STRIDES = [0.1, 0.2, 0.4, 0.8]


def fma(a, b, c):
    """A correctly rounded float64 a * b + c."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


# ------------------------------------------------------------------------------ numpy restatement of the kernels
def restate_job(mode, row, cls_type):
    """rj_jobs_kernel for one collector row -> (status, cut (7,), box record, det corners (8, 3), box2d, prob)."""
    r = detection_records(row.reshape(1, 12), cls_type)[0]
    x1, y1, x2, y2 = r[2:6]
    h, w, l = r[6:9]
    tx, ty, tz = r[9:12]
    ry, score = r[12], r[13]
    box = np.array([tx, ty - h * 0.5, tz, l, w, h, ry])
    st = 0 if np.isfinite(box).all() else _lib.REFINE_ROW_NONFINITE
    if not (l > 0 and w > 0 and h > 0):
        st |= _lib.REFINE_ROW_EXTENTS
    if mode == _lib.REFINE_DET and (y2 - y1 < 5 or x2 - x1 < 1):
        st |= _lib.REFINE_ROW_DROPPED
    cut = box.copy()
    cut[3:6] = cut[3:6] * 1.2
    rec = rx.box_record(cut)
    if mode == _lib.REFINE_DET and st:
        rec["half"] = -1.0
    c, s = np.cos(ry), np.sin(ry)
    corners = np.empty((8, 3))
    for i in range(8):
        xc, yc, zc = _corner(i, l * 0.5, h * 0.5, w * 0.5)
        corners[i] = [(c * xc + s * zc) + box[0], yc + box[1], (-s * xc + c * zc) + box[2]]
    return st, cut, rec, corners, np.array([x1, y1, x2, y2]), score


def _corner(i, hl, hh, hw):
    return (-hl if i & 2 else hl), (hh if i < 4 else -hh), (-hw if (i + 1) & 2 else hw)


def restate_table(cut, strides):
    """rj_table_kernel for one kept job -> (frustum_angle, corners (8, 3), record fields dict, T, degenerate)."""
    c, s = np.cos(cut[6]), np.sin(cut[6])
    hl, hw, hh = cut[3] * 0.5, cut[4] * 0.5, cut[5] * 0.5
    corners = np.empty((8, 3))
    for i in range(8):
        xc, yc, zc = _corner(i, hl, hh, hw)
        corners[i] = [fma(s, zc, c * xc) + cut[0], yc + cut[1], fma(c, zc, -s * xc) + cut[2]]
    pc = (corners[0] + corners[6]) * 0.5
    z1 = -hw
    T = [max(0, int(np.ceil((hw - z1) / st))) for st in strides]
    rec = dict(rot=cut[6], cs=c, sn=s, ref_center=pc, line0=np.array([0.0, 0.0, z1]),
               line_delta=np.array([0.0, 0.0, hw - z1]), z_start=z1, z_step=[(z1 + st) - z1 for st in strides])
    return -np.arctan2(cut[2], cut[0]), corners, rec, T, (min(T) < 1 or hw - z1 == 0)


def _ulp(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


# ------------------------------------------------------------------------------ a collector's host metadata
def random_rows(rng, n):
    rows = np.empty((n, 12), np.float32)
    rows[:, 0] = rng.uniform(0, 1000, n)
    rows[:, 1] = rng.uniform(0, 300, n)
    rows[:, 2] = rows[:, 0] + rng.uniform(0.5, 200, n)
    rows[:, 3] = rows[:, 1] + rng.uniform(2, 150, n)
    rows[:, 4] = rng.uniform(-20, 20, n)
    rows[:, 5] = rng.uniform(0.5, 2.5, n)
    rows[:, 6] = rng.uniform(2, 70, n)
    rows[:, 7] = rng.uniform(0.8, 3, n)
    rows[:, 8] = rng.uniform(0.4, 2.5, n)
    rows[:, 9] = rng.uniform(0.4, 6, n)
    rows[:, 10] = rng.uniform(-np.pi, np.pi, n)
    rows[:, 11] = rng.uniform(0, 1, n)
    return rows


def fake_collected(dets):
    """{idx: {class: rows}} -> (a CollectedDetections-like object with its host metadata and host rows)."""
    segments, keep, rows = [], [], []
    for idx, by_class in dets.items():
        for ct, r in by_class.items():
            segments.append((idx, ct))
            keep.append(len(r))
            rows.append(np.asarray(r, np.float32).reshape(-1, 12))
    off = np.concatenate([[0], np.cumsum(keep)]).astype(np.int32)
    return SimpleNamespace(segments=segments, order=np.arange(len(segments)), host_seg_offsets=off,
                           host_keep_count=np.asarray(keep, np.int32), num_rows=int(off[-1]),
                           rows_h=np.concatenate(rows) if rows else np.zeros((0, 12), np.float32))


def edge_dets(rng):
    """Random rows plus the edge cases: 2-D boxes at exactly 5 px / 1 px after '%.4f', non-whitelisted classes, an
    image without detections (7), an image outside image_ids (99)."""
    d = {3: {"Car": random_rows(rng, 6), "Van": random_rows(rng, 2), "Pedestrian": random_rows(rng, 3)},
         5: {"Cyclist": random_rows(rng, 2), "Car": random_rows(rng, 4)},
         99: {"Car": random_rows(rng, 3)}}
    e = d[5]["Car"]
    e[0, 1], e[0, 3] = 10.00004, 15.00004            # ymax - ymin == 5 after rounding: kept
    e[1, 1], e[1, 3] = 10.0, 14.99994                # 4.9999: dropped
    e[2, 0], e[2, 2] = 20.00004, 21.00004            # xmax - xmin == 1: kept
    e[3, 0], e[3, 2] = 20.0, 20.99994                # dropped
    return d


def jobs_of_plan(plan, col):
    out = []
    for p in range(len(plan["row"])):
        idx, ct = int(plan["image"][p]), plan["types"][p]
        for n in range(int(plan["offsets"][p + 1] - plan["offsets"][p])):
            out.append((idx, ct, n, col.rows_h[plan["row"][p] + n], int(plan["frame"][p])))
    return out


@pytest.mark.parametrize("whitelist", [("Car",), ("Pedestrian", "Cyclist"), ("Car", "Pedestrian", "Cyclist")])
def test_det_jobs_match_job_table(whitelist):
    rng = np.random.RandomState(len(whitelist))
    dets = edge_dets(rng)
    image_ids = [3, 7, 5]
    col = fake_collected(dets)
    plan = rx.collected_plan(image_ids, col, whitelist)
    jobs, _ = rx.job_table(_lib.REFINE_DET, image_ids, rx.RefineFrustumExtractor._dets(dets, image_ids), None,
                           whitelist)
    kept = []
    for idx, ct, n, row, frame in jobs_of_plan(plan, col):
        st, cut, rec, _, box2d, prob = restate_job(_lib.REFINE_DET, row, ct)
        assert plan["frame_ids"][frame] == idx
        if st == 0:
            kept.append((idx, ct, n, cut, rec, box2d, prob))
        else:
            assert st == _lib.REFINE_ROW_DROPPED and (rec["half"] == -1).all()
    assert [(i, c, n) for i, c, n, *_ in kept] == \
        [(jb["frame"], jb["obj"].type, int(jb["obj"].line.rsplit(" ", 1)[1])) for jb in jobs]
    for (idx, ct, n, cut, rec, box2d, prob), jb in zip(kept, jobs):
        assert cut.tobytes() == jb["cut"].tobytes()
        assert rec.tobytes() == rx.box_record(jb["cut"]).tobytes()
        assert box2d.tobytes() == jb["obj"].box2d.tobytes() and prob == jb["obj"].score
    if "Car" in whitelist:
        assert sum(1 for k in kept if k[0] == 5 and k[1] == "Car") == 2            # the 5 px and 1 px boxes stay
    assert rx.iou_thresh(whitelist) == (0.5 if "Car" in whitelist else 0.25)


@pytest.mark.parametrize("bad", ["zero_l", "negative_w", "nan_h", "nan_tx"])
def test_bad_extents_are_flagged_where_job_table_raises(bad):
    rng = np.random.RandomState(9)
    dets = {4: {"Car": random_rows(rng, 3)}}
    col_field, value = {"zero_l": (9, 0.0), "negative_w": (8, -1.0), "nan_h": (7, np.nan), "nan_tx": (4, np.nan)}[bad]
    dets[4]["Car"][1, col_field] = value
    with pytest.raises(ValueError, match=r"detections\[4\]\['Car'\] row 1"):
        rx.job_table(_lib.REFINE_DET, [4], rx.RefineFrustumExtractor._dets(dets, [4]), None, ("Car",))
    st = [restate_job(_lib.REFINE_DET, r, "Car")[0] for r in dets[4]["Car"]]
    assert st[0] == 0 and st[2] == 0
    assert st[1] & (_lib.REFINE_ROW_NONFINITE if bad.startswith("nan") else _lib.REFINE_ROW_EXTENTS)
    if bad == "nan_tx":
        assert st[1] & _lib.REFINE_ROW_NONFINITE
    # matched mode: a non-finite box raises at once, a non-positive extent only once matched
    m = rx.RefineFrustumExtractor._dets(dets, [4])
    gt = {4: [rx.KittiObject("Car", 0, 0, 0, [0, 0, 50, 50], 1.5, 1.6, 3.9, (0, 1, 20), 0)]}
    if bad in ("nan_h", "nan_tx"):
        with pytest.raises(ValueError, match="row 1"):
            rx.job_table(_lib.REFINE_MATCHED, [4], m, gt, ("Car",))
    else:
        jobs, _ = rx.job_table(_lib.REFINE_MATCHED, [4], m, gt, ("Car",))
        assert len(jobs) == 3


def test_matched_plan_skips_images_without_ground_truth():
    rng = np.random.RandomState(4)
    dets = edge_dets(rng)
    col = fake_collected(dets)
    gt = {3: [], 5: [rx.KittiObject("Car", 0, 0, 0, [0, 0, 50, 50], 1.5, 1.6, 3.9, (0, 1, 20), 0)], 7: []}
    plan = rx.collected_plan([3, 7, 5], col, ("Car",), gt)
    jobs, _ = rx.job_table(_lib.REFINE_MATCHED, [3, 7, 5], rx.RefineFrustumExtractor._dets(dets, [3, 7, 5]), gt,
                           ("Car",))
    got = jobs_of_plan(plan, col)
    assert [(i, c) for i, c, *_ in got] == [(jb["frame"], jb["obj"].type) for jb in jobs]
    assert plan["frame_ids"] == [5]
    for (idx, ct, n, row, _), jb in zip(got, jobs):
        st, cut, rec, corners, _, _ = restate_job(_lib.REFINE_MATCHED, row, ct)
        assert cut.tobytes() == jb["cut"].tobytes() and rec.tobytes() == rx.box_record(jb["cut"]).tobytes()
        assert (_ulp(corners, rx.iou_corners(jb["box"])[0]) <= 1).all()


def test_table_matches_result_and_frustum_table():
    rng = np.random.RandomState(7)
    rows = random_rows(rng, 400)
    cuts, types = [], []
    for i, r in enumerate(rows):
        ct = KITTI_CLASSES[i % 3]
        cuts.append(restate_job(_lib.REFINE_DET, r, ct)[1])
        types.append(ct)
    probs = [float(detection_records(r.reshape(1, 12), "Car")[0, 13]) for r in rows]
    host = frustum_table("refine", STRIDES, 70.0, False, KITTI_CLASSES, types, prob_list=probs,
                         pred_box3d_list=[rx.compute_box_3d_obj_array(c) for c in cuts],
                         pred_box3d_size_list=[c[3:6] for c in cuts], pred_box3d_angle_list=[c[6] for c in cuts])
    same = total = 0
    for i, cut in enumerate(cuts):
        fa, corners, rec, T, degenerate = restate_table(cut, STRIDES)
        assert not degenerate
        assert fa == rx.frustum_angle(cut)
        want = rx.compute_box_3d_obj_array(cut)
        assert (_ulp(corners, want) <= 4).all()
        same += int((corners == want).sum())
        total += corners.size
        h = host[i]
        assert list(h["T"][:4]) == T and h["cls_index"] == KITTI_CLASSES.index(types[i]) and h["rgb_prob"] == probs[i]
        for k in ("rot", "cs", "sn", "line0", "line_delta", "z_start"):
            assert np.array(rec[k]).tobytes() == np.array(h[k]).tobytes(), k
        assert np.array(rec["z_step"]).tobytes() == h["z_step"][:4].tobytes()
        assert (_ulp(rec["ref_center"], h["ref_center"]) <= 4).all()
    print("pred_box3d corners bit-identical to numpy's np.dot here: %d / %d" % (same, total))


def test_matched_records_match_frustum_table():
    rng = np.random.RandomState(8)
    rows = random_rows(rng, 100)
    gts = [rx.KittiObject("Car", 0, 0, 0, [0, 0, 50, 50], *map(float, r[7:10]), tuple(map(float, r[4:7])),
                          float(r[10])) for r in random_rows(rng, 100)]
    terms = rx.gt_terms(gts, [rx.obj_array(g) for g in gts])
    cuts = [restate_job(_lib.REFINE_MATCHED, r, "Car")[1] for r in rows]
    b3 = [rx.compute_box_3d_obj_array(rx.obj_array(g)) for g in gts]
    host = frustum_table("refine", STRIDES, 70.0, True, KITTI_CLASSES, ["Car"] * 100, box3d_list=b3,
                         heading_list=[g.ry for g in gts], size_list=[np.array([g.l, g.w, g.h]) for g in gts],
                         pred_box3d_list=[rx.compute_box_3d_obj_array(c) for c in cuts],
                         pred_box3d_size_list=[c[3:6] for c in cuts], pred_box3d_angle_list=[c[6] for c in cuts])
    same = 0
    for i, (cut, t) in enumerate(zip(cuts, terms)):
        pc = restate_table(cut, STRIDES)[2]["ref_center"]
        c, s = np.cos(cut[6]), np.sin(cut[6])
        dx, dy, dz = t["center"] - pc
        center = np.array([fma(dx, c, dz * -s), dy, fma(dx, s, dz * c)])
        h = host[i]
        assert (np.abs(center - h["center"]) <= 4 * np.spacing(np.abs([dx, dy, dz]).max())).all()
        same += int((center == h["center"]).sum())
        assert t["heading"] - cut[6] == h["heading"] and t["dist"] == h["dist"]
        assert t["size"].tobytes() == h["size"].tobytes()
    print("ground-truth centres in the predicted frame bit-identical to numpy's np.dot here: %d / 300" % same)


# ------------------------------------------------------------------------------ C ABI
def test_struct_layouts():
    assert C.sizeof(_lib.RefineJobData) == 12 * 8 + 8
    assert C.sizeof(_lib.RefineGtTerms) == 8 * 8
    assert C.sizeof(_lib.RefineJobsArgs) == 16 + 14 * 8
    assert _lib.RefineJobsArgs.rows.offset == 16 and _lib.RefineJobsArgs.job_data.offset == 16 + 13 * 8
    assert _lib.RefineFrustumTableArgs.stride.offset == 24
    assert _lib.RefineFrustumTableArgs.kept.offset == 24 + 8 * _lib.MAX_SCALES
    assert C.sizeof(_lib.RefineFrustumTableArgs) == 24 + 8 * _lib.MAX_SCALES + 7 * 8
    assert _lib.REFINE_LIST_COLS == 1 + 24 + 3 + 1 + 4 + 1


def test_exports_and_header():
    import os
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                            "frustum_b200.h")).read()
    for name in ("fcn_refine_jobs_from_rows", "fcn_refine_frustum_table"):
        assert name in _lib.SIGNATURES and ("FCN_API int %s(" % name) in hdr
    for m in ("FCN_REFINE_ROW_NONFINITE 1", "FCN_REFINE_ROW_EXTENTS 2", "FCN_REFINE_ROW_DROPPED 4",
              "FCN_REFINE_LIST_COLS 34"):
        assert "#define " + m in hdr
    try:
        lib = _lib.load()
    except RuntimeError:
        pytest.skip("libfrustum_b200.so is not built")
    a = _lib.RefineJobsArgs()
    a.mode = 7
    assert lib.fcn_refine_jobs_from_rows(C.byref(a), None) != 0
    t = _lib.RefineFrustumTableArgs()
    t.mode, t.num_scales = _lib.REFINE_DET, 0
    assert lib.fcn_refine_frustum_table(C.byref(t), None) != 0
    a.mode, a.num_pieces, a.num_jobs = _lib.REFINE_DET, 0, 0
    off = np.zeros(1, np.int32)
    a.host_piece_offsets = a.host_piece_row = off.ctypes.data
    assert lib.fcn_refine_jobs_from_rows(C.byref(a), None) == 0           # nothing to do, nothing launched
