"""CPU: tests/frame_ref.py, the restatement of fcn_frame_extract's tables that tests/test_gpu_frame_stages.py holds
the device to, checked against oracle/frustum_extract and on hand-built slot tables."""
import numpy as np

import frame_ref as fr
from oracle.frustum_extract import extract

NAMES = ("Car", "Pedestrian", "Cyclist")


def test_unlimited_budget_keeps_what_the_oracle_keeps():
    """With P_out above every frame's points the batch is oracle/frustum_extract's kept list over the clamped
    frames: the same frustums in (frame, detection) order, points, boxes, angles, P and scores; dummies after."""
    rng = np.random.default_rng(5)
    frames = fr.synth_frames(rng, 4, 3000, 6)
    P, D = 2500, 5                                   # every scan and detection list is cut
    inp = fr.stage(frames, P, D)
    t = fr.frame_tables(*inp, P_out=1 << 23, class_mask=0b101)
    assert t["status"] == fr.SCAN_POINTS | fr.DETS
    ids, types, probs, boxes = [], [], [], []
    for f, (_, _, _, dets) in enumerate(frames):
        for c, p, b in dets[:D]:
            ids.append(f), types.append(NAMES[c]), probs.append(np.float32(p)), boxes.append(b)
    want = extract({f: x[0][:P] for f, x in enumerate(frames)}, {f: x[1] for f, x in enumerate(frames)},
                   {f: x[2] for f, x in enumerate(frames)}, ids, types, probs, boxes,
                   type_whitelist=("Car", "Cyclist"))
    w_ids, w_box, w_pts, w_types, w_angle, w_prob, _ = want
    K = len(w_ids)
    assert 0 < K < 4 * D and int(t["valid"].sum()) == K
    assert t["valid"][:K].all() and not t["valid"][K:].any()
    assert [int(d) // D for d in t["det_index"][:K]] == list(w_ids)
    assert [NAMES[c] for c in t["cls_index"][:K]] == list(w_types)
    off = t["offsets"]
    for k in range(K):
        assert np.array_equal(t["points"][off[k]:off[k + 1]], w_pts[k])
    assert np.array_equal(t["box2d"][:K], np.array(w_box))
    assert np.array_equal(t["frustum_angle"][:K], np.array(w_angle))
    assert np.array_equal(t["rgb_prob"][:K], np.array(w_prob, np.float32))
    for k in range(K):
        assert np.array_equal(t["P"][k], frames[w_ids[k]][1]["P2"])
    # dummies: one point at the origin each, box (0, 0, 1, 1), a unit P, no slot
    assert np.array_equal(np.diff(off[K:]), np.ones(4 * D - K)) and not t["points"][off[K]:].any()
    assert (t["det_index"][K:] == -1).all() and (t["box2d"][K:] == [0, 0, 1, 1]).all()
    assert (t["P"][K:] == fr.UNIT_P).all()


def test_budget_keeps_the_longest_prefix_that_fits():
    dp = [5, -1, 3, 4, 2]                            # points of each kept slot, -1: dropped by the count pass
    assert fr.budget(dp, 14).tolist() == dp                         # filled exactly
    assert fr.budget(dp, 13).tolist() == [5, -1, 3, 4, -1]          # one point over: the last one drops
    assert fr.budget(dp, 8).tolist() == [5, -1, 3, -1, -1]          # a later small one fits no more once one drops
    assert fr.budget(dp, 4).tolist() == [-1] * 5                    # a large first frustum drops every one
    assert fr.budget([-1, -1], 1).tolist() == [-1, -1]


def test_class_ranks_count_only_the_slots_that_fit():
    rank, seg_class = fr.class_ranks([1, 0, 1, 2], [True, True, True, True])
    assert rank == [1, 0, 2] and seg_class.tolist() == [1, 0, 2]
    # a Pedestrian kept, then the frame's only Car and Cyclist dropped for the budget: one segment, Pedestrian's
    rank, seg_class = fr.class_ranks([1, 0, 2], [True, False, False])
    assert rank == [-1, 0, -1] and seg_class.tolist() == [1, -1, -1]
    rank, seg_class = fr.class_ranks([0, 0], [False, False])
    assert rank == [-1, -1, -1] and seg_class.tolist() == [-1, -1, -1]


def test_budget_drops_whole_classes_from_the_segment_table():
    """A frame whose later frustums exceed P_out: the dropped frustums' classes get no segment, the kept ones keep
    their ranks, and bit 4 is set."""
    rng = np.random.default_rng(9)
    frames = fr.synth_frames(rng, 1, 4000, 3, classes=(1, 0, 2))
    inp = fr.stage(frames, 4000, 3)
    full = fr.frame_tables(*inp, P_out=1 << 23)
    dp = full["det_points"]
    assert (dp > 0).all() and full["seg_class"][0].tolist() == [frames[0][3][0][0], frames[0][3][1][0],
                                                                frames[0][3][2][0]]
    t = fr.frame_tables(*inp, P_out=int(dp[0]))
    assert t["status"] == fr.OUT_POINTS
    assert t["valid"].tolist() == [1, 0, 0]
    assert t["seg_class"][0].tolist() == [frames[0][3][0][0], -1, -1] and t["seg"][0] == 0
    t = fr.frame_tables(*inp, P_out=int(dp.sum()))
    assert t["status"] == 0 and t["valid"].tolist() == [1, 1, 1]


def test_counts_and_bad_detections_set_their_bits():
    rng = np.random.default_rng(11)
    frames = fr.synth_frames(rng, 3, 500, 3)
    scans, sc, calibs, hw, boxes, cls, prob, dc = fr.stage(frames, 400, 3, scan_counts=[-1, 400, 401],
                                                           det_counts=[3, -1, 4])
    cls[0, 1] = 3
    boxes[0, 2, 1] = np.nan
    t = fr.frame_tables(scans, sc, calibs, hw, boxes, cls, prob, dc, P_out=1 << 20)
    assert t["status"] == fr.SCAN_POINTS | fr.DETS | fr.BAD_DET
    # frame 0 has no points, frame 1 no detections: only frame 2's can be kept
    assert all(d // 3 == 2 for d in t["det_index"] if d >= 0)
