"""CPU: tests/sunrgbd_frame_ref.py, the restatement of fcn_sunrgbd_frame_extract that tests/test_gpu_sunrgbd_frame.py
holds the device to, checked against oracle/sunrgbd_extract over whole frame sets and on hand-built slot tables."""
import numpy as np

import sunrgbd_frame_ref as sr
from frustum_convnet_b200 import _lib
from frustum_convnet_b200.train_inputs import SUNRGBD_CLASSES, frustum_table
from oracle import sunrgbd_extract as ox
from resample_ref import choice_row

STRIDES, MAX_DEPTH = (0.1, 0.2, 0.4, 0.8, 1.6), 8.0
SEED, CALL = 77, 2 ** 62 + 3


def _tables(inp, P_out=1 << 23, class_mask=(1 << 10) - 1):
    return sr.frame_tables(*inp, P_out=P_out, class_mask=class_mask, seed=SEED, call=CALL, strides=STRIDES,
                           max_depth=MAX_DEPTH)


def test_unlimited_budget_keeps_what_the_oracle_keeps():
    """With P_out above every frame's points the batch is oracle/sunrgbd_extract's kept list over all the clamped
    frames at once (its generator drawing each capped job's row under that job's slot): the same frustums in (frame,
    detection) order, points in choice order, angles and records; dummies after."""
    frames = sr.synth_frames(3, 3)
    P, D = 70000, 5                                  # every cloud and detection list is cut
    inp = sr.stage(frames, P, D)
    mask = sum(1 << c for c in {d[0] for _, _, dets in frames for d in dets[1:3]})
    t = _tables(inp, class_mask=mask)
    assert t["status"] == sr.SCAN_POINTS | sr.DETS
    ids, types, probs, boxes, rows = [], [], [], [], []
    for f, (_, _, dets) in enumerate(frames):
        for j, (c, p, b) in enumerate(dets[:D]):
            ids.append(f), types.append(SUNRGBD_CLASSES[c]), probs.append(p), boxes.append(b)
            n = t["det_points"][f * D + j]
            if n > sr.CAP:
                rows.append((int(n), choice_row(int(n), sr.CAP, SEED, f * D + j, CALL)))
    wl = [c for i, c in enumerate(SUNRGBD_CLASSES) if (mask >> i) & 1]
    L, trace = ox.from_rgb_detections({f: x[0][:P] for f, x in enumerate(frames)},
                                      {f: x[1] for f, x in enumerate(frames)}, ids, types, boxes, probs,
                                      type_whitelist=wl, rng=sr._Rows(rows))
    K = len(L["id"])
    assert 0 < K < 3 * D and int(t["valid"].sum()) == K
    assert any(len(p) == sr.CAP for p in L["input"]) and any(len(p) < sr.CAP for p in L["input"])
    assert t["valid"][:K].all() and not t["valid"][K:].any()
    assert [int(d) // D for d in t["det_index"][:K]] == list(L["id"])
    assert [SUNRGBD_CLASSES[c] for c in t["cls_index"][:K]] == list(L["type"])
    off = t["offsets"]
    for k in range(K):
        assert np.array_equal(t["points"][off[k]:off[k + 1]], L["input"][k])
    assert np.array_equal(t["angle"][:K], np.array(L["frustum_angle"]))
    assert np.array_equal(t["rgb_prob"][:K], np.array(L["box2d_prob"], np.float32))
    assert np.array_equal(t["box2d"][:K], np.array(L["box2d"], np.float32))
    want = frustum_table("sunrgbd", STRIDES, MAX_DEPTH, False, SUNRGBD_CLASSES, L["type"],
                         frustum_angle_list=L["frustum_angle"], box2d_list=L["box2d"], calib_K_list=L["calib_K"],
                         calib_R_list=L["calib_R"], prob_list=L["box2d_prob"])
    assert t["records"][:K].tobytes() == want.tobytes()
    # dummies: one point at the origin each, box (0, 0, 1, 1), no slot, the unit record with the fixed T
    assert np.array_equal(np.diff(off[K:]), np.ones(3 * D - K)) and not t["points"][off[K]:].any()
    assert (t["det_index"][K:] == -1).all() and (t["box2d"][K:] == [0, 0, 1, 1]).all()
    dummy = t["records"][K:]
    assert (dummy["rot"] == np.pi / 2).all() and (dummy["K"] == np.eye(3).reshape(9)).all()
    assert (dummy["Rtilt"] == np.eye(3).reshape(9)).all() and (dummy["T"][:, :5] == [80, 40, 20, 10, 5]).all()
    # the cap rows: the slot's draw for every candidate with n > 2048, zeros elsewhere
    for d in range(3 * D):
        n = t["det_points"][d]
        assert np.array_equal(t["cap_choice"][d], choice_row(int(n), sr.CAP, SEED, d, CALL) if n > sr.CAP else
                              np.zeros(sr.CAP, np.int32)), d


def test_budget_keeps_the_longest_prefix_that_fits():
    dp = [2048, -1, 300, 1500, 40]
    assert sr.budget(dp, 3888).tolist() == dp                          # filled exactly
    assert sr.budget(dp, 3887).tolist() == [2048, -1, 300, 1500, -1]   # one point over: the last one drops
    assert sr.budget(dp, 2400).tolist() == [2048, -1, 300, -1, -1]     # a later small one fits no more
    assert sr.budget(dp, 2047).tolist() == [-1] * 5                    # below the first frustum: none
    assert sr.budget([-1, -1], 1).tolist() == [-1, -1]


def test_class_ranks_count_only_the_slots_that_fit():
    rank, seg_class = sr.class_ranks([9, 3, 9, 0], [True, True, True, True])
    assert rank[9] == 0 and rank[3] == 1 and rank[0] == 2 and seg_class.tolist() == [9, 3, 0] + [-1] * 7
    rank, seg_class = sr.class_ranks([4, 7, 2], [True, False, False])
    assert rank[4] == 0 and rank[7] == rank[2] == -1 and seg_class.tolist() == [4] + [-1] * 9


def test_budget_drops_whole_classes_from_the_segment_table():
    frames = sr.synth_frames(8, 1)
    inp = sr.stage(frames, 90000, 4)
    full = _tables(inp)
    kept = full["kept"]
    assert (kept[:3] > 0).all()
    t = _tables(inp, P_out=int(kept[0]))
    assert t["status"] & sr.OUT_POINTS and t["valid"].tolist() == [1, 0, 0, 0]
    assert t["seg_class"][0].tolist() == [frames[0][2][0][0]] + [-1] * 9 and t["seg"][0] == 0


def test_counts_and_bad_detections_set_their_bits():
    frames = sr.synth_frames(11, 4)
    P, D = 50000, 3
    clouds, cc, calibs, boxes, cls, prob, dc = sr.stage(frames, P, D, cloud_counts=[-1, P, P + 1, 0],
                                                        det_counts=[3, -1, 4, 0])
    cls[2, 1] = 10
    boxes[2, 2, 1] = np.nan
    t = _tables((clouds, cc, calibs, boxes, cls, prob, dc))
    assert t["status"] == sr.SCAN_POINTS | sr.DETS | sr.BAD_DET
    # frame 0 and 3 have no points, frame 1 no detections, frame 2 only its first detection is good
    assert [int(d) for d in t["det_index"] if d >= 0] in ([], [6])
    assert (t["det_points"][[7, 8]] == -1).all() and t["det_points"][6] >= 0
    assert np.dtype(_lib.TrainFrustum) == t["records"].dtype
