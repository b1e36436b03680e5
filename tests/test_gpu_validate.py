"""GPU: the validation pass (csrc/validate.cu, frustum_convnet_b200/validate.py) against the numpy oracle, the drop-in
model's own eval-with-labels path and the reference's AverageMeter arithmetic; determinism, capture and errors."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_validate_cpu import make_batch

pytestmark = pytest.mark.gpu

KEYS = 14


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _kitti():
    from frustum_convnet_b200 import config
    cfg, _ = config.load_workload("car")
    return cfg, np.asarray(config.DATASET_INFO["KITTI"].MEAN_SIZE_ARRAY, np.float32)


class _Table:
    """Caller-owned epoch table + one fcn_val_batch per call, on logits placed in a plan-shaped pitched buffer."""

    def __init__(self, capacity=64):
        from frustum_convnet_b200 import _lib
        self.lib, self.cap = _lib, capacity
        self.table = torch.zeros((capacity, _lib.VAL_ROW), dtype=torch.float32, device="cuda")
        self.state = torch.zeros(4, dtype=torch.int32, device="cuda")
        self.res = torch.zeros(C.sizeof(_lib.ValResult), dtype=torch.uint8, device="cuda")
        self.keep = []

    def args(self, d, ms, pitch_extra=3, ld=128, with_iou=True):
        lib = self.lib
        B, _, T2 = d["cls"].shape
        lg = torch.full((B, T2 + pitch_extra, ld), 1e30, dtype=torch.float32, device="cuda")
        lg[:, :T2, 0:2] = _cuda(d["cls"]).permute(0, 2, 1)
        lg[:, :T2, 2:2 + d["reg"].shape[1]] = _cuda(d["reg"]).permute(0, 2, 1)
        ts = dict(lg=lg, ref2=_cuda(d["center_ref2"]), lab=_cuda(d["cls_label"]), sc=_cuda(d["size_class"].reshape(-1)),
                  c=_cuda(d["box3d_center"]), h=_cuda(d["box3d_heading"].reshape(-1)), s=_cuda(d["box3d_size"]),
                  ms=_cuda(ms), part=torch.zeros(int(lib.load().fcn_val_partials_floats(B, T2)), device="cuda"))
        a = lib.ValBatchArgs()
        a.B, a.T2, a.NH, a.NS, a.with_iou, a.capacity = B, T2, 12, len(ms), int(with_iou), self.cap
        a.logit_pitch, a.ld_logit = T2 + pitch_extra, ld
        a.logits, a.center_ref2, a.cls_label, a.size_class = (ts[k].data_ptr() for k in ("lg", "ref2", "lab", "sc"))
        a.box3d_center, a.box3d_heading, a.box3d_size, a.mean_size = (ts[k].data_ptr() for k in ("c", "h", "s", "ms"))
        a.w_box, a.w_head_reg, a.w_size_reg, a.w_corner, a.iou_thresh = 1.0, 20.0, 20.0, 10.0, 0.7
        a.partials, a.state, a.table = ts["part"].data_ptr(), self.state.data_ptr(), self.table.data_ptr()
        self.keep.append(ts)
        return a

    def run(self, a):
        self.lib.call("fcn_val_batch", C.byref(a), torch.cuda.current_stream().cuda_stream)

    def finalize(self):
        self.lib.call("fcn_val_finalize", self.table.data_ptr(), self.cap, self.state.data_ptr(), self.res.data_ptr(),
                      torch.cuda.current_stream().cuda_stream)
        return self.lib.ValResult.from_buffer_copy(self.res.cpu().numpy().tobytes())

    def rows(self):
        n = min(int(self.state[0]), self.cap)
        return self.table[:n].cpu().numpy()


def _check_against_oracle(got, d, ms, info_vals, loss_tol=1e-5):
    vals, info = info_vals
    for i in range(8):
        assert abs(got[i] - vals[i]) <= loss_tol * max(1.0, abs(vals[i])), (i, got[i], vals[i])
    for i in (8, 9, 10):
        assert got[i] == vals[i], (i, got[i], vals[i])
    for i in (11, 12):
        assert abs(got[i] - vals[i]) <= 1e-4, (i, got[i], vals[i])
    near = int((np.abs(info["iou3d"] - 0.7) < 1e-4).sum())
    assert abs(got[13] - vals[13]) <= near / info["nfg"] + 1e-7, (got[13], vals[13], near)


def _batches(seed, n, B=6, T2=37, last_B=3):
    _, ms = _kitti()
    rng = np.random.default_rng(seed)
    out_size = 3 + 24 + 4 * len(ms)
    return [make_batch(rng, B if i < n - 1 else last_B, T2, 12, ms, out_size) for i in range(n)]


def test_kernel_matches_the_oracle_and_finalize_replays_average_meter():
    from oracle import validate as ov
    _, ms = _kitti()
    tb = _Table()
    batches = _batches(11, 5)
    expect = []
    for d in batches:
        tb.run(tb.args(d, ms))
        expect.append(ov.batch_values(d["cls"], d["reg"], d["center_ref2"], d["cls_label"], d["size_class"],
                                      d["box3d_center"], d["box3d_heading"], d["box3d_size"], ms, 12, details=True))
    rows = tb.rows()
    assert rows.shape == (5, 18)
    for r, d, e in zip(rows, batches, expect):
        _check_against_oracle(r, d, ms, e)
        assert r[14] == d["cls"].shape[0] and r[15] == e[1]["nfg"] and r[16] == e[1]["nkeep"]
    assert any(0 < e[0][13] < 1 for e in expect) and all(e[0][12] > 0 for e in expect)
    res = tb.finalize()
    keys = ["k%d" % i for i in range(KEYS)]
    states, meters = ov.average_meters(rows[:, :KEYS], rows[:, 14].astype(int), keys)
    assert res.rows == 5 and res.status == 0
    for i, k in enumerate(keys):
        assert res.avg[i] == states[k] and res.sum[i] == meters[k][0] and res.count == meters[k][1]


def test_kernel_without_iou_gives_nan_and_is_deterministic_across_runs_streams_and_graphs():
    _, ms = _kitti()
    batches = _batches(12, 3, B=32, T2=140, last_B=17)

    def epoch(mode, with_iou=True):
        tb = _Table()
        args = [tb.args(d, ms, with_iou=with_iou) for d in batches]
        if mode == "eager":
            for a in args:
                tb.run(a)
        elif mode == "stream":
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for a in args:
                    tb.run(a)
            torch.cuda.current_stream().wait_stream(s)
        else:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for a in args:
                    tb.run(a)
            g.replay()
        torch.cuda.synchronize()
        return tb.rows()
    ref = epoch("eager")
    for mode in ("eager", "stream", "graph"):
        assert np.array_equal(epoch(mode).view(np.int32), ref.view(np.int32)), mode
    no_iou = epoch("eager", with_iou=False)
    assert np.isnan(no_iou[:, 11:14]).all() and np.array_equal(no_iou[:, :11], ref[:, :11])


def test_kernel_flags_batches_without_foreground_and_overflow():
    _, ms = _kitti()
    batches = _batches(13, 4)
    batches[2]["cls_label"][batches[2]["cls_label"] == 1] = 0
    tb = _Table(capacity=3)
    for d in batches:
        tb.run(tb.args(d, ms))
    res = tb.finalize()
    assert res.added == 4 and res.rows == 3 and res.first_no_fg == 2
    from frustum_convnet_b200 import _lib
    assert res.status == _lib.VAL_NO_FG | _lib.VAL_OVERFLOW


# ----------------------------------------------------------------------------------- end to end (Validator)
def _model(workload, precision, seed=7):
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload(workload)
    if w["arch"].num_scales == 5:
        from frustum_convnet_b200.det_base_sunrgbd import PointNetDet
    else:
        from frustum_convnet_b200.det_base import PointNetDet
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=seed)
    m = PointNetDet(3, num_vec=w["num_vec"])
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    for mod in m.modules():        # the drop-in's feature and FCN submodules run their own engines
        if hasattr(mod, "resolved_precision"):
            mod.precision = precision
    return m.cuda().eval(), cfg


def _data(workload, B, seed, md=None):
    from frustum_convnet_b200 import synth
    d = synth.make_frustums(workload, B, seed=seed, max_depth=md, with_labels=True)
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


EPOCHS = {
    "car": [(4, 21, 17.5), (4, 22, 17.5), (3, 23, 17.5)],
    "sunrgbd": [(3, 31, None), (2, 32, None)],
    "refine_car": [(4, 41, None), (2, 42, None)],
    "people": [(3, 51, 7.0), (2, 52, 12.0)],          # two T pyramids in one epoch
}


@pytest.mark.parametrize("workload", sorted(EPOCHS))
def test_validator_agrees_with_the_dropin_eval_with_labels_path(workload):
    from frustum_convnet_b200.validate import Validator
    from oracle import validate as ov
    m, cfg = _model(workload, 0)
    batches = [_data(workload, B, s, md) for B, s, md in EPOCHS[workload]]
    val = Validator(m)
    for d in batches:
        val.add(d)
    states = val.finalize()
    assert list(states) == list(ov.LOSS_KEYS) + ["cls_acc", "head_acc", "size_acc", "IoU_2D", "IoU_3D",
                                                 "IoU_" + str(cfg.IOU_THRESH)]
    got = val.per_batch()
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        rows = []
        with torch.no_grad():
            for d in batches:
                losses, metrics = m(d)
                rows.append([float(v) for v in list(losses.values()) + list(metrics.values())])
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    rows = np.array(rows, np.float32)
    np.testing.assert_allclose(got, rows, rtol=2e-4, atol=2e-4)
    expect, _ = ov.average_meters(got, [d["point_cloud"].shape[0] for d in batches], list(states))
    assert list(states.values()) == list(expect.values())


def test_validator_tf32_against_the_oracle_on_the_engine_logits():
    from frustum_convnet_b200.validate import Validator
    from oracle import validate as ov
    m, cfg = _model("car", 1)
    ms = np.asarray(m.mean_size_array, np.float32)
    val = Validator(m)
    for B, s, md in EPOCHS["car"]:
        d = _data("car", B, s, md)
        val.add(d)
        T = [d["center_ref%d" % (i + 1)].shape[2] for i in range(4)]
        plan = m.engine().plan(B, d["point_cloud"].shape[2], T)
        lg, pitch, ld, ref2 = plan.head_logits()
        T2 = T[1]
        cls = lg[:, :T2, 0:2].permute(0, 2, 1).cpu().numpy()
        reg = lg[:, :T2, 2:2 + m.engine().out_size].permute(0, 2, 1).cpu().numpy()
        h = {k: v.cpu().numpy() for k, v in d.items()}
        e = ov.batch_values(cls, reg, h["center_ref2"], h["cls_label"], h["size_class"], h["box3d_center"],
                            h["box3d_heading"], h["box3d_size"], ms, 12, details=True)
        _check_against_oracle(val.per_batch()[-1], None, ms, e)


def test_validator_capture_determinism_and_errors():
    from frustum_convnet_b200.validate import Validator
    m, _ = _model("car", 1)
    batches = [_data("car", B, s, md) for B, s, md in EPOCHS["car"]]
    val = Validator(m)
    for d in batches:
        val.add(d)
    s1, t1 = val.finalize(), val.per_batch()
    val.reset()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for d in batches:
            val.add(d)
    s2, t2 = val.finalize(), val.per_batch()
    assert s1 == s2 and np.array_equal(t1.view(np.int32), t2.view(np.int32))
    # capture (on the stream whose plans the epoch above warmed up): every replay appends the batches again
    val.reset()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        for d in batches:
            val.add(d)
    g.replay()
    g.replay()
    t3 = val.per_batch()
    assert t3.shape[0] == 6
    assert np.array_equal(t3[:3].view(np.int32), t1.view(np.int32)) and np.array_equal(t3[3:].view(np.int32),
                                                                                          t1.view(np.int32))
    # overflow names the capacity needed; a batch without foreground names its index
    small = Validator(m, capacity=2)
    for d in batches:
        small.add(d)
    with pytest.raises(RuntimeError, match="capacity=3"):
        small.finalize()
    bad = dict(batches[1])
    bad["cls_label"] = torch.where(bad["cls_label"] == 1, torch.zeros_like(bad["cls_label"]), bad["cls_label"])
    v2 = Validator(m)
    for d in (batches[0], bad, batches[2]):
        v2.add(d)
    with pytest.raises(RuntimeError, match="batch 1 "):
        v2.finalize()
    m.train()
    with pytest.raises(RuntimeError, match="eval"):
        v2.add(batches[0])
    m.eval()
    d4 = dict(batches[0])
    d4["point_cloud"] = torch.cat([d4["point_cloud"], d4["point_cloud"][:, :1]], 1)
    with pytest.raises(ValueError):
        v2.add(d4)


def test_validator_follows_weight_updates():
    """One TrainStep.step between two epochs (train mode, fused Adam, back to eval) changes the states, and the second
    epoch equals a freshly built Validator's."""
    from frustum_convnet_b200 import synth
    from frustum_convnet_b200.train_engine import TrainStep
    from frustum_convnet_b200.validate import Validator
    m, _ = _model("car", 1)
    batches = [_data("car", B, s, md) for B, s, md in EPOCHS["car"]]
    val = Validator(m)
    for d in batches:
        val.add(d)
    s1 = val.finalize()
    train = {k: torch.from_numpy(v).cuda() for k, v in synth.make_frustums("car", 8, seed=77, with_labels=True).items()}
    m.train()
    TrainStep(m, lr=1e-3).step(train)
    m.eval()
    val.reset()
    for d in batches:
        val.add(d)
    s2 = val.finalize()
    fresh = Validator(m)
    for d in batches:
        fresh.add(d)
    assert s2 != s1 and fresh.finalize() == s2


def test_device_built_val_batches_give_the_reference_provider_states():
    """Val batches from TrainBatchBuilder (no flip, no shift) against the same batches from the numpy restatement of
    the reference providers (oracle/train_inputs.py)."""
    from test_gpu_train_inputs import CAR, random_lists
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    from frustum_convnet_b200.validate import Validator
    from oracle import train_inputs as oti
    rng = np.random.default_rng(21)
    L = random_lists("det", 300, rng)
    tb = TrainBatchBuilder("det", CAR, 1024, max_depth=70.0, random_flip=False, random_shift=False)
    tb.set_dataset(L["input_list"], L["type_list"], ("Car", "Pedestrian", "Cyclist"),
                   **{k: v for k, v in L.items() if k not in ("input_list", "type_list")})
    m, _ = _model("car", 0)
    v_dev, v_ref = Validator(m), Validator(m)
    order = rng.permutation(300)
    for k, B in enumerate((16, 16, 7)):
        index = order[k * 16: k * 16 + B]
        np.random.seed(300 + k)
        draws = tb.draw(index)
        v_dev.add(tb.build(index, draws))
        ref = oti.build("det", L, index, draws, CAR, 70.0, random_flip=False, random_shift=False, labels=True)
        ref.pop("_margins", None)
        v_ref.add({key: torch.from_numpy(np.ascontiguousarray(v)).cuda() for key, v in ref.items()})
    a, b = v_dev.finalize(), v_ref.finalize()
    assert list(a) == list(b)
    np.testing.assert_allclose(list(a.values()), list(b.values()), rtol=1e-4, atol=1e-6)


# ----------------------------------------------------------------------------------- reference fixtures
from test_validate_cpu import FIXTURES, load_val_fixture, oracle_of  # noqa: E402


def _allow(info):
    """Largest legitimate deviation of each discrete metric: rows whose reference argmax margin is below 1e-3 or whose
    3-D IoU lies within 1e-4 of the threshold may flip."""
    a = np.zeros(3)
    a[0] = (info["cls_margin"] < 1e-3).sum() / info["nkeep"]
    a[1] = (info["head_margin"] < 1e-3).sum() / info["nfg"]
    a[2] = (info["size_margin"] < 1e-3).sum() / info["nfg"]
    return a


@pytest.mark.parametrize("name", FIXTURES)
def test_kernel_on_the_reference_logits_matches_the_reference_values(name):
    g, batches = load_val_fixture(name)
    ms = np.asarray(g["mean_size"], np.float32)
    thr = float(g["iou_thresh"])
    tb = _Table()
    for d in batches:
        a = tb.args(d, ms)
        a.NH = int(g["num_bins"])
        a.iou_thresh = thr
        a.w_box, a.w_head_reg, a.w_size_reg, a.w_corner = (float(x) for x in g["loss_weights"])
        tb.run(a)
    rows = tb.rows()
    for i, d in enumerate(batches):
        ref = g["values"][i]
        _, info = oracle_of(g, d, details=True)
        got = rows[i]
        for j in range(8):
            assert abs(got[j] - ref[j]) <= 1e-5 * max(1.0, abs(ref[j])), (name, i, j, got[j], ref[j])
        for j in (8, 9, 10):
            assert got[j] == np.float32(ref[j]), (name, i, j, got[j], ref[j])
        for j in (11, 12):
            assert abs(got[j] - ref[j]) <= 1e-4, (name, i, j, got[j], ref[j])
        near = int((np.abs(info["iou3d"] - thr) < 1e-4).sum())
        assert abs(got[13] - np.float32(ref[13])) <= near / info["nfg"], (name, i, got[13], ref[13])


def _fixture_model(name, precision):
    from oracle import validate as ov
    workload, wseed, _ = ov.VAL_CASES[name]
    return _model(workload, precision, seed=wseed)


@pytest.mark.parametrize("name", FIXTURES)
def test_validator_fp32_matches_the_reference_validate(name):
    from frustum_convnet_b200.validate import Validator
    g, batches = load_val_fixture(name)
    m, cfg = _fixture_model(name, 0)
    val = Validator(m)
    for d in batches:
        val.add({k: _cuda(v) for k, v in d.items() if k not in ("cls", "reg")})
    states = val.finalize()
    assert list(states) == [str(k) for k in g["keys"]]
    got = val.per_batch()
    thr = float(g["iou_thresh"])
    for i, d in enumerate(batches):
        ref = g["values"][i]
        _, info = oracle_of(g, d, details=True)
        allow = _allow(info)
        flips = allow[1] > 0 or allow[2] > 0            # a flipped predicted class moves the IoU of its row
        for j in range(8):
            assert abs(got[i, j] - ref[j]) <= 2e-4 * max(1.0, abs(ref[j])), (name, i, j, got[i, j], ref[j])
        for j in (8, 9, 10):
            assert abs(got[i, j] - ref[j]) <= allow[j - 8] + 1e-7, (name, i, j, got[i, j], ref[j])
        if not flips:
            for j in (11, 12):
                assert abs(got[i, j] - ref[j]) <= 2e-4 * max(1.0, abs(ref[j])), (name, i, j, got[i, j], ref[j])
            near = (np.abs(info["iou3d"] - thr) < 1e-4).sum() / info["nfg"]
            assert abs(got[i, 13] - ref[13]) <= near + 1e-7, (name, i, got[i, 13], ref[13])
    for j, (k, v) in enumerate(states.items()):
        if j < 8:
            assert abs(v - g["states"][j]) <= 2e-4 * max(1.0, abs(g["states"][j])), (k, v, g["states"][j])


@pytest.mark.parametrize("name", FIXTURES)
def test_validator_tf32_logits_and_values(name):
    from frustum_convnet_b200.validate import Validator
    g, batches = load_val_fixture(name)
    m, _ = _fixture_model(name, 1)
    val = Validator(m)
    thr = float(g["iou_thresh"])
    for i, d in enumerate(batches):
        dd = {k: _cuda(v) for k, v in d.items() if k not in ("cls", "reg")}
        val.add(dd)
        S = m.ARCH.num_scales
        T = [dd["center_ref%d" % (s + 1)].shape[2] for s in range(S)]
        plan = m.engine().plan(dd["point_cloud"].shape[0], dd["point_cloud"].shape[2], T)
        lg, _, _, _ = plan.head_logits()
        T2, osz = T[1], d["reg"].shape[1]
        cls = lg[:, :T2, 0:2].permute(0, 2, 1).cpu().numpy()
        reg = lg[:, :T2, 2:2 + osz].permute(0, 2, 1).cpu().numpy()
        for mine, ref in ((cls, d["cls"]), (reg, d["reg"])):      # the benchmarked-configuration bar
            assert float(np.abs(mine - ref).max()) <= 2.5e-3 * max(1.0, float(np.abs(ref).max())), name
        e, info = oracle_of(g, d, details=True, cls=cls, reg=reg)
        got = val.per_batch()[i]
        for j in range(8):
            assert abs(got[j] - e[j]) <= 1e-5 * max(1.0, abs(e[j])), (name, i, j, got[j], e[j])
        for j in (8, 9, 10):
            assert got[j] == e[j], (name, i, j, got[j], e[j])
        for j in (11, 12):
            assert abs(got[j] - e[j]) <= 1e-4, (name, i, j, got[j], e[j])
        near = int((np.abs(info["iou3d"] - thr) < 1e-4).sum())
        assert abs(got[13] - e[13]) <= near / info["nfg"] + 1e-7, (name, i, got[13], e[13])
