"""CPU: the validation pass's C ABI (section 12) - argument validation before any CUDA call - and its
numpy oracle, checked against the drop-in model's own eval-with-labels loss code (train_path.losses_from_logits)
and against the reference's AverageMeter arithmetic."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import ROOT


def make_batch(rng, B, T2, NH, mean_size, out_size, near=True, neg_rows=True):
    """Head logits (B,2,T2), (B,out,T2), center_ref2 (B,3,T2) and labels with non-zero size classes, headings over
    several bins, label -1 rows and (near=True) foreground boxes whose decode lies close to the GT box."""
    NS = len(mean_size)
    ms = np.asarray(mean_size, np.float32)
    ref2 = np.zeros((B, 3, T2), np.float32)
    ref2[:, 2] = (np.arange(T2) * 0.5 + 0.25)[None]
    lab = rng.integers(0 if not neg_rows else -1, 2, (B, T2)).astype(np.int64)
    lab[:, T2 // 2] = 1
    sc = rng.integers(0, NS, B).astype(np.int64)
    head = rng.uniform(-np.pi, np.pi, B).astype(np.float32)
    ctr = np.stack([rng.normal(0, 1, B), rng.normal(1, 0.2, B), rng.uniform(0, T2 * 0.5, B)], 1).astype(np.float32)
    size = (ms[sc] * rng.uniform(0.9, 1.1, (B, 3))).astype(np.float32)
    cls = rng.normal(0, 1.5, (B, 2, T2)).astype(np.float32)
    reg = rng.normal(0, 1, (B, out_size, T2)).astype(np.float32)
    if near:
        apc = 2 * np.pi / NH
        for b in range(B):
            hc = int(np.floor(((head[b] % (2 * np.pi)) + apc / 2) % (2 * np.pi) / apc)) % NH
            shifted = ((head[b] % (2 * np.pi)) + apc / 2) % (2 * np.pi)
            res = (shifted - (hc * apc + apc / 2)) / (apc / 2)
            for t in range(T2):
                noise = rng.uniform(0.0, 0.6)
                reg[b, 0:3, t] = ctr[b] - ref2[b, :, t] + rng.normal(0, noise, 3)
                reg[b, 3 + hc, t] += 4.0
                reg[b, 3 + NH + hc, t] = res + rng.normal(0, noise)
                reg[b, 3 + 2 * NH + sc[b], t] += 4.0
                o = 3 + 2 * NH + NS + 3 * sc[b]
                reg[b, o:o + 3, t] = (size[b] - ms[sc[b]]) / ms[sc[b]] + rng.normal(0, 0.3 * noise, 3)
    return dict(cls=cls, reg=reg, center_ref2=ref2, cls_label=lab, size_class=sc.reshape(B, 1),
                box3d_center=ctr, box3d_heading=head.reshape(B, 1), box3d_size=size)


def _kitti():
    from frustum_convnet_b200 import config
    cfg, _ = config.load_workload("car")
    return cfg, config.DATASET_INFO["KITTI"].MEAN_SIZE_ARRAY


def test_argument_validation_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    assert lib.fcn_val_batch(None, None) == -1
    a = _lib.ValBatchArgs()
    assert lib.fcn_val_batch(C.byref(a), None) == -1 and b"bad sizes" in lib.fcn_last_error()
    a.B, a.T2, a.NH, a.NS, a.logit_pitch, a.ld_logit, a.capacity = 2, 10, 12, 8, 9, 128, 4
    assert lib.fcn_val_batch(C.byref(a), None) == -1 and b"logit_pitch" in lib.fcn_last_error()
    a.logit_pitch, a.ld_logit = 11, 40
    assert lib.fcn_val_batch(C.byref(a), None) == -1 and b"ld_logit" in lib.fcn_last_error()
    a.ld_logit = 128
    assert lib.fcn_val_batch(C.byref(a), None) == -1 and b"NULL" in lib.fcn_last_error()
    a.B, a.T2 = 4096, 4096
    assert lib.fcn_val_batch(C.byref(a), None) == -1 and b"2^24" in lib.fcn_last_error()
    assert lib.fcn_val_finalize(None, 4, None, None, None) == -1 and b"NULL" in lib.fcn_last_error()
    assert lib.fcn_val_finalize(None, -1, None, None, None) == -1 and b"capacity" in lib.fcn_last_error()
    assert lib.fcn_val_partials_floats(32, 140) == 35 * 16
    assert lib.fcn_val_partials_floats(0, 140) == -1


class _Model:
    training = False
    gpu_iou_metrics = False
    num_bins = 12

    def __init__(self, mean_size):
        self.mean_size_array = np.asarray(mean_size)
        self.num_size_cluster = len(mean_size)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matches_the_dropin_loss_code(seed):
    """oracle.validate.batch_values == train_path.losses_from_logits (the drop-in's eval-with-labels branch, whose
    IoU is the device kernel and so is compared against the oracle IoU separately on the GPU)."""
    from frustum_convnet_b200.train_path import losses_from_logits
    from oracle import validate as ov
    cfg, ms = _kitti()
    rng = np.random.default_rng(seed)
    B, T2 = 5, 23
    out_size = 3 + 2 * 12 + 4 * len(ms)
    d = make_batch(rng, B, T2, 12, ms, out_size)
    vals = ov.batch_values(d["cls"], d["reg"], d["center_ref2"], d["cls_label"], d["size_class"], d["box3d_center"],
                           d["box3d_heading"], d["box3d_size"], ms, 12, with_iou=True)
    data = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in d.items()}
    data["point_cloud"] = torch.zeros((B, 3, 8))
    cs = data["cls"].permute(0, 2, 1).reshape(-1, 2)
    rg = data["reg"].permute(0, 2, 1).reshape(B * T2, -1)
    losses, metrics = losses_from_logits(_Model(ms), cs, rg, data["center_ref2"], data)
    ref = [float(losses[k]) for k in ov.LOSS_KEYS] + [float(metrics[k]) for k in ("cls_acc", "head_acc", "size_acc")]
    np.testing.assert_allclose(vals[:11], ref, rtol=1e-6, atol=1e-7)
    assert np.isfinite(vals[11:]).all() and vals[12] > 0


def test_average_meter_replay_is_the_reference_arithmetic():
    from oracle import validate as ov

    class AverageMeter:        # utils/utils.py:51-67
        def __init__(self):
            self.val = self.avg = self.sum = 0
            self.count = 1e-14

        def update(self, val, n=1):
            self.val = val
            self.sum += val * n
            self.count += n
            self.avg = self.sum / self.count
    rng = np.random.default_rng(5)
    rows = rng.normal(0, 3, (7, 14)).astype(np.float32)
    bs = [32, 32, 32, 32, 32, 32, 11]
    keys = ["k%d" % i for i in range(14)]
    states, meters = ov.average_meters(rows, bs, keys)
    for i, k in enumerate(keys):
        m = AverageMeter()
        for r, n in zip(rows, bs):
            m.update(float(r[i]), n)
        assert states[k] == m.avg and meters[k] == (m.sum, m.count)


# ----------------------------------------------------------------------------------- reference fixtures
# tests/golden/validate_{kitti,sunrgbd,refine}.npz: the reference's own validate() (oracle/make_golden_validate.py)
FIXTURES = ("kitti", "sunrgbd", "refine")


def load_val_fixture(name):
    """-> (fixture dict, list of per-batch numpy dicts: regenerated inputs + stored labels + stored logits)."""
    from oracle import validate as ov
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "validate_%s.npz" % name)))
    inputs = ov.epoch_inputs(name)
    chk = ov.checksum(inputs)
    assert abs(chk - float(g["input_checksum"])) <= 1e-6 * max(1.0, abs(chk)), "synthetic generator drifted"
    batches = []
    for i, d in enumerate(inputs):
        d = dict(d)
        for k in ("cls_label", "size_class", "box3d_center", "box3d_heading", "box3d_size", "cls", "reg"):
            d[k] = g["%s%d" % (k, i)]
        batches.append(d)
    return g, batches


def oracle_of(g, d, details=False, cls=None, reg=None):
    from oracle import validate as ov
    return ov.batch_values(d["cls"] if cls is None else cls, d["reg"] if reg is None else reg, d["center_ref2"],
                           d["cls_label"], d["size_class"], d["box3d_center"], d["box3d_heading"], d["box3d_size"],
                           g["mean_size"], int(g["num_bins"]), weights=tuple(g["loss_weights"]),
                           iou_thresh=float(g["iou_thresh"]), details=details)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_the_reference_batches(name):
    g, batches = load_val_fixture(name)
    for i, d in enumerate(batches):
        np.testing.assert_allclose(oracle_of(g, d), g["values"][i], rtol=1e-6, atol=1e-7, err_msg="batch %d" % i)


@pytest.mark.parametrize("name", FIXTURES)
def test_float64_replay_reproduces_the_reference_meters_bit_exactly(name):
    from oracle import validate as ov
    g, _ = load_val_fixture(name)
    keys = [str(k) for k in g["keys"]]
    states, meters = ov.average_meters(g["values"], g["batch_sizes"], keys)
    for i, k in enumerate(keys):
        assert states[k] == g["states"][i], k
        assert meters[k] == (g["meter_sum"][i], g["meter_count"][i]), k


def test_fixtures_cover_the_cases():
    seen_pyramids, partial, iou_mid, all_bins = set(), 0, False, set()
    for name in FIXTURES:
        g, batches = load_val_fixture(name)
        bs = g["batch_sizes"]
        partial += int(bs[-1] < bs[0])
        assert list(g["keys"][-1:]) == ["IoU_" + str(float(g["iou_thresh"]))] and len(g["keys"]) == 14
        assert g["states"][11] > 0 and g["states"][12] > 0, name          # IoU_2D, IoU_3D
        iou_mid |= bool(0 < g["states"][13] < 1)
        labels = np.concatenate([d["cls_label"].reshape(-1) for d in batches])
        assert (labels == -1).any() and (labels == 0).any() and (labels == 1).any()
        sc = np.concatenate([d["size_class"].reshape(-1) for d in batches])
        assert (sc > 0).any()
        head = np.concatenate([d["box3d_heading"].reshape(-1) for d in batches])
        bins = np.floor(((head % (2 * np.pi)) + np.pi / 12) % (2 * np.pi) / (np.pi / 6)).astype(int)
        assert len(set(bins.tolist())) >= 2, name
        all_bins |= set(bins.tolist())
        if name == "refine":
            seen_pyramids = {tuple(d["center_ref%d" % (s + 1)].shape[2] for s in range(4)) for d in batches}
    assert partial == len(FIXTURES) and len(seen_pyramids) >= 2 and iou_mid and len(all_bins) >= 5
    sizes = sum(os.path.getsize(os.path.join(ROOT, "tests", "golden", "validate_%s.npz" % n)) for n in FIXTURES)
    assert sizes < 1 << 20
