"""ORACLE (test infrastructure) - fixtures of the validation pass (csrc/validate.cu, frustum_convnet_b200/validate.py).

Runs the UNMODIFIED reference ``validate()`` of train/train_net_det.py on a list of batch dicts (the data_loader) with
the reference's own PointNetDet (oracle/ref_import.py shims) and seeded weights.  Around it:
  * ``Tensor.cuda`` is an identity (everything stays on the CPU);
  * the zeros stub of the Boost IoU in the model's module is replaced by oracle/box_iou.rbbox_iou_3d_pair, so the IoU
    keys mean something;
  * ``TrainingStates`` is wrapped to capture every batch's reduced values (the 14 ``.item()`` floats), the batch
    sizes, the final ``get_states(avg=True)`` and each meter's (sum, count);
  * forward hooks on ``cls_out`` / ``reg_out`` store each batch's head logits.
Labels are made here from the reference's own eval decode of the same batch: synthetic cls_label rows (with -1 rows),
random non-zero size classes and headings over all bins, and for every other frustum a GT box placed near the decode
of one of its rows (marked foreground with its neighbours), so the IoU metrics are neither all 0 nor all 1.

    python -m oracle.make_golden_validate          # authoring container only (needs /root/reference)

Inputs are regenerated from seeds (oracle.validate.epoch_inputs, checksum stored); labels, logits and results are
stored in tests/golden/validate_<name>.npz."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from frustum_convnet_b200 import config, synth  # noqa: E402
from oracle import box_iou as obox  # noqa: E402
from oracle import ref_import  # noqa: E402
from oracle import validate as ov  # noqa: E402


def make_labels(d, outs, mean_size, rng):
    """Labels for one batch from the reference's eval outputs `outs` (cls_probs, center, heading, size, ...)."""
    B, T2 = outs[0].shape[0], outs[0].shape[1]
    NS = len(mean_size)
    cls = rng.integers(-1, 2, size=(B, T2)).astype(np.int64)
    cls[:, T2 // 2] = 1
    sc = rng.integers(0, NS, B).astype(np.int64)
    sc[0] = max(1, sc[0])                                         # at least one non-zero size class per batch
    head = rng.uniform(-np.pi, np.pi, B)
    ctr = rng.normal(0.0, 0.2, (B, 3))
    size = mean_size[sc] * rng.uniform(0.9, 1.1, (B, 3))
    center_p, head_p, size_p = (o.numpy().astype(np.float64) for o in outs[1:4])
    for b in range(0, B, 2):
        ok = np.nonzero((size_p[b] > 0.3).all(-1))[0]
        if len(ok) == 0:
            continue
        t = int(ok[len(ok) // 2])
        cls[b, max(0, t - 1): t + 2] = 1
        ctr[b] = center_p[b, t] + rng.normal(0, 0.05, 3)
        head[b] = head_p[b, t] + rng.normal(0, 0.03)
        size[b] = size_p[b, t] * (1 + rng.normal(0, 0.03, 3))
    return {"cls_label": cls, "size_class": sc.reshape(B, 1), "box3d_center": ctr.astype(np.float32),
            "box3d_heading": head.reshape(B, 1).astype(np.float32), "box3d_size": size.astype(np.float32)}


def run_case(name):
    import importlib
    workload, wseed, _ = ov.VAL_CASES[name]
    w = config.WORKLOADS[workload]
    model, cfg = ref_import.load_reference_model(w["yaml"], w["num_vec"])
    sys.modules[type(model).__module__].rbbox_iou_3d_pair = obox.rbbox_iou_3d_pair
    sys.modules.pop("train.train_net_det", None)
    drv = importlib.import_module("train.train_net_det")
    assert drv.cfg is cfg
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=wseed)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    model.eval()
    mean_size = np.asarray(model.mean_size_array, np.float64)
    inputs = ov.epoch_inputs(name)
    rng = np.random.default_rng(wseed + 1000)
    loader, labels = [], []
    for d in inputs:
        with torch.no_grad():
            outs = model({k: torch.from_numpy(v) for k, v in d.items()})
        lab = make_labels(d, outs, mean_size, rng)
        labels.append(lab)
        loader.append({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in {**d, **lab}.items()})
    cap = {"vals": [], "bs": []}
    logits = []
    hooks = [model.cls_out.register_forward_hook(lambda m, i, o: logits.append(["cls", o.numpy().copy()])),
             model.reg_out.register_forward_hook(lambda m, i, o: logits.append(["reg", o.numpy().copy()]))]

    class Capture(drv.TrainingStates):
        def update_states(self, states, batch_size=1):
            cap["vals"].append([states[k] for k in states])
            cap["keys"] = list(states)
            cap["bs"].append(batch_size)
            return super().update_states(states, batch_size)

        def get_states(self, avg=True):
            s = super().get_states(avg)
            cap["states"] = [s[k] for k in s]
            cap["meters"] = [(m.sum, m.count) for m in self.average_meters.values()]
            return s
    drv.TrainingStates = Capture
    torch.Tensor.cuda = lambda self, *a, **k: self
    drv.validate(loader, model, 0, None)
    for h in hooks:
        h.remove()
    cls = [o for k, o in logits if k == "cls"]
    reg = [o for k, o in logits if k == "reg"]
    assert len(cls) == len(inputs) and cap["keys"][-1] == "IoU_" + str(cfg.IOU_THRESH)
    rec = {"input_checksum": np.array(ov.checksum(inputs)), "keys": np.array(cap["keys"]),
           "batch_sizes": np.array(cap["bs"], dtype=np.int64), "values": np.array(cap["vals"], dtype=np.float64),
           "states": np.array(cap["states"], dtype=np.float64),
           "meter_sum": np.array([m[0] for m in cap["meters"]], dtype=np.float64),
           "meter_count": np.array([m[1] for m in cap["meters"]], dtype=np.float64),
           "iou_thresh": np.float64(cfg.IOU_THRESH), "num_bins": np.int64(cfg.DATA.NUM_HEADING_BIN),
           "mean_size": np.asarray(model.mean_size_array, np.float32),
           "loss_weights": np.array([cfg.LOSS.BOX_LOSS_WEIGHT, cfg.LOSS.HEAD_REG_WEIGHT, cfg.LOSS.SIZE_REG_WEIGHT,
                                     cfg.LOSS.CORNER_LOSS_WEIGHT], dtype=np.float64)}
    for i, (c, r, lab) in enumerate(zip(cls, reg, labels)):
        rec["cls%d" % i], rec["reg%d" % i] = c, r
        for k, v in lab.items():
            rec["%s%d" % (k, i)] = v
    path = os.path.join(ROOT, "tests", "golden", "validate_%s.npz" % name)
    np.savez_compressed(path, **rec)
    print(name, "->", path, "%.1f KB" % (os.path.getsize(path) / 1024), "states", np.round(rec["states"], 4))


if __name__ == "__main__":
    assert ref_import.reference_available(), "needs /root/reference (authoring container only)"
    for n in (sys.argv[1:] or ov.VAL_CASES):
        run_case(n)
