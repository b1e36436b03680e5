"""ORACLE (test infrastructure) - fixture of the fused detection loss and its gradient (csrc/loss.cu, fcn_det_loss;
float64 restatement tests/loss_ref.py).

Runs the reference's own ``PointNetDet`` train branch (models/det_base.py:414-525) on the CPU with the head outputs
replaced by crafted logits (tests/loss_ref.make_case: branch points of every loss term, exact arg-max ties):
  * the feature and FCN sub-networks are stubs (their output is discarded), forward hooks on ``cls_out`` /
    ``reg_out`` return leaf tensors holding the crafted logits, so autograd gives d(total)/d(logits);
  * ``num_bins``, ``num_size_cluster`` and ``mean_size_array`` are set per case (NH = 12 with NS = 1, 3, 10,
    NH = NS = 32 and NH = 9), the four loss weights to distinct values;
  * the zeros stub of the Boost IoU is replaced by oracle/box_iou.rbbox_iou_3d_pair;
  * ``angle_encode``, ``angle_decode`` and ``size_decode`` of the model's module are wrapped to record the heading
    class / residual labels and the predicted heading and size classes (the discrete decisions).
Everything is recorded in float32, as the reference computes it.

    python -m oracle.make_golden_det_loss          # authoring container only (needs the reference checkout)

writes tests/golden/det_loss_edges.npz."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import box_iou as obox  # noqa: E402
from oracle import ref_import  # noqa: E402
import loss_ref  # noqa: E402

# name -> (NH, NS, B, T2, seed); mirrored in tests/test_det_loss_cpu.py
# nh12_ns3 has one frustum per GT heading kind of loss_ref.HEADING_KINDS (bin boundaries +- 1 ulp, 0, +-pi,
# 2 pi - ulp, 2 pi, below -2 pi, above 2 pi, ...); nh9_ns3 has a bin width where float32(2 pi) / NH is 1 ulp off
CASES = {"nh12_ns3": (12, 3, 16, 12, 11), "nh12_ns1": (12, 1, 3, 20, 12), "nh12_ns10": (12, 10, 3, 20, 13),
         "nh32_ns32": (32, 32, 2, 16, 14), "nh9_ns3": (9, 3, 16, 8, 15)}
WEIGHTS = (2.3, 17.0, 13.0, 5.5)
IOU_THRESH = 0.7


class _Stub(torch.nn.Module):
    def __init__(self, fn):
        super().__init__()
        self.fn = fn

    def forward(self, *a):
        return self.fn(*a)


def run_case(model, cfg, mod, NH, NS, B, T2, seed):
    c = loss_ref.make_case(B, T2, NH, NS, seed)
    W = 3 + 2 * NH + 4 * NS
    model.num_bins, model.num_size_cluster = NH, NS
    model.mean_size_array = c["mean_size"].astype(np.float64)
    cfg.LOSS.BOX_LOSS_WEIGHT, cfg.LOSS.HEAD_REG_WEIGHT, cfg.LOSS.SIZE_REG_WEIGHT, cfg.LOSS.CORNER_LOSS_WEIGHT = WEIGHTS
    cfg.IOU_THRESH = IOU_THRESH
    model.feat_net = _Stub(lambda *a: (None, None, None, None))
    model.conv_net = _Stub(lambda *a: torch.zeros(B, 768, T2))
    lc = torch.from_numpy(c["cls"].reshape(B, T2, 2).transpose(0, 2, 1).copy()).requires_grad_(True)
    lr_ = torch.from_numpy(c["reg"].reshape(B, T2, W).transpose(0, 2, 1).copy()).requires_grad_(True)
    hooks = [model.cls_out.register_forward_hook(lambda m, i, o: lc),
             model.reg_out.register_forward_hook(lambda m, i, o: lr_)]
    rec = {"encode": [], "decode": [], "size": []}
    enc, dec, sdec = mod.angle_encode, mod.angle_decode, mod.size_decode

    def w_enc(*a, **k):
        r = enc(*a, **k)
        rec["encode"].append([t.detach().clone() for t in r])
        return r

    def w_dec(res, cid, *a, **k):
        rec["decode"].append(cid.detach().clone())
        return dec(res, cid, *a, **k)

    def w_sdec(off, ms, cid):
        rec["size"].append(cid.detach().clone())
        return sdec(off, ms, cid)
    mod.angle_encode, mod.angle_decode, mod.size_decode = w_enc, w_dec, w_sdec
    try:
        data = {"point_cloud": torch.zeros(B, 3, 1), "one_hot": torch.zeros(B, 3),
                "cls_label": torch.from_numpy(c["cls_label"]), "size_class": torch.from_numpy(c["size_class"]).view(B, 1),
                "box3d_center": torch.from_numpy(c["box3d_center"]),
                "box3d_heading": torch.from_numpy(c["box3d_heading"]).view(B, 1),
                "box3d_size": torch.from_numpy(c["box3d_size"]),
                "center_ref1": torch.zeros(B, 3, T2), "center_ref2": torch.from_numpy(c["center_ref2"]),
                "center_ref3": torch.zeros(B, 3, T2), "center_ref4": torch.zeros(B, 3, T2)}
        losses, metrics = model(data)
        losses["total_loss"].backward()
    finally:
        mod.angle_encode, mod.angle_decode, mod.size_decode = enc, dec, sdec
        for h in hooks:
            h.remove()
    out = dict(c)
    out["losses"] = np.array([float(v) for v in losses.values()], np.float32)
    out["metrics"] = np.array([float(v) for v in metrics.values()], np.float32)
    out["dcls"] = lc.grad.permute(0, 2, 1).reshape(B * T2, 2).numpy().astype(np.float32)
    out["dreg"] = lr_.grad.permute(0, 2, 1).reshape(B * T2, W).numpy().astype(np.float32)
    out["hc"] = rec["encode"][0][0].numpy().astype(np.int64)
    out["hres_lab"] = rec["encode"][0][1].numpy().astype(np.float32)
    assert len(rec["decode"]) == 2 and len(rec["size"]) == 2
    out["h_arg"] = rec["decode"][1].numpy().astype(np.int64)
    out["s_arg"] = rec["size"][1].numpy().astype(np.int64)
    return out


def main():
    assert ref_import.reference_available(), "needs the reference checkout (authoring container only)"
    model, cfg = ref_import.load_reference_model("det_sample.yaml", 3)
    mod = sys.modules[type(model).__module__]
    mod.rbbox_iou_3d_pair = obox.rbbox_iou_3d_pair
    model.train()
    torch.manual_seed(0)
    rec = {"weights": np.array(WEIGHTS, np.float32), "iou_thresh": np.float32(IOU_THRESH)}
    for name, (NH, NS, B, T2, seed) in CASES.items():
        for k, v in run_case(model, cfg, mod, NH, NS, B, T2, seed).items():
            rec["%s/%s" % (name, k)] = v
    path = os.path.join(ROOT, "tests", "golden", "det_loss_edges.npz")
    np.savez_compressed(path, **rec)
    print(path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
