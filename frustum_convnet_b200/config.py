"""Host-side mirror of the configuration surface the frustum hot path reads.

The reference keeps one global, Detectron-style ``cfg`` object
(/root/reference/configs/config.py:57-192) that the model consults at
construction time (models/det_base.py:112 ``cfg.DATA.HEIGHT_HALF``, :233
``cfg.DATA.DATASET_NAME``, :245 ``cfg.DATA.NUM_HEADING_BIN``, :465-468
``cfg.LOSS.*``, :500 ``cfg.IOU_THRESH``).  This module mirrors only those keys
plus the data-shape keys the synthetic generator needs.

Drop-in rule: when this package is imported from inside the reference tree
(``configs.config`` importable) the *reference's own* cfg object is used, so
``merge_cfg_from_file`` calls made by train/test drivers are honoured.  Outside
the reference tree (the GPU box) the local mirror below is used and
``merge_cfg_from_file`` reads our own ``cfgs/*.yaml``.
"""
from __future__ import annotations

import ast
import copy
import os
from typing import List, NamedTuple

import numpy as np
import yaml


class CfgNode(dict):
    """dict with attribute access (same surface as the reference AttrDict,
    configs/collections.py:24-62, minus immutability bookkeeping)."""

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError as e:  # pragma: no cover - error path
            raise AttributeError(name) from e

    def __setattr__(self, name, value):
        self[name] = value


def _defaults() -> CfgNode:
    c = CfgNode()
    c.TRAIN = CfgNode(BATCH_SIZE=32, OPTIMIZER="adam", BASE_LR=0.001, WEIGHT_DECAY=0.0,
                      MOMENTUM=0.9)
    c.TEST = CfgNode(BATCH_SIZE=32, METHOD="top")
    c.MODEL = CfgNode(FILE="", NUM_CLASSES=2)
    c.DATA = CfgNode(
        DATASET_NAME="KITTI", MAX_DEPTH=70, NUM_SAMPLES=1024, NUM_HEADING_BIN=12,
        STRIDE=(0.25, 0.5, 1.0, 2.0), HEIGHT_HALF=(0.25, 0.5, 1.0, 2.0),
        WITH_EXTRA_FEAT=False, CAR_ONLY=True, PEOPLE_ONLY=False,
    )
    c.LOSS = CfgNode(BOX_LOSS_WEIGHT=1.0, CORNER_LOSS_WEIGHT=10.0, HEAD_REG_WEIGHT=20.0,
                     SIZE_REG_WEIGHT=20.0)
    c.IOU_THRESH = 0.7
    c.NUM_GPUS = 1
    return c


_local_cfg = _defaults()


def _reference_cfg():
    try:
        from configs.config import cfg as ref_cfg  # type: ignore
        if "DATA" in ref_cfg and "HEIGHT_HALF" in ref_cfg.DATA:
            return ref_cfg
    except Exception:
        pass
    return None


def get_cfg():
    """The cfg object the drop-in modules read (reference's if present)."""
    ref = _reference_cfg()
    return ref if ref is not None else _local_cfg


cfg = _local_cfg


def reset_cfg():
    _local_cfg.clear()
    _local_cfg.update(_defaults())


def _decode(v):
    if isinstance(v, dict):
        return CfgNode({k: _decode(x) for k, x in v.items()})
    if isinstance(v, str):
        try:
            return ast.literal_eval(v)
        except (ValueError, SyntaxError):
            return v
    return v


def _merge(a: dict, b: CfgNode, path=""):
    for k, v in a.items():
        v = _decode(copy.deepcopy(v))
        if isinstance(v, CfgNode) and isinstance(b.get(k), CfgNode):
            _merge(v, b[k], path + k + ".")
        else:
            if isinstance(v, list) and isinstance(b.get(k), tuple):
                v = tuple(v)
            b[k] = v  # unknown keys are accepted: our yamls are a subset/superset


def merge_cfg_from_file(path: str):
    """Same role as configs/config.py:231-235 for the local mirror."""
    with open(path, "r") as f:
        y = yaml.safe_load(f)
    _merge(y, _local_cfg)
    return _local_cfg


CFG_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cfgs")


# --------------------------------------------------------------------------
# dataset constants (values are dataset facts, cf. datasets/dataset_info.py:3-39)
# --------------------------------------------------------------------------
_KITTI_CLASSES = ("Car", "Pedestrian", "Cyclist")
_KITTI_MEAN = np.array([
    [3.88311640418, 1.62856739989, 1.52563191462],
    [0.84422524, 0.66068622, 1.76255119],
    [1.76282397, 0.59706367, 1.73698127],
])
_SUN_CLASSES = ("bathtub", "bed", "bookshelf", "chair", "desk", "dresser", "night_stand",
                "sofa", "table", "toilet")
_SUN_MEAN = np.array([
    [0.765840, 1.398258, 0.472728], [2.114256, 1.620300, 0.927272],
    [0.404671, 1.071108, 1.688889], [0.591958, 0.552978, 0.827272],
    [0.695190, 1.346299, 0.736364], [0.528526, 1.002642, 1.172878],
    [0.500618, 0.632163, 0.683424], [0.923508, 1.867419, 0.845495],
    [0.791118, 1.279516, 0.718182], [0.699104, 0.454178, 0.756250],
])


class _Category:
    def __init__(self, classes, mean):
        self.CLASSES = list(classes)
        self.NUM_SIZE_CLUSTER = len(classes)
        self.MEAN_SIZE_ARRAY = np.asarray(mean, dtype=np.float64)


DATASET_INFO = {"KITTI": _Category(_KITTI_CLASSES, _KITTI_MEAN),
                "SUNRGBD": _Category(_SUN_CLASSES, _SUN_MEAN)}


# --------------------------------------------------------------------------
# architecture table (det_base.py:114-124,167-183; det_base_sunrgbd.py:115-128,178-200)
# --------------------------------------------------------------------------
class ArchSpec:
    """Static shape description of one PointNetDet variant."""

    def __init__(self, name, nsample, mlps, block1_out, reg_in, block_widths=(), deconv_out=256):
        self.name = name
        self.nsample = tuple(nsample)       # K per scale
        self.mlps = tuple(tuple(m) for m in mlps)  # (C1,C2,C3) per scale
        self.num_scales = len(nsample)
        self.block1_out = block1_out        # ConvFeatNet block1_conv1 width
        self.reg_in = reg_in                # channels entering the heads
        self.block_widths = tuple(block_widths)   # ConvFeatNet blocks 2..S: conv1 / conv2 / merge width
        self.deconv_out = deconv_out        # width of every transposed conv = its slice of the heads' concat


ARCH_KITTI = ArchSpec("kitti", (32, 64, 64, 128),
                      ((64, 64, 128), (64, 64, 128), (128, 128, 256), (256, 256, 512)),
                      128, 768, (128, 256, 512))
ARCH_SUNRGBD = ArchSpec("sunrgbd", (128, 128, 256, 256, 256),
                        ((64, 64, 128), (64, 64, 128), (128, 128, 256), (256, 256, 512),
                         (256, 256, 512)),
                        64, 1024, (128, 256, 512, 512))


class FcnLayer(NamedTuple):
    """One layer of ConvFeatNet + heads.  Every consumer reads the graph from these fields, never from a name."""
    name: str       # state-dict name under ``conv_net.``; "heads" stands for cls_out + reg_out
    kind: str       # "conv" (k=3, padding 1) | "merge" (1x1 over [block output, pooled feature]) | "deconv" | "heads"
    srcs: tuple     # ((producer, channels), ...) in K order; a producer is a layer name or "feat<i>" (PointNet scale i)
    Cout: int       # None for the heads: their width is set by the dataset's regression size
    k: int
    stride: int
    level: int      # pyramid level (0-based scale) of the output positions; the concat and the heads are at level 1
    c_off: int = 0  # deconv: first column of its output in the concat


def fcn_layers(arch: ArchSpec, num_vec: int) -> List[FcnLayer]:
    """ConvFeatNet + heads in reference order (det_base.py:167-183,196-224,367-368; det_base_sunrgbd.py:178-200)."""
    S, V, D = arch.num_scales, num_vec, arch.deconv_out
    L = [FcnLayer("block1_conv1", "conv", (("feat1", arch.mlps[0][2] + V),), arch.block1_out, 3, 1, 0)]
    for i, w in enumerate(arch.block_widths, 2):
        c1, c2 = "block%d_conv1" % i, "block%d_conv2" % i
        L += [FcnLayer(c1, "conv", ((L[-1].name, L[-1].Cout),), w, 3, 2, i - 1),
              FcnLayer(c2, "conv", ((c1, w),), w, 3, 1, i - 1),
              FcnLayer("block%d_merge" % i, "merge", ((c2, w), ("feat%d" % i, arch.mlps[i - 1][2] + V)), w, 1, 1, i - 1)]
    merges = [m for m in L if m.kind == "merge"]
    deconvs = [FcnLayer("block%d_deconv" % (j + 2), "deconv", ((m.name, m.Cout),), D, 2 ** j, 2 ** j, 1, D * j)
               for j, m in enumerate(merges)]
    return L + deconvs + [FcnLayer("heads", "heads", tuple((d.name, D) for d in deconvs), None, 1, 1, 1)]


# Named workloads of BASELINE.json `configs` -> (yaml, dataset, num_vec, arch)
WORKLOADS = {
    "car": dict(yaml="det_sample.yaml", num_vec=3, arch=ARCH_KITTI),
    "people": dict(yaml="det_sample_people.yaml", num_vec=3, arch=ARCH_KITTI),
    "sunrgbd": dict(yaml="det_sample_sunrgbd.yaml", num_vec=10, arch=ARCH_SUNRGBD),
    "refine_car": dict(yaml="refine_car.yaml", num_vec=3, arch=ARCH_KITTI),
}


def load_workload(name: str):
    """Reset the local cfg, merge ``cfgs/<yaml>`` and return (cfg, workload dict)."""
    w = WORKLOADS[name]
    reset_cfg()
    merge_cfg_from_file(os.path.join(CFG_DIR, w["yaml"]))
    return _local_cfg, w
