"""Seeded synthetic frustums and seeded model parameters.

There is no dataset and no checkpoint offline, so every test, golden fixture
and benchmark draws from this generator.  It mimics what the reference data
providers emit (channel-first float32, see datasets/provider_sample.py:187-193,
249-254) and how they build the T depth-section centres
(``generate_ref``: provider_sample.py:291-327 for the detection stage,
provider_sample_refine.py:336-385 for the refinement stage).

Everything is generated with numpy's PCG64 (stable across versions/machines),
never with torch RNG, so the same seed yields the same bytes in the authoring
container and on the GPU box.
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np

from .config import DATASET_INFO, WORKLOADS, ArchSpec, fcn_layers

_PRESETS = {
    # name: (N, strides, max_depth, z0 range, sigma, kind)
    "car": dict(N=1024, strides=(0.25, 0.5, 1.0, 2.0), max_depth=70.0, z0=(5.0, 60.0),
                sigma=0.8, kind="det"),
    "people": dict(N=1024, strides=(0.1, 0.2, 0.4, 0.8), max_depth=70.0, z0=(5.0, 60.0),
                   sigma=0.8, kind="det"),
    "sunrgbd": dict(N=2048, strides=(0.1, 0.2, 0.4, 0.8, 1.6), max_depth=8.0, z0=(1.0, 6.0),
                    sigma=0.3, kind="det"),
    "refine_car": dict(N=512, strides=(0.1, 0.2, 0.4, 0.8), max_depth=None, z0=None,
                       sigma=None, kind="refine"),
}


def section_counts(workload: str, max_depth=None):
    """T per scale for a workload (len(arange(0, max_depth, s)))."""
    p = _PRESETS[workload]
    if p["kind"] == "refine":
        half = 0.977
        return tuple(len(np.arange(-half, half, s)) for s in p["strides"])
    md = p["max_depth"] if max_depth is None else max_depth
    return tuple(len(np.arange(0, md, s)) for s in p["strides"])


def make_frustums(workload: str, B: int, seed: int = 1234, max_depth=None, N=None,
                  with_labels: bool = False):
    """Return a dict of numpy arrays keyed like the reference data dict
    (models/det_base.py:336-347)."""
    p = _PRESETS[workload]
    w = WORKLOADS[workload]
    rng = np.random.default_rng(seed)
    N = p["N"] if N is None else N
    V = w["num_vec"]
    out = OrderedDict()
    if p["kind"] == "det":
        md = float(p["max_depth"] if max_depth is None else max_depth)
        lo, hi = p["z0"]
        hi = min(hi, md * 0.85)
        lo = min(lo, hi * 0.5)
        z0 = rng.uniform(lo, hi, size=(B, 1))
        n_obj = N // 2
        z_obj = rng.normal(z0, p["sigma"], size=(B, n_obj))
        z_bg = rng.uniform(0.0, md, size=(B, N - n_obj))
        z = np.concatenate([z_obj, z_bg], axis=1)
        z = np.clip(z, 0.0, md)
        # shuffle so object points are not the first half of the index range
        perm = np.argsort(rng.random((B, N)), axis=1)
        z = np.take_along_axis(z, perm, axis=1)
        x = z * np.tan(rng.uniform(-0.08, 0.08, size=(B, N)))
        y = rng.uniform(-1.5, 1.5, size=(B, N))
        pc = np.stack([x, y, z], axis=1)  # (B,3,N)
        # 10 % duplicated points (with-replacement resampling, provider_sample.py:164-171)
        ndup = N // 10
        for b in range(B):
            dst = rng.choice(N, size=ndup, replace=False)
            src = rng.integers(0, N, size=ndup)
            pc[b][:, dst] = pc[b][:, src]
        out["point_cloud"] = pc.astype(np.float32)
        for i, s in enumerate(p["strides"]):
            zc = np.arange(0, md, s) + s / 2.0  # float64 then cast, as the provider does
            c = np.zeros((B, 3, len(zc)), dtype=np.float64)
            c[:, 2, :] = zc[None, :]
            out["center_ref%d" % (i + 1)] = c.astype(np.float32)
    else:
        hx, hy, hz = 2.33, 0.92, 0.977
        pc = np.stack([rng.uniform(-hx, hx, size=(B, N)), rng.uniform(-hy, hy, size=(B, N)),
                       rng.uniform(-hz, hz, size=(B, N))], axis=1)
        out["point_cloud"] = pc.astype(np.float32)
        for i, s in enumerate(p["strides"]):
            zc = np.arange(-hz, hz, s) + s / 2.0
            c = np.zeros((B, 3, len(zc)), dtype=np.float64)
            c[:, 2, :] = zc[None, :]
            out["center_ref%d" % (i + 1)] = c.astype(np.float32)
    one_hot = np.zeros((B, V), dtype=np.float32)
    one_hot[np.arange(B), rng.integers(0, V, size=B) if V > 3 else 0] = 1.0
    out["one_hot"] = one_hot
    if with_labels:
        T2 = out["center_ref2"].shape[2]
        cls = rng.integers(-1, 2, size=(B, T2)).astype(np.int64)
        cls[:, T2 // 2] = 1  # at least one foreground section per frustum (det_base.py:416)
        out["cls_label"] = cls
        mean = DATASET_INFO["KITTI" if V == 3 else "SUNRGBD"].MEAN_SIZE_ARRAY
        out["size_class"] = np.zeros((B, 1), dtype=np.int64)
        out["box3d_center"] = rng.normal(0.0, 0.2, size=(B, 3)).astype(np.float32)
        out["box3d_heading"] = rng.uniform(-0.3, 0.3, size=(B, 1)).astype(np.float32)
        out["box3d_size"] = np.tile(mean[0][None, :], (B, 1)).astype(np.float32)
    return out


# --------------------------------------------------------------------------
# parameters
# --------------------------------------------------------------------------
def reg_out_size(dataset: str, num_bins: int = 12) -> int:
    return 3 + num_bins * 2 + DATASET_INFO[dataset].NUM_SIZE_CLUSTER * 4


def make_state_dict(arch: ArchSpec, num_vec: int, dataset: str, seed: int = 7,
                    num_bins: int = 12):
    """Seeded parameters/buffers under the reference's state-dict names
    (SURVEY.md section 8(b)).  BN affine and running statistics are randomised so
    that BN folding is actually exercised (default init would hide errors)."""
    rng = np.random.default_rng(seed)
    sd = OrderedDict()

    def bn(prefix, c):
        sd[prefix + ".weight"] = rng.uniform(0.5, 1.5, size=c).astype(np.float32)
        sd[prefix + ".bias"] = rng.normal(0, 0.1, size=c).astype(np.float32)
        sd[prefix + ".running_mean"] = rng.normal(0, 0.1, size=c).astype(np.float32)
        sd[prefix + ".running_var"] = rng.uniform(0.5, 1.5, size=c).astype(np.float32)
        sd[prefix + ".num_batches_tracked"] = np.array(0, dtype=np.int64)

    for i, mlp in enumerate(arch.mlps):
        cin = 3
        for j, co in enumerate(mlp):
            p = "feat_net.pointnet%d.conv%d" % (i + 1, j + 1)
            sd[p + ".0.weight"] = rng.normal(0, np.sqrt(2.0 / cin), size=(co, cin, 1, 1)).astype(np.float32)
            bn(p + ".1", co)
            cin = co
    for L in fcn_layers(arch, num_vec):
        if L.kind == "heads":       # drawn below, under their own names
            continue
        ci, co, k, p = sum(c for _, c in L.srcs), L.Cout, L.k, "conv_net." + L.name
        if L.kind == "deconv":
            sd[p + ".0.weight"] = rng.normal(0, np.sqrt(2.0 / (co * k)), size=(ci, co, k)).astype(np.float32)
        else:
            sd[p + ".0.weight"] = rng.normal(0, np.sqrt(2.0 / (ci * k)), size=(co, ci, k)).astype(np.float32)
        bn(p + ".1", co)
    osz = reg_out_size(dataset, num_bins)
    bound = np.sqrt(6.0 / arch.reg_in)
    sd["reg_out.weight"] = rng.uniform(-bound, bound, size=(osz, arch.reg_in, 1)).astype(np.float32)
    sd["reg_out.bias"] = rng.normal(0, 0.05, size=osz).astype(np.float32)
    sd["cls_out.weight"] = rng.uniform(-bound, bound, size=(2, arch.reg_in, 1)).astype(np.float32)
    sd["cls_out.bias"] = rng.normal(0, 0.05, size=2).astype(np.float32)
    return sd
