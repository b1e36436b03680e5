"""GPU: persistent FCN kernel (csrc/fcn_mega.cu, ``fcn_mega_forward``) - all conv layers + heads + decode in one
launch with dynamic job fetching and per-tile dependency counters.

It performs the SAME wgmma arithmetic per output tile as the per-layer TMA GEMM (same K order, same epilogue),
so the two paths must agree BIT-EXACTLY; parity with the oracle then follows from tests/test_gpu_tc.py and
tests/test_gpu_bench_config.py (which run whichever path is the default)."""
import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, load_golden
from test_gpu_parity import build_model, cuda_data, dev

pytestmark = pytest.mark.gpu


def _forward(monkeypatch, mega, w, sd, cfg, d, graph=False, grid=None, shape=None):
    monkeypatch.setenv("FCN_MEGA", "1" if mega else "0")
    if grid is not None:
        monkeypatch.setenv("FCN_MEGA_GRID", str(grid))
    else:
        monkeypatch.delenv("FCN_MEGA_GRID", raising=False)
    m = build_model(w, sd, cfg, precision=1, graph=graph)
    out = [o.clone() for o in m(d)]
    plan = m.engine().plan(*shape)
    assert (plan.mega_args is not None) == bool(mega)
    cls, reg = plan.logits()
    return m, plan, out, cls.clone(), reg.clone()


def _shape(data, w):
    S = w["arch"].num_scales
    return (data["point_cloud"].shape[0], data["point_cloud"].shape[2],
            [data["center_ref%d" % (i + 1)].shape[2] for i in range(S)])


@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_mega_equals_per_layer_path_bit_exact(name, monkeypatch):
    g, data, sd, w, cfg = load_golden(name)
    d = cuda_data(data)
    shape = _shape(data, w)
    _, _, o0, c0, r0 = _forward(monkeypatch, False, w, sd, cfg, d, shape=shape)
    m1, p1, o1, c1, r1 = _forward(monkeypatch, True, w, sd, cfg, d, shape=shape)
    assert torch.equal(c0, c1) and torch.equal(r0, r1)
    for a, b in zip(o0, o1):
        assert torch.equal(a, b)
    # self-cleaning scheduler state: counters back to zero, epoch counts the forwards; repeated forwards identical
    torch.cuda.synchronize()
    st = p1.mega_sync.cpu().numpy()
    assert st[0] == 0 and st[1] == 0 and st[2] == 1 and not st[4:].any()
    for rep in range(3):
        o2 = m1(d)
        for a, b in zip(o1, o2):
            assert torch.equal(a, b)
    torch.cuda.synchronize()
    st = p1.mega_sync.cpu().numpy()
    assert st[0] == 0 and st[1] == 0 and st[2] == 4 and not st[4:].any()


@pytest.mark.parametrize("grid", [1, 3, 40])
def test_mega_any_grid_size(grid, monkeypatch):
    """Deadlock-freedom does not depend on co-residency: 1 CTA (fully serial, every dependency produced by the
    same CTA), 3 CTAs (deep cross-CTA waits) and 40 CTAs give the same bits as the per-layer path."""
    g, data, sd, w, cfg = load_golden("car_full_b1")
    d = cuda_data(data)
    shape = _shape(data, w)
    _, _, o0, c0, r0 = _forward(monkeypatch, False, w, sd, cfg, d, shape=shape)
    _, _, o1, c1, r1 = _forward(monkeypatch, True, w, sd, cfg, d, grid=grid, shape=shape)
    assert torch.equal(r0, r1) and torch.equal(c0, c1)
    for a, b in zip(o0, o1):
        assert torch.equal(a, b)


def test_mega_full_size_b32_graph_and_streams(monkeypatch):
    """B=32 car (648 jobs), CUDA graph, 8 forwards in flight on 8 streams (8 persistent kernels competing for the
    SMs - the co-residency case the dynamic scheduler exists for) == per-layer path, bit-exact."""
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload("car")
    sd = synth.make_state_dict(w["arch"], 3, "KITTI", seed=7)
    data = synth.make_frustums("car", 32, seed=1234)
    d = cuda_data(data)
    shape = _shape(data, w)
    _, _, o0, c0, r0 = _forward(monkeypatch, False, w, sd, cfg, d, shape=shape)
    monkeypatch.setenv("FCN_MEGA", "1")
    m = build_model(w, sd, cfg, precision=1, graph=True)
    m.copy_outputs = False
    streams = [torch.cuda.Stream(device=dev()) for _ in range(8)]
    outs = [None] * 8
    for rep in range(4):
        for s, st in enumerate(streams):
            with torch.cuda.stream(st):
                outs[s] = m(d)
    torch.cuda.synchronize()
    assert len(m.engine()._plans) == 8 and all(p.mega_args is not None for p in m.engine()._plans.values())
    for s in range(8):
        for a, b in zip(o0, outs[s]):
            assert torch.equal(a, b), "stream %d" % s


@pytest.mark.parametrize("wl,B", [("people", 2), ("sunrgbd", 8)])
def test_mega_other_workloads(wl, B, monkeypatch):
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload(wl)
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=7)
    data = synth.make_frustums(wl, B, seed=77)
    d = cuda_data(data)
    shape = _shape(data, w)
    _, _, o0, c0, r0 = _forward(monkeypatch, False, w, sd, cfg, d, shape=shape)
    _, _, o1, c1, r1 = _forward(monkeypatch, True, w, sd, cfg, d, graph=True, shape=shape)
    assert torch.equal(r0, r1) and torch.equal(c0, c1)
    for a, b in zip(o0, o1):
        assert torch.equal(a, b)


@pytest.mark.parametrize("wl,B", [("car", 3), ("people", 2)])
def test_mega_wide_tiles_bit_exact(wl, B, monkeypatch):
    """256-wide N tiles (32-wide K stages, 64 x 256 register accumulators per warpgroup): same K order per output element as the
    128-wide tiles and the per-layer GEMMs -> bit-identical.  ("auto" picks them for >= 24 tiles per layer.)"""
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload(wl)
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=11)
    data = synth.make_frustums(wl, B, seed=5)
    d = cuda_data(data)
    shape = _shape(data, w)
    monkeypatch.setenv("FCN_MEGA_NT256", "0")
    _, _, o0, c0, r0 = _forward(monkeypatch, False, w, sd, cfg, d, shape=shape)
    monkeypatch.setenv("FCN_MEGA_NT256", "1")
    _, p1, o1, c1, r1 = _forward(monkeypatch, True, w, sd, cfg, d, graph=True, shape=shape)
    assert any(x.NT == 256 for x in p1.mega_descs())
    assert torch.equal(r0, r1) and torch.equal(c0, c1)
    for a, b in zip(o0, o1):
        assert torch.equal(a, b)


# ------------------------------------------------------------------ every intermediate buffer, per-layer bounds
def _buffers(plan):
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in plan.buf.items()}


def _assert_pads_zero(plan, bufs, what):
    for k, v in bufs.items():
        T = plan.valid_T[k]
        assert not v[:, T:].any(), "%s: pad rows of %s are not zero" % (what, k)


def _compare_buffers(monkeypatch, w, sd, cfg, data):
    d = cuda_data(data)
    shape = _shape(data, w)
    _, p0, o0, _, _ = _forward(monkeypatch, False, w, sd, cfg, d, shape=shape)
    b0 = _buffers(p0)
    _, p1, o1, _, _ = _forward(monkeypatch, True, w, sd, cfg, d, shape=shape)
    b1 = _buffers(p1)
    assert set(b0) == set(b1) and {"block1_conv1", "cat", "logits"} <= set(b0)
    for k in b0:
        assert torch.equal(b0[k], b1[k]), "buffer %s differs between the persistent and per-layer paths" % k
    _assert_pads_zero(p0, b0, "per-layer")
    _assert_pads_zero(p1, b1, "persistent")
    for a, b in zip(o0, o1):
        assert torch.equal(a, b)
    return p1


@pytest.mark.parametrize("name", ["car_full_b1", "sunrgbd_full_b2", "people_small_b2"])
def test_mega_intermediate_buffers_bit_exact(name, monkeypatch):
    """Every activation buffer of the plan (one per conv / merge layer, cat, logits), not just the six outputs."""
    g, data, sd, w, cfg = load_golden(name)
    _compare_buffers(monkeypatch, w, sd, cfg, data)


@pytest.mark.parametrize("B", [4, 5])
def test_mega_block1_rows_at_tile_boundary(B, monkeypatch):
    """car: B * P_m of the block-1 layers = 4 * 288 = 9 full 128-row tiles, and one frustum more (11.25 tiles)."""
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload("car")
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=17)
    data = synth.make_frustums("car", B, seed=31 + B)
    plan = _compare_buffers(monkeypatch, w, sd, cfg, data)
    assert (B * plan.P[0] % 128 == 0) == (B == 4)


def _layer_specs(plan):
    """exact_ref.ConvSpec of every layer of the plan, reading the plan's own (float64, device) input buffers and
    the packed weights as the tensor cores consume them (TF32-rounded)."""
    import exact_ref as X
    eng = plan.eng
    bufs = {k: v.double() for k, v in plan.buf.items()}
    specs = []
    for L, a in zip(eng.layers, plan.conv_args):
        segs = [X.ConvSeg(bufs[src], c, plan.valid_T[src], tap, st) for (src, c, tap, st) in L.segs]
        wt = X.tf32(L._wt_host.double())
        # round_out is applied by the caller's bound, not by the float64 reference
        spec = X.ConvSpec(plan.B, a.T_out, a.P_m, segs, wt, L.bias.double().cpu(), L.Cout, L.up, L.relu,
                          0, bufs[L.out], a.T_store, a.c_off)
        specs.append((L, spec, a.round_out))
    return specs


@pytest.mark.parametrize("nt256", ["1", "0"])
@pytest.mark.parametrize("wl,B", [("car", 32), ("people", 8), ("sunrgbd", 32)])
def test_mega_layerwise_error_bound(wl, B, nt256, monkeypatch):
    """At the benchmarked shapes, every element of every layer output of the persistent kernel stays within
        |out - ref| <= 2^-11 |ref| (TF32 rounding of the output, round_out layers) + K 2^-23 (sum |a||w| + |b|)
    of a float64 recomputation from the layer's own inputs (worst-case fp32 accumulation error over K terms with a
    factor-2 margin for the tensor core's operand alignment).  Far tighter than the whole-tensor oracle bounds."""
    import exact_ref as X
    from frustum_convnet_b200 import config, synth
    monkeypatch.setenv("FCN_MEGA_NT256", nt256)
    cfg, w = config.load_workload(wl)
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=23)
    data = synth.make_frustums(wl, B, seed=29)
    d = cuda_data(data)
    _, plan, _, _, _ = _forward(monkeypatch, True, w, sd, cfg, d, shape=_shape(data, w))
    assert any(x.NT == 256 for x in plan.mega_descs()) == (nt256 == "1")
    torch.cuda.synchronize()
    worst = 0.0
    for L, spec, round_out in _layer_specs(plan):
        _, pre, S = X.conv_ref(spec, with_abs=True)
        ref = torch.relu(pre) if spec.relu else pre
        n_t = ref.shape[1]
        got = spec.out[:, :n_t, spec.c_off:spec.c_off + spec.Cout]
        bound = spec.K_pad * 2.0 ** -23 * S
        if round_out:
            bound = bound + 2.0 ** -11 * ref.abs()
        err = (got - ref).abs()
        ratio = float((err / bound.clamp(min=1e-300)).max())
        worst = max(worst, ratio)
        print("%s B=%d NT256=%s %-16s max err %.3e  max err/bound %.3f" % (wl, B, nt256, L.name,
                                                                            float(err.max()), ratio))
        assert (err <= bound).all(), "%s: %d elements exceed the bound (max ratio %.3f)" % (
            L.name, int((err > bound).sum()), ratio)
    print("%s B=%d NT256=%s largest error/bound %.3f" % (wl, B, nt256, worst))
