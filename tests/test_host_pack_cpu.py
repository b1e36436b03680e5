"""Host-side weight packing, checked on the CPU against the reference-generated golden fixtures.

The engine turns the reference state dict into GEMM operands (BN folded, kernel taps / concat sources laid out
along K, transposed-conv taps laid out along N, heads fused, tensor-core stage images pre-swizzled).  These
tests replay the packed operands with plain float64 matmuls - no CUDA, no oracle - and compare with what the
reference itself produced (tests/golden/*.npz: `x`, `cls`, `reg` of models/det_base.py:163-224,367-368), so a
packing bug cannot hide behind a kernel bug or vice versa.
"""
import numpy as np
import pytest
import torch

from frustum_convnet_b200 import config
from frustum_convnet_b200.engine import FrustumEngine, pack_sw128, tf32_rna


def _engine(golden_loader, name):
    g, data, sd, w, cfg = golden_loader(name)
    tsd = {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}
    eng = FrustumEngine(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, cfg.DATA.HEIGHT_HALF, 12, tsd, "cpu",
                        precision=1)
    return eng, g


def _replay_fcn(eng, feats):
    """feats: list of (B, T_i, C_i) float64 position-major maps -> (x (B,T2,768), cls, reg) float64."""
    B = feats[0].shape[0]
    buf = {"feat%d" % (i + 1): f for i, f in enumerate(feats)}
    T2 = feats[1].shape[1]
    ncat = 256 * (eng.arch.num_scales - 1)
    buf["cat"] = torch.zeros(B, T2, ncat, dtype=torch.float64)
    for lay in eng.layers:
        stride = lay.segs[0][3]
        T_src = buf[lay.segs[0][0]].shape[1]
        T_out = (T_src - 1) // stride + 1
        cols = []
        for src, C, tap, s in lay.segs:
            x = buf[src]
            a = torch.zeros(B, T_out, (C + 31) // 32 * 32, dtype=torch.float64)
            for t in range(T_out):
                ts = t * s + tap
                if 0 <= ts < x.shape[1]:
                    a[:, t, :C] = x[:, ts, :C]
            cols.append(a)
        A = torch.cat(cols, 2)
        if A.shape[2] < lay.K_pad:   # 64-wide K stages: trailing all-zero block
            A = torch.cat([A, torch.zeros(B, T_out, lay.K_pad - A.shape[2], dtype=torch.float64)], 2)
        assert A.shape[2] == lay.wt.shape[0] == lay.K_pad
        out = A @ lay.wt.double() + lay.bias.double()
        if lay.relu:
            out = out.clamp_min(0)
        if lay.out == "cat":       # transposed conv: column group j -> position t*up + j
            for j in range(lay.up):
                tt = torch.arange(T_out) * lay.up + j
                keep = tt < T2
                buf["cat"][:, tt[keep], lay.c_off: lay.c_off + lay.Cout] = \
                    out[:, keep, j * lay.Cout:(j + 1) * lay.Cout]
        else:
            assert lay.up == 1
            buf[lay.out] = out[:, :, :lay.Cout]
    return buf["cat"], buf["logits"][:, :, :2], buf["logits"][:, :, 2:2 + eng.out_size]


@pytest.mark.parametrize("name", ["car_small_b3", "people_small_b2"])
def test_packed_fcn_operands_reproduce_reference_outputs(golden_loader, name):
    eng, g = _engine(golden_loader, name)
    S = eng.arch.num_scales
    feats = [torch.from_numpy(g["feat%d" % (i + 1)]).double().permute(0, 2, 1).contiguous() for i in range(S)]
    x, cls, reg = _replay_fcn(eng, feats)
    for mine, ref in ((x, g["x"]), (cls, g["cls"]), (reg, g["reg"])):
        ref = torch.from_numpy(ref).double().permute(0, 2, 1)
        assert mine.shape == ref.shape
        # fp32 reference vs float64 replay of fp32-rounded folded weights
        assert float((mine - ref).abs().max()) <= 2e-4 * max(1.0, float(ref.abs().max()))


def test_layer_table_matches_reference_fcn_structure(golden_loader):
    eng, _ = _engine(golden_loader, "car_small_b3")
    names = [l.name for l in eng.layers]
    assert names == ["block1_conv1",
                     "block2_conv1", "block2_conv2", "block2_merge",
                     "block3_conv1", "block3_conv2", "block3_merge",
                     "block4_conv1", "block4_conv2", "block4_merge",
                     "block2_deconv", "block3_deconv", "block4_deconv", "heads"]
    for l in eng.layers:
        assert l.K_pad % 64 == 0 and l.n_cols % 64 == 0 and l.wt.shape == (l.K_pad, l.n_cols)
    # transposed convs: kernel == stride == 1, 2, 4 (det_base.py:181-183)
    assert [l.up for l in eng.layers if "deconv" in l.name] == [1, 2, 4]


def test_tf32_rounding_is_nearest_ties_away():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(4096).astype(np.float32) * 37.0,
                        np.float32([0.0, -0.0, 1.0, -1.0, 1e-30, 3.0e38]),
                        # exact ties: 1 + (2k+1) * 2^-11
                        np.float32([1.0 + (2 * k + 1) * 2.0 ** -11 for k in range(8)]),
                        -np.float32([1.0 + (2 * k + 1) * 2.0 ** -11 for k in range(8)])])
    got = tf32_rna(torch.from_numpy(x)).numpy()
    m, e = np.frexp(x.astype(np.float64))          # |m| in [0.5, 1): 11 significant bits survive
    want = np.sign(m) * np.floor(np.abs(m) * 2048.0 + 0.5) / 2048.0 * np.exp2(e.astype(np.float64))
    assert np.array_equal(got.astype(np.float64), want)
    assert np.all((got.view(np.uint32) & 0x1FFF) == 0)      # 13 low mantissa bits cleared


@pytest.mark.parametrize("n_chunk", [64, 128, 256])
def test_sw128_stage_image_layout(n_chunk):
    """Image element (chunk nc, K block kb, row n, 16-byte slot p, e) == W[nc*n_chunk + n, kb*32 + (p ^ (n & 7))*4 + e]."""
    rng = np.random.default_rng(1)
    co, ci = 2 * n_chunk, 96
    w = torch.from_numpy(rng.standard_normal((co, ci)).astype(np.float32))
    img = pack_sw128(w, n_chunk).view(co // n_chunk, ci // 32, n_chunk, 8, 4)
    wr = tf32_rna(w)
    for nc in range(co // n_chunk):
        for kb in range(ci // 32):
            for n in (0, 1, 7, 8, 13, n_chunk - 1):
                for p in range(8):
                    src = kb * 32 + (p ^ (n & 7)) * 4
                    assert torch.equal(img[nc, kb, n, p], wr[nc * n_chunk + n, src: src + 4])
    # every stage is a whole number of 1024-byte swizzle atoms (8 rows x 128 B)
    assert (n_chunk * 128) % 1024 == 0


def test_bench_host_helpers():
    import bench
    ring = bench._OutRing(4)
    views = [ring(10, "cpu") for _ in range(4)]
    assert all(v.data_ptr() == ring.buf.data_ptr() + 40 * k for k, v in enumerate(views))
    with pytest.raises(AssertionError):
        ring(10, "cpu")
    assert bench.host_threads() >= 1
    assert "det_sample.yaml" in bench.workload_name("car", 32)
    s = bench.ClockSampler(0)       # no NVML / nvidia-smi in the CPU container: must degrade, not raise
    s.start()
    out = s.stop()
    assert "reasons" in out and "sm_mhz" in out
    assert set(bench.ALGO) >= set(config.WORKLOADS) - {"refine_car"}


@pytest.mark.parametrize("name", ["car_small_b3", "sunrgbd_full_b2"])
def test_packed_pointnet_weights_reproduce_reference_features(golden_loader, name):
    """Folded (conv1x1 + BN) weights of every scale, replayed in float64 on the reference's own grouping
    (golden idx/cnt), give the reference's pooled features (det_base.py:62-103,126-159)."""
    g, data, sd, w, cfg = golden_loader(name)
    eng, _ = _engine(golden_loader, name)
    pc = torch.from_numpy(data["point_cloud"]).double()                     # (B,3,N)
    B = pc.shape[0]
    for i, lay in enumerate(eng.pn):
        idx = torch.from_numpy(g["idx%d" % (i + 1)].astype(np.int64))        # (B,T,K)
        cnt = torch.from_numpy(g["cnt%d" % (i + 1)].astype(np.int64))
        ctr = torch.from_numpy(data["center_ref%d" % (i + 1)]).double()      # (B,3,T)
        T, K = idx.shape[1], idx.shape[2]
        grouped = torch.gather(pc, 2, idx.view(B, 1, T * K).expand(-1, 3, -1)).view(B, 3, T, K)
        x = (grouped - ctr.unsqueeze(3)).permute(0, 2, 3, 1)                  # (B,T,K,3)
        for j in (1, 2, 3):
            x = (x @ lay["w%dt" % j].double() + lay["b%d" % j].double()).clamp_min(0)
        feat = (x * (cnt > 0).view(B, T, 1, 1)).max(2)[0]                     # (B,T,C3)
        ref = torch.from_numpy(g["feat%d" % (i + 1)]).double().permute(0, 2, 1)
        C3 = feat.shape[2]
        assert float((feat - ref[:, :, :C3]).abs().max()) <= 2e-4 * max(1.0, float(ref.abs().max()))
        one_hot = torch.from_numpy(data["one_hot"]).double()
        assert torch.equal(ref[:, :, C3:], one_hot[:, None, :].expand(-1, T, -1))


@pytest.mark.parametrize("wl", ["car", "people", "sunrgbd"])
def test_roofline_denominators_follow_from_the_architecture(wl):
    """bench.ALGO (SURVEY.md 8(d): algorithmic bytes and nominal FLOPs per frustum) recomputed from the layer
    widths, section counts and sample counts - the numbers `roofline.achieved` / `hbm.achieved` are built on."""
    import bench
    from frustum_convnet_b200 import synth
    cfg, w = config.load_workload(wl)
    arch, V = w["arch"], w["num_vec"]
    T, K, N = list(synth.section_counts(wl)), arch.nsample, synth._PRESETS[wl]["N"]
    mac = sum(t * k * (3 * c1 + c1 * c2 + c2 * c3) for (c1, c2, c3), t, k in zip(arch.mlps, T, K))
    level = {}
    for L in config.fcn_layers(arch, V):
        level[L.name] = L.level
        if L.kind == "heads":
            continue
        ci = sum(c for _, c in L.srcs)
        lv = level[L.srcs[0][0]] if L.kind == "deconv" else L.level
        mac += T[lv] * ci * L.Cout * L.k       # conv: per output position; transposed conv: per input position
    n_reg = 39 if arch.num_scales == 4 else 67   # det_base.py:248 / det_base_sunrgbd.py
    mac += T[1] * arch.reg_in * (2 + n_reg)
    n_size = 3 if arch.num_scales == 4 else 10
    out_bytes = T[1] * (2 + 3 + 1 + 3 + 12 + n_size) * 4
    in_bytes = (3 * N + 3 * sum(T) + V) * 4
    assert bench.ALGO[wl]["gflop"] == pytest.approx(2 * mac / 1e9, rel=2e-4)
    assert bench.ALGO[wl]["bytes"] == pytest.approx(in_bytes + out_bytes, rel=3e-3)
