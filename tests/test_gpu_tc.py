"""GPU: TF32 tensor-core (wgmma) path.

Tolerance: kind::tf32 keeps a 10-bit mantissa (operands rounded with cvt.rna, fp32 accumulate), the
same arithmetic PyTorch/cuDNN use for convolutions by default on Ampere+ GPUs
(torch.backends.cudnn.allow_tf32 = True).  Stated bounds (tests/test_gpu_bench_config.py has the derivation):
linear tensors (features, FCN output, logits, centre offsets)  max|a-b| <= 2.5e-3 * max(1, max|ref|)  and
rms(a-b) <= 1.5e-3 * rms(ref); softmax outputs  max|dp| <= 0.5 * 2.5e-3 * max|logits_ref|, rms <= 1e-3.
Errors are printed.
"""
import numpy as np
import pytest
import torch

from conftest import GOLDEN_CASES, load_golden
from test_gpu_bench_config import _unambiguous, close_tf32
from test_gpu_parity import build_model, close, cuda_data, dev

pytestmark = pytest.mark.gpu
TF32_TOL = 2.5e-3


@pytest.mark.parametrize("N,K", [(128, 32), (128, 64), (64, 64), (128, 192), (64, 128), (64, 256), (256, 128)])
def test_umma_selftest_matches_fp64_matmul(N, K):
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200.engine import pack_sw128, tf32_rna
    g = torch.Generator().manual_seed(N * 1000 + K)
    A = torch.randn(128, K, generator=g)
    W = torch.randn(N, K, generator=g)
    img = pack_sw128(W.to(dev()), N)
    D = torch.full((128, N), float("nan"), device=dev())
    Ad = A.to(dev()).contiguous()
    _lib.call("fcn_selftest_umma", N, K, Ad.data_ptr(), img.data_ptr(), D.data_ptr(),
              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref = tf32_rna(A).double() @ tf32_rna(W).double().t()
    err = float((D.cpu().double() - ref).abs().max())
    print("umma selftest N=%d K=%d max err %.3e" % (N, K, err))
    assert err < 1e-3 * max(1.0, float(ref.abs().max())), err


@pytest.mark.parametrize("N,K", [(64, 256), (128, 224), (256, 128), (256, 32)])
def test_umma_selftest_exact_integer_operands(N, K):
    """m64nNk8 for N = 64, 128, 256 with integer operands (every partial sum an integer < 2^22, so the fp32
    accumulation is exact in any order): the product must be bit-identical to the int64 matmul."""
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200.engine import pack_sw128
    g = torch.Generator().manual_seed(N + K)
    A = torch.randint(-1000, 1001, (128, K), generator=g)       # < 2^11: TF32 values
    W = torch.randint(-15, 16, (N, K), generator=g)
    assert int((A.abs() @ W.abs().t()).max()) < (1 << 22)
    img = pack_sw128(W.float().to(dev()), N)
    D = torch.full((128, N), float("nan"), device=dev())
    Ad = A.float().to(dev()).contiguous()
    _lib.call("fcn_selftest_umma", N, K, Ad.data_ptr(), img.data_ptr(), D.data_ptr(),
              torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    ref = (A @ W.t()).float()
    bad = int((D.cpu() != ref).sum())
    assert bad == 0, "%d of %d elements differ from the exact product" % (bad, ref.numel())


def test_umma_selftest_rejects_k_beyond_shared_memory():
    from frustum_convnet_b200 import _lib
    x = torch.zeros(128 * 256, device=dev())
    for N, K in ((128, 256), (256, 160)):
        with pytest.raises(RuntimeError, match="shared memory"):
            _lib.call("fcn_selftest_umma", N, K, x.data_ptr(), x.data_ptr(), x.data_ptr(),
                      torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("cluster", ["1", "0"])
@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_pointnet_feat_tf32_matches_golden(name, cluster, monkeypatch):
    """cluster=1: the 128- and 256-channel scales on 2-CTA clusters (weight stages multicast to both CTAs);
    cluster=0: 1-CTA kernel everywhere."""
    monkeypatch.setenv("FCN_PN_CLUSTER", cluster)
    g, data, sd, w, cfg = load_golden(name)
    m = build_model(w, sd, cfg)
    m.feat_net.precision = 1
    d = cuda_data(data)
    S = w["arch"].num_scales
    feats = m.feat_net(d["point_cloud"], [d["center_ref%d" % (i + 1)] for i in range(S)], None, d["one_hot"])
    for i, f in enumerate(feats):
        ref = g["feat%d" % (i + 1)]
        err = float(np.abs(f.cpu().numpy() - ref).max())
        print("%s feat%d tf32 max err %.3e (max |ref| %.2f)" % (name, i + 1, err, np.abs(ref).max()))
        close_tf32(f, ref, "%s feat%d tf32" % (name, i + 1))


@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_conv_feat_net_and_forward_tf32_match_golden(name):
    """FCN on tensor cores (up to 11 chained TF32 GEMMs) and the whole forward, all six outputs."""
    g, data, sd, w, cfg = load_golden(name)
    m = build_model(w, sd, cfg)
    m.conv_net.precision = 1
    S = w["arch"].num_scales
    feats = [torch.from_numpy(g["feat%d" % (i + 1)]).to(dev()) for i in range(S)]
    x = m.conv_net(*feats)
    close_tf32(x, g["x"], name + " conv_net tf32")
    m.precision = 1
    out = m(cuda_data(data))
    B = data["point_cloud"].shape[0]
    plan = m.engine().plan(B, data["point_cloud"].shape[2],
                           [data["center_ref%d" % (i + 1)].shape[2] for i in range(S)])
    cls, reg = plan.logits()
    close_tf32(cls.view(B, -1, 2).permute(0, 2, 1), g["cls"], name + " cls logits tf32")
    close_tf32(reg.view(B, -1, reg.shape[1]).permute(0, 2, 1), g["reg"], name + " reg logits tf32")
    ref2 = np.transpose(data["center_ref2"], (0, 2, 1))
    close_tf32(out[1].cpu().numpy() - ref2, g["out1"] - ref2, name + " centre offsets tf32")
    nb = 12
    ns = g["out5"].shape[-1]
    groups = {0: g["cls"], 4: g["reg"][:, 3:3 + nb], 5: g["reg"][:, 3 + 2 * nb:3 + 2 * nb + ns]}
    for j in (0, 4, 5):
        close_tf32(out[j], g["out%d" % j], "%s out%d softmax tf32" % (name, j),
                   max_lim=0.5 * TF32_TOL * float(np.abs(groups[j]).max()), rms_lim=1e-3)
    ok = _unambiguous([torch.from_numpy(g["out%d" % j]) for j in range(6)])
    close_tf32(out[2], g["out2"], name + " heading tf32", mask=ok)
    close_tf32(out[3], g["out3"], name + " size tf32", mask=ok)


def test_tf32_full_size_car_b32_vs_fp32_path():
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload("car")
    sd = synth.make_state_dict(w["arch"], 3, "KITTI", seed=21)
    m0 = build_model(w, sd, cfg)
    m1 = build_model(w, sd, cfg)
    m1.precision = 1
    data = synth.make_frustums("car", 32, seed=77)
    d = cuda_data(data)
    o0 = m0(d)
    o1 = m1(d)
    for j in (0, 1, 4, 5):
        close(o1[j], o0[j], tol=1e-2, what="tf32 vs fp32 out%d" % j)
    o2 = m1(d)
    for a, b in zip(o1, o2):
        assert torch.equal(a, b)      # deterministic (max-combine is order independent)


@pytest.mark.parametrize("variant", ["FCN_CONV_TMA=0", "FCN_GROUP_SCAN=1", "FCN_PN_CLUSTER=0"])
@pytest.mark.parametrize("name", ["car_full_b1", "sunrgbd_full_b2"])
def test_alternative_kernel_variants_match_golden(name, variant, monkeypatch):
    """The documented alternative kernels (cp.async-gather conv GEMM, section-scan grouping, 1-CTA PointNet
    at 128/256 channels) stay parity-green: whole forward vs the reference fixture."""
    k, v = variant.split("=")
    monkeypatch.setenv(k, v)
    g, data, sd, w, cfg = load_golden(name)
    m = build_model(w, sd, cfg)
    m.precision = 1
    out = m(cuda_data(data))
    lim = 0.5 * TF32_TOL * float(np.abs(g["cls"]).max())
    close_tf32(out[0], g["out0"], variant + " cls_probs", max_lim=lim, rms_lim=1e-3)
    ref2 = np.transpose(data["center_ref2"], (0, 2, 1))
    close_tf32(out[1].cpu().numpy() - ref2, g["out1"] - ref2, variant + " centre offsets")
    close_tf32(out[4], g["out4"], variant + " heading_probs",
               max_lim=0.5 * TF32_TOL * float(np.abs(g["reg"][:, 3:15]).max()), rms_lim=1e-3)
