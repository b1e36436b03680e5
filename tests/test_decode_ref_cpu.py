"""The float32 restatement of the eval decode (tests/decode_ref.py) on the CPU, against three things:

  * the reference's own outputs: on every golden case the centre, heading and size of the fixture are reproduced
    bit-exactly, and the fixture's arg-max labels lie in the restatement's label sets;
  * torch's softmax and argmax (the model's eval branch, restated with torch operations) on the crafted edge rows
    of decode_ref.crafted_rows, non-finite rows included;
  * csrc/decode.cuh compiled with g++ twice: without multiply-add contraction it passes every case; with
    contraction the bit-exact heading and size checks fail, which proves the cases can see a contracted decode
    on a machine without a GPU.
"""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

import decode_ref as D
from conftest import GOLDEN_CASES, load_golden
from toolchain import fma_cpu, host_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "frustum_convnet_b200", "csrc", "decode.cuh")
NHS = (1, 2, 12, 24, 64)
NSS = (1, 3, 10, 64)
MODES = {"no_contraction": ("-ffp-contract=off",), "contracted": ("-mfma", "-ffp-contract=fast")}

# the CUDA intrinsics decode.cuh uses, as plain host functions (one rounding each)
CUDA_SHIM = r'''
#pragma once
#include <math.h>
#define __device__
#define __forceinline__ inline
template <class T> inline T __ldg(const T *p) { return *p; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fmul_rn(float a, float b) { return a * b; }
'''

HARNESS = r'''
#include "%s"
extern "C" void host_decode(int B, int T, int pitch, int ld, int NH, int NS, const float *logits,
                            const float *center_ref, const float *mean_size, float *cls, float *center,
                            float *heading, float *size, float *hp, float *sp) {
    fcn::DecodeOut out = {cls, center, heading, size, hp, sp};
    for (int r = 0; r < B * T; ++r) {
        const int b = r / T, t = r - b * T;
        fcn::decode_row(logits + ((size_t)b * pitch + t) * ld, r, b, t, T, NH, NS, center_ref, mean_size, &out, 1);
    }
}
'''


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("decode_host")
    (d / "cuda_runtime.h").write_text(CUDA_SHIM)
    return {mode: host_library(HARNESS % HDR, flags, (str(d),)) for mode, flags in MODES.items()
            if mode != "contracted" or fma_cpu()}


def host_decode(lib, rows, B, T, NH, NS, center_ref, mean_size):
    rows = np.ascontiguousarray(rows, np.float32)
    cr = np.ascontiguousarray(center_ref, np.float32)
    ms = np.ascontiguousarray(mean_size, np.float32)
    R = B * T
    outs = [np.full(s, np.float32(-7.0), np.float32) for s in ((R, 2), (R, 3), (R,), (R, 3), (R, NH), (R, NS))]
    P = ctypes.c_void_p
    lib.host_decode(B, T, T, rows.shape[1], NH, NS, P(rows.ctypes.data), P(cr.ctypes.data), P(ms.ctypes.data),
                    *[P(o.ctypes.data) for o in outs])
    return outs


def _mean_size(NS, seed=0):
    """Cluster mean sizes for NS clusters (the datasets' own where NS matches one)."""
    from frustum_convnet_b200.config import DATASET_INFO
    for info in DATASET_INFO.values():
        if info.NUM_SIZE_CLUSTER == NS:
            return info.MEAN_SIZE_ARRAY.astype(np.float32)
    return np.random.default_rng(seed).uniform(0.2, 4.0, (NS, 3)).astype(np.float32)


def _crafted_case(NH, NS, seed=0):
    mean = _mean_size(NS, seed)
    rows, fam = D.crafted_rows(NH, NS, seed=seed, mean_size=mean)
    B = 2
    rows = np.concatenate([rows, rows[:len(rows) % B]]) if len(rows) % B else rows
    T = len(rows) // B
    cr = np.random.default_rng(seed + 1).normal(0, 10, (B, 3, T)).astype(np.float32)
    return rows, fam, B, T, cr, mean


def check_families(o, fam, outs, hl, sl, what):
    """The family expectations that the general check does not already pin: explicit labels, exact class
    probabilities, the angle at and just above pi, the exact zero size."""
    cls, _, heading, size, _, _ = [np.asarray(x) for x in outs]
    heading = heading.reshape(-1)
    for name, v in fam.items():
        if name == "cls_want":
            continue
        idx, hls, sls = v
        for i, h, s in zip(idx, hls, sls):
            if h is not None:
                assert hl[i] == h, "%s %s row %d: heading label %d, want %d" % (what, name, i, hl[i], h)
            if s is not None:
                assert sl[i] == s, "%s %s row %d: size label %d, want %d" % (what, name, i, sl[i], s)
    assert np.array_equal(cls.reshape(-1, 2)[fam["cls_exact"][0]], fam["cls_want"]), what
    hl_pi, _, res_up = D.residuals_at_pi(o.NH)
    assert heading[fam["at_pi"][0][0]] == D.PI32, what
    above = D._pre_wrap(hl_pi, res_up, o.NH)
    assert above > D.PI32 and heading[fam["above_pi"][0][0]] == np.float32(above - D.TWO_PI32) < 0, what
    if o.NH > 1:
        assert above == np.nextafter(D.PI32, np.float32(np.inf)), what
    assert heading[fam["negative"][0][0]] < 0, what
    assert (size.reshape(-1, 3)[fam["size_zero"][0][0]] == 0).all(), what


# ------------------------------------------------------------------ the reference's outputs
@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_restatement_reproduces_reference_outputs(name):
    from frustum_convnet_b200.config import DATASET_INFO
    g, data, sd, w, cfg = load_golden(name)
    B, _, T = g["cls"].shape
    NH = cfg.DATA.NUM_HEADING_BIN
    NS = g["out5"].shape[2]
    rows = np.concatenate([g["cls"], g["reg"]], 1).transpose(0, 2, 1).reshape(B * T, -1)
    mean = DATASET_INFO[cfg.DATA.DATASET_NAME].MEAN_SIZE_ARRAY
    o = D.decode(rows, B, T, NH, NS, data["center_ref2"], mean)
    hl, sl = D.check(o, g["out0"], g["out1"], g["out2"], g["out3"], g["out4"], g["out5"], what=name)
    assert np.array_equal(hl, g["out4"].reshape(B * T, NH).argmax(1))
    # the fixture's heading is the float32 decode of its own label, not the float64 one
    a64 = hl * (2 * np.pi / NH) + o.hr[np.arange(B * T), hl].astype(np.float64) * (np.pi / NH)
    assert not np.array_equal(np.where(a64 > np.pi, a64 - 2 * np.pi, a64).astype(np.float32), g["out2"].reshape(-1))


# ------------------------------------------------------------------ torch's softmax / argmax on the crafted rows
def torch_decode(rows, B, T, NH, NS, center_ref, mean_size):
    """The model's eval-branch decode in torch float32 operations (softmax, argmax, gather, python-double
    constants), as the original code runs it on the CPU."""
    x = torch.from_numpy(np.asarray(rows, np.float32))
    R = B * T
    hs, hr = x[:, 5:5 + NH], x[:, 5 + NH:5 + 2 * NH]
    ss, sr = x[:, 5 + 2 * NH:5 + 2 * NH + NS], x[:, 5 + 2 * NH + NS:5 + 2 * NH + 4 * NS].reshape(R, NS, 3)
    cls = torch.softmax(x[:, 0:2], -1)
    hp, sp = torch.softmax(hs, -1), torch.softmax(ss, -1)
    hl, sl = torch.argmax(hp, -1), torch.argmax(sp, -1)
    r = torch.arange(R)
    bin_width = 2 * math.pi / NH
    ang = hl.to(torch.float32) * bin_width + hr[r, hl] * (bin_width / 2)
    ang = torch.where(ang > math.pi, ang - 2 * math.pi, ang)
    ex = torch.from_numpy(np.asarray(mean_size, np.float32))[sl]
    size = sr[r, sl] * ex + ex
    ctr = x[:, 2:5] + torch.from_numpy(np.asarray(center_ref, np.float32)).permute(0, 2, 1).reshape(R, 3)
    return [t.numpy() for t in (cls, ctr, ang, size, hp, sp)], hl.numpy(), sl.numpy()


@pytest.mark.parametrize("NS", NSS)
@pytest.mark.parametrize("NH", NHS)
def test_restatement_matches_torch_on_crafted_rows(NH, NS):
    rows, fam, B, T, cr, mean = _crafted_case(NH, NS)
    outs, thl, tsl = torch_decode(rows, B, T, NH, NS, cr, mean)
    o = D.decode(rows, B, T, NH, NS, cr, mean)
    hl, sl = D.check(o, *outs, what="torch NH=%d NS=%d" % (NH, NS))
    assert np.array_equal(hl, thl) and np.array_equal(sl, tsl)
    check_families(o, fam, outs, hl, sl, "torch NH=%d NS=%d" % (NH, NS))


def test_crafted_rows_see_contraction():
    """Every (NH, NS) case has rows whose heading and whose size change under a fused multiply-add (the heading only
    for NH > 1: with one bin the bin start is 0 and res * half + 0 rounds once either way)."""
    for NH in NHS:
        for NS in NSS:
            rows, fam, B, T, cr, mean = _crafted_case(NH, NS)
            o = D.decode(rows, B, T, NH, NS, cr, mean)
            hl = D.first_max(np.where(o.hL, o.hp[0], -1.0))
            sl = D.first_max(np.where(o.sL, o.sp[0], -1.0))
            h, s = D.contraction_sensitive(o, hl, sl)
            assert (h.sum() >= 4 or NH == 1) and s.sum() >= 4, (NH, NS, int(h.sum()), int(s.sum()))


# ------------------------------------------------------------------ csrc/decode.cuh on the host
def _host_cases():
    for NH in NHS:
        for NS in NSS:
            yield (NH, NS) + _crafted_case(NH, NS, seed=NH * 100 + NS)


def test_host_header_without_contraction_passes_every_case(host_lib):
    lib = host_lib["no_contraction"]
    for NH, NS, rows, fam, B, T, cr, mean in _host_cases():
        what = "NH=%d NS=%d" % (NH, NS)
        outs = host_decode(lib, rows, B, T, NH, NS, cr, mean)
        o = D.decode(rows, B, T, NH, NS, cr, mean)
        hl, sl = D.check(o, *outs, what="host " + what)
        check_families(o, fam, outs, hl, sl, "host " + what)
    from frustum_convnet_b200.config import DATASET_INFO
    for name in GOLDEN_CASES:
        g, data, sd, w, cfg = load_golden(name)
        B, _, T = g["cls"].shape
        NH, NS = cfg.DATA.NUM_HEADING_BIN, g["out5"].shape[2]
        rows = np.concatenate([g["cls"], g["reg"]], 1).transpose(0, 2, 1).reshape(B * T, -1)
        mean = DATASET_INFO[cfg.DATA.DATASET_NAME].MEAN_SIZE_ARRAY
        outs = host_decode(lib, rows, B, T, NH, NS, data["center_ref2"], mean)
        D.check(D.decode(rows, B, T, NH, NS, data["center_ref2"], mean), *outs, what="host " + name)


def test_host_header_with_contraction_fails_the_bit_exact_checks(host_lib):
    if "contracted" not in host_lib:
        pytest.skip("the host CPU has no FMA instructions")
    lib = host_lib["contracted"]
    bad_h = bad_s = 0
    for NH, NS, rows, fam, B, T, cr, mean in _host_cases():
        what = "NH=%d NS=%d" % (NH, NS)
        outs = host_decode(lib, rows, B, T, NH, NS, cr, mean)
        o = D.decode(rows, B, T, NH, NS, cr, mean)
        hl, sl = D.first_max(outs[4]), D.first_max(outs[5])
        bad_h += int((outs[2].view(np.int32) != D.heading_of(o, hl).view(np.int32)).sum())
        bad_s += int((outs[3].view(np.int32) != D.size_of(o, sl).view(np.int32)).any(1).sum())
        with pytest.raises(AssertionError, match="heading|size"):
            D.check(o, *outs, what="contracted " + what)
    print("\ncontracted host build: %d headings and %d sizes differ from the two-rounding decode" % (bad_h, bad_s))
    assert bad_h > 0 and bad_s > 0
