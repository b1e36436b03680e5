"""GPU: the eval decode (csrc/decode.cuh ``decode_row``) against its float32 restatement (tests/decode_ref.py), in
both places it runs - the stand-alone ``fcn_decode_eval`` and the heads epilogue of the persistent FCN kernel -
and the layout helpers ``fcn_bct_to_btc`` / ``fcn_btc_to_bct`` against ``permute``, bit for bit.

Probabilities are checked within the bound derived in decode_ref.py, the labels must lie in its label sets, and
the centre, heading and size must be the bit-exact float32 decode of the label the kernel's own probabilities
name.  The crafted rows (decode_ref.crafted_rows) put exact and float32-probability ties, 1-ulp near ties,
saturated and -inf scores, non-finite rows, the heading wrap (last bin, residual exactly at f32(pi) and one float
above), large residuals and the exact-zero size in front of the arg-maxes and the decode, and include rows whose
heading and size change under a fused multiply-add."""
import numpy as np
import pytest
import torch

import decode_ref as D
from test_decode_ref_cpu import _mean_size, check_families

pytestmark = pytest.mark.gpu

NHS = (1, 2, 12, 24, 64)
NSS = (1, 3, 10, 64)
SHAPES = ((1, 1), (1, 127), (2, 64), (3, 43), (31, 129))      # B*T = 1, 127, 128, 129, 3999
SENTINEL = -12345.0
GUARD = 96


def _dev():
    return torch.device("cuda:0")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _outputs(R, NH, NS):
    """Six output views into ONE sentinel-filled block with a guard tail behind the last."""
    widths = (2, 3, 1, 3, NH, NS)
    block = torch.full((R * sum(widths) + GUARD,), SENTINEL, dtype=torch.float32, device=_dev())
    outs, off = [], 0
    for wd in widths:
        outs.append(block[off:off + R * wd])
        off += R * wd
    return block, outs


def _decode_eval(B, T, pitch, ld, NH, NS, lg, cr, ms, outs):
    from frustum_convnet_b200 import _lib
    _lib.call("fcn_decode_eval", B, T, pitch, ld, NH, NS, lg.data_ptr() if lg is not None else None,
              cr.data_ptr(), ms.data_ptr(), *[o.data_ptr() for o in outs], _stream())


def _rows_for(NH, NS, R, seed, mean):
    """The crafted rows first (when they fit), then random rows; returns (rows (R, W), families or None)."""
    rows, fam = D.crafted_rows(NH, NS, seed=seed, n_random=0, mean_size=mean)
    if R < len(rows):
        return D.crafted_rows(NH, NS, seed=seed + 1, n_random=R, mean_size=mean)[0][-R:], None
    extra = D.crafted_rows(NH, NS, seed=seed + 2, n_random=R - len(rows), mean_size=mean)[0][len(rows):]
    return np.concatenate([rows, extra]), fam


@pytest.mark.parametrize("NS", NSS)
@pytest.mark.parametrize("NH", NHS)
def test_decode_eval_matches_restatement(NH, NS):
    mean = _mean_size(NS, seed=NS)
    ms = torch.from_numpy(mean).to(_dev())
    W = D.row_width(NH, NS)
    seen_h = seen_s = 0
    for k, (B, T) in enumerate(SHAPES):
        R = B * T
        rows, fam = _rows_for(NH, NS, R, seed=1000 * NH + 10 * NS + k, mean=mean)
        # pad rows (t >= T) and pad columns (>= W) hold NaN: the kernel must not read them
        pitch = T + (0, 3, 1, 5, 2)[k]
        ld = W + (0, 1, 7, 3, 64)[k]
        lg = np.full((B, pitch, ld), np.nan, np.float32)
        lg[:, :T, :W] = rows.reshape(B, T, W)
        cr = np.random.default_rng(k).normal(0, 20, (B, 3, T)).astype(np.float32)
        block, outs = _outputs(R, NH, NS)
        _decode_eval(B, T, pitch, ld, NH, NS, torch.from_numpy(lg).to(_dev()), torch.from_numpy(cr).to(_dev()), ms, outs)
        torch.cuda.synchronize()
        got = [o.cpu().numpy() for o in outs]
        assert (block[-GUARD:] == SENTINEL).all(), "guard tail overwritten"
        what = "NH=%d NS=%d B=%d T=%d" % (NH, NS, B, T)
        o = D.decode(rows, B, T, NH, NS, cr, mean)
        hl, sl = D.check(o, *got, what=what)
        if fam is not None:
            check_families(o, fam, got, hl, sl, what)
        h, s = D.contraction_sensitive(o, hl, sl)
        seen_h += int(h.sum())
        seen_s += int(s.sum())
    # a contracted heading / size decode would have changed rows of these cases
    assert (seen_h > 0 or NH == 1) and seen_s > 0, (seen_h, seen_s)


def test_decode_eval_refusals_and_empty_launch():
    NH, NS = 12, 3
    W = D.row_width(NH, NS)
    B, T = 2, 5
    lg = torch.zeros((B, T, W + 1), dtype=torch.float32, device=_dev())
    cr = torch.zeros((B, 3, T), dtype=torch.float32, device=_dev())
    ms = torch.ones((64, 3), dtype=torch.float32, device=_dev())
    block, outs = _outputs(B * T * 10, 64, 64)
    bad = [(B, T, T, W, 0, NS), (B, T, T, W, 65, NS), (B, T, T, W, NH, 0), (B, T, T, D.row_width(NH, 65), NH, 65),
           (B, T, T, W - 1, NH, NS), (B, T, T - 1, W, NH, NS), (-1, T, T, W, NH, NS)]
    for args in bad:
        with pytest.raises(RuntimeError):
            _decode_eval(*args[:4], args[4], args[5], lg, cr, ms, outs)
    # B*T = 0: nothing is launched and nothing written (even with a NULL logit pointer)
    _decode_eval(0, T, T, W, NH, NS, None, cr, ms, outs)
    _decode_eval(B, 0, 0, W, NH, NS, None, cr, ms, outs)
    torch.cuda.synchronize()
    assert (block == SENTINEL).all()


# ------------------------------------------------------------------ layout helpers
def _btc(B, C, T, pitch, ld, src, dst):
    from frustum_convnet_b200 import _lib
    _lib.call("fcn_bct_to_btc", B, C, T, pitch, ld, src.data_ptr(), dst.data_ptr(), _stream())


def _bct(B, C, T, pitch, ld, src, dst):
    from frustum_convnet_b200 import _lib
    _lib.call("fcn_btc_to_bct", B, C, T, pitch, ld, src.data_ptr(), dst.data_ptr(), _stream())


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("C", [1, 31, 32, 33, 65, 300])
def test_layout_helpers_bit_exact(C):
    rng = np.random.default_rng(C)
    for T in (1, 31, 32, 33, 65, 300):
        for ld in (C, C + 1, (C + 31) // 32 * 32 + 32):
            for pitch in (T, T + 1, T + 40):
                for B in (1, 3):
                    x = rng.normal(0, 1, (B, C, T)).astype(np.float32)
                    x.reshape(-1)[::7] = -0.0                          # sign bits and NaN payloads travel as bits
                    x.reshape(-1)[3::11] = np.nan
                    src = torch.from_numpy(x).to(_dev())
                    n = B * pitch * ld
                    dst_block = torch.full((n + GUARD,), SENTINEL, dtype=torch.float32, device=_dev())
                    dst = dst_block[:n].view(B, pitch, ld)
                    _btc(B, C, T, pitch, ld, src, dst)
                    what = (B, C, T, pitch, ld)
                    assert torch.equal(_bits(dst[:, :T, :C]), _bits(src.permute(0, 2, 1))), what
                    assert (dst[:, :T, C:] == 0).all() and not torch.signbit(dst[:, :T, C:]).any(), what
                    assert (dst[:, T:, :] == SENTINEL).all() and (dst_block[n:] == SENTINEL).all(), what
                    # position-major with NaN in the pad rows and columns -> channel-first
                    y = torch.full((B, pitch, ld), float("nan"), dtype=torch.float32, device=_dev())
                    y[:, :T, :C] = torch.from_numpy(rng.normal(0, 1, (B, T, C)).astype(np.float32)).to(_dev())
                    back_block = torch.full((B * C * T + GUARD,), SENTINEL, dtype=torch.float32, device=_dev())
                    back = back_block[:B * C * T].view(B, C, T)
                    _bct(B, C, T, pitch, ld, y, back)
                    assert torch.equal(_bits(back), _bits(y[:, :T, :C].permute(0, 2, 1))), what
                    assert (back_block[B * C * T:] == SENTINEL).all(), what
                    # round trip is the identity
                    rt = torch.empty_like(src)
                    _bct(B, C, T, pitch, ld, dst, rt)
                    assert torch.equal(_bits(rt), _bits(src)), what


def test_layout_helpers_refusals():
    buf = torch.zeros(4096, dtype=torch.float32, device=_dev())
    for fn in (_btc, _bct):
        for args in ((1, 0, 4, 4, 4), (1, 4, 0, 4, 4), (1, 4, 4, 4, 3), (1, 4, 4, 3, 4), (-1, 4, 4, 4, 4)):
            with pytest.raises(RuntimeError):
                fn(*args, buf, buf)
        fn(0, 4, 4, 4, 4, buf, buf)                                    # B = 0: nothing to do
    torch.cuda.synchronize()
    assert not buf.any()


# ------------------------------------------------------------------ both engine eval paths
WORKLOADS = {"car": (32, 64), "people": (32, 64), "sunrgbd": (32, 48)}    # benchmarked B, a NH with ld_logit = 192


def _engine(monkeypatch, wl, NH, mega, sd=None, seed=7):
    from frustum_convnet_b200 import config, synth
    from frustum_convnet_b200.engine import FrustumEngine
    monkeypatch.setenv("FCN_MEGA", "1" if mega else "0")
    cfg, w = config.load_workload(wl)
    if sd is None:
        sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=seed, num_bins=NH)
    tsd = {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}
    return FrustumEngine(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, cfg.DATA.HEIGHT_HALF, NH, tsd, _dev(),
                         precision=1), cfg, w


def _run(eng, w, data):
    S = w["arch"].num_scales
    d = {k: torch.from_numpy(v).to(_dev()) for k, v in data.items()}
    centers = [d["center_ref%d" % (i + 1)] for i in range(S)]
    out = [o.clone() for o in eng.forward(d["point_cloud"], centers, d.get("one_hot"))]
    plan = eng.plan(d["point_cloud"].shape[0], d["point_cloud"].shape[2], [c.shape[2] for c in centers])
    torch.cuda.synchronize()
    cls, reg = plan.logits()
    rows = torch.cat([cls, reg], 1).cpu().numpy()
    return plan, [o.cpu().numpy() for o in out], rows


def _check_plan(plan, eng, data, out, rows, what):
    B, T2 = plan.B, plan.T[1]
    o = D.decode(rows, B, T2, eng.num_bins, eng.num_size, data["center_ref2"], eng.mean_size.cpu().numpy())
    return D.check(o, *out, what=what), o


@pytest.mark.parametrize("wl", list(WORKLOADS))
def test_engine_eval_paths_match_restatement(wl, monkeypatch):
    """Both eval paths decode the plan's own logits as the restatement does, at the benchmarked B, for the default
    12 heading bins, 1, 24 and a bin count whose logit row needs 192 columns (three 64-column heads tiles: the
    persistent kernel refuses it and the planner runs the per-layer path)."""
    from frustum_convnet_b200 import synth
    B, nh192 = WORKLOADS[wl]
    data = synth.make_frustums(wl, B, seed=41)
    for NH in (12, 1, 24, nh192):
        res = {}
        for mega in (True, False):
            eng, cfg, w = _engine(monkeypatch, wl, NH, mega, seed=13 + NH)
            assert (eng.ld_logit == 192) == (NH == nh192)
            plan, out, rows = _run(eng, w, data)
            assert (plan.mega_args is not None) == (mega and eng.ld_logit <= 128), (wl, NH, mega)
            _check_plan(plan, eng, data, out, rows, "%s NH=%d mega=%d" % (wl, NH, mega))
            res[mega] = (out, rows)
        assert np.array_equal(res[True][1], res[False][1]), (wl, NH)
        for a, b in zip(res[True][0], res[False][0]):
            assert np.array_equal(a.view(np.int32), b.view(np.int32)), (wl, NH)
        if NH == nh192:
            # the persistent kernel itself refuses a heads layer of more than one N tile
            plan._build_mega()
            assert plan.mega_args is not None and any(d.kind == "heads" and d.n_tiles == 3 for d in plan.mega_descs())
            with pytest.raises(RuntimeError, match="single N tile"):
                plan._launch_mega(plan.in_centers[1])


CRAFTED_HEADS = ("tie_first", "prob_tie", "wrap_last_bin", "at_pi", "above_pi", "negative", "large_res", "size_zero",
                 "fma_sensitive", "neg_inf", "cls_exact")


@pytest.mark.parametrize("wl,NH", [("car", 12), ("sunrgbd", 24)])
def test_engine_crafted_heads(wl, NH, monkeypatch):
    """Zero head weights and a crafted bias: every logit row of the plan IS the crafted row, so the ties, the wrap
    and exactly-pi reach the persistent kernel's heads epilogue (and the per-layer path) through the GEMM."""
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload(wl)
    NS = config.DATASET_INFO[cfg.DATA.DATASET_NAME].NUM_SIZE_CLUSTER
    mean = config.DATASET_INFO[cfg.DATA.DATASET_NAME].MEAN_SIZE_ARRAY.astype(np.float32)
    crafted, fam = D.crafted_rows(NH, NS, seed=5, n_random=0, mean_size=mean)
    pick = sorted({int(i) for name in CRAFTED_HEADS for i in fam[name][0]})
    data = synth.make_frustums(wl, 3, seed=43)
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=19, num_bins=NH)
    sd = {k: np.array(v) for k, v in sd.items()}
    sd["cls_out.weight"][:] = 0
    sd["reg_out.weight"][:] = 0
    engines = {mega: _engine(monkeypatch, wl, NH, mega, sd=sd)[0] for mega in (True, False)}
    for i in pick:
        sd["cls_out.bias"][:] = crafted[i, 0:2]
        sd["reg_out.bias"][:] = crafted[i, 2:]
        for mega, eng in engines.items():
            eng.pack({k: torch.from_numpy(v) for k, v in sd.items()})
            plan, out, rows = _run(eng, w, data)
            assert (plan.mega_args is not None) == mega
            assert (rows.view(np.int32) == crafted[i].view(np.int32)).all(), "logits are not the crafted row"
            (hl, sl), o = _check_plan(plan, eng, data, out, rows, "%s NH=%d row %d mega=%d" % (wl, NH, i, mega))
            for name, v in fam.items():
                if name != "cls_want" and i in v[0]:
                    j = list(v[0]).index(i)
                    assert v[1][j] is None or (hl == v[1][j]).all(), (name, i, mega)
                    assert v[2][j] is None or (sl == v[2][j]).all(), (name, i, mega)
            heading = out[2].reshape(-1)
            if i in fam["at_pi"][0]:
                assert (heading == D.PI32).all()
            if i in fam["above_pi"][0]:
                assert (heading < 0).all()
            if i in fam["cls_exact"][0]:
                want = fam["cls_want"][list(fam["cls_exact"][0]).index(i)]
                assert (out[0].reshape(-1, 2) == want).all()
