"""Persistent FCN kernel (csrc/fcn_mega.cu): its host tables, executed on the CPU.

A numpy "executor" walks the job table the way the kernel does - tiles of 128 flattened (frustum, position) rows x
NT columns, A operand = the segment boxes at row offset r0*stride + tap of the PADDED position-major maps (rows
outside the map read as zero, exactly the TMA out-of-bounds fill), packed weights, bias/ReLU, pixel-shuffled
store, per-tile completion counters - in a RANDOMISED dependency-respecting schedule (what dynamic job fetching
by many CTAs amounts to), and must reproduce the reference's golden FCN output / logits.  Checks the table
(topological order, dependency coverage, addressing) independently of the hardware mechanics."""
import numpy as np
import pytest
import torch

from frustum_convnet_b200 import mega
from frustum_convnet_b200.engine import FrustumEngine, _Plan


def _plan(golden_loader, name, nt256=False):
    g, data, sd, w, cfg = golden_loader(name)
    tsd = {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}
    eng = FrustumEngine(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, cfg.DATA.HEIGHT_HALF, 12, tsd, "cpu",
                        precision=1)
    eng.use_tma = False          # no driver here: tensor maps are not encoded, the tables do not need them
    eng.mega_nt256 = nt256
    B = data["point_cloud"].shape[0]
    T = [data["center_ref%d" % (i + 1)].shape[2] for i in range(w["arch"].num_scales)]
    return eng, _Plan(eng, B, data["point_cloud"].shape[2], tuple(T)), g


def _execute(eng, plan, feats, seed):
    descs = plan.mega_descs()
    map_keys, rows, jobs, nflags = mega.build_tables(descs)
    buf = {k: np.zeros(tuple(v.shape), dtype=np.float64) for k, v in plan.buf.items()}
    for i, f in enumerate(feats):                       # (B, T_i, C) valid rows of the padded feature maps
        buf["feat%d" % (i + 1)][:, :f.shape[1], :f.shape[2]] = f
    flat = {k: v.reshape(-1, v.shape[2]) for k, v in buf.items()}
    flags = np.zeros(nflags, dtype=np.int64)
    wts = [L.wt.double().numpy() for L in eng.layers]
    bias = [L.bias.double().numpy() for L in eng.layers]
    rng = np.random.default_rng(seed)
    pending = list(range(len(jobs)))
    fetched = 0
    inflight = []
    while fetched < len(jobs) or inflight:
        # "CTAs" fetch jobs strictly in table order, but complete them in any dependency-respecting order
        while fetched < len(jobs) and len(inflight) < 9:
            inflight.append(fetched)
            fetched += 1
        ready = [j for j in inflight if all((flags[f:f + c] >= t).all() for f, c, t in jobs[j]["deps"])]
        assert ready, "deadlock: no fetched job is runnable (table not topological?)"
        j = ready[int(rng.integers(len(ready)))]
        inflight.remove(j)
        jb = jobs[j]
        L, row = descs[jb["layer"]], rows[jb["layer"]]
        r0 = jb["m"] * mega.ROWS
        A = []
        for (src, c, tap, st), sg in zip(L.segs, row["segs"]):
            x = flat[src]
            a = np.zeros((mega.ROWS, sg["kblocks"] * 32))
            for i in range(mega.ROWS):
                rr = (r0 + i) * st + tap
                if 0 <= rr < x.shape[0]:
                    a[i, :min(x.shape[1], a.shape[1])] = x[rr, :a.shape[1]]
            A.append(a)
        A = np.concatenate(A, 1)
        W = wts[jb["layer"]]
        if A.shape[1] < W.shape[0]:
            A = np.concatenate([A, np.zeros((mega.ROWS, W.shape[0] - A.shape[1]))], 1)
        n0 = jb["n"] * L.NT
        D = A @ W[:, n0:n0 + L.NT] + bias[jb["layer"]][n0:n0 + L.NT]
        if L.relu:
            D = np.maximum(D, 0)
        out = buf[L.out]
        for i in range(mega.ROWS):
            r = r0 + i
            b, rt = divmod(r, L.P_m)
            if r >= L.n_rows or rt >= L.T_out:
                continue
            for c0 in range(0, L.NT, 32):
                n = n0 + c0
                if n >= L.up * L.Cout:
                    continue
                jj, co = divmod(n, L.Cout)
                tt = rt * L.up + jj
                if tt >= L.T_store:
                    continue
                out[b, tt, L.c_off + co: L.c_off + co + 32] = D[i, c0:c0 + 32]
        flags[row["flag_base"] + jb["m"]] += mega.EPI_WARPS
    for i, L in enumerate(descs):                       # every counter ends at its target
        assert (flags[rows[i]["flag_base"]: rows[i]["flag_base"] + L.m_tiles] == mega.EPI_WARPS * L.n_tiles).all()
    return buf, len(jobs), len(map_keys)


@pytest.mark.parametrize("name,seed,nt256", [("car_small_b3", 1, False), ("people_small_b2", 2, False),
                                             ("sunrgbd_full_b2", 3, False), ("car_small_b3", 4, True),
                                             ("sunrgbd_full_b2", 5, True)])
def test_job_table_execution_reproduces_reference_fcn(golden_loader, name, seed, nt256):
    eng, plan, g = _plan(golden_loader, name, nt256)
    if nt256:
        assert any(d.NT == 256 and d.k_atoms == 1 for d in plan.mega_descs())
    S = eng.arch.num_scales
    feats = [np.transpose(g["feat%d" % (i + 1)], (0, 2, 1)).astype(np.float64) for i in range(S)]
    buf, njobs, nmaps = _execute(eng, plan, feats, seed)
    T2 = plan.T[1]
    x = np.transpose(buf["cat"][:, :T2, :], (0, 2, 1))
    lg = buf["logits"][:, :T2, :]
    for mine, ref, what in ((x, g["x"], "x"), (np.transpose(lg[:, :, :2], (0, 2, 1)), g["cls"], "cls"),
                            (np.transpose(lg[:, :, 2:2 + eng.out_size], (0, 2, 1)), g["reg"], "reg")):
        err = np.abs(mine - ref).max()
        assert err <= 2e-3 * max(1.0, np.abs(ref).max()), (name, what, err)
    # pad rows between frustums stayed zero (the conv zero padding of the flattened row space relies on it)
    for k, v in buf.items():
        Tk = plan.valid_T.get(k)
        if Tk is not None and not k.startswith("feat"):
            assert not v[:, Tk:, :].any(), k


def test_full_size_car_table_shape():
    """B=32 car: 648 jobs, 17 load + 13 store tensor maps, interleaved side deconvs; heads tiles wait for all three deconvs."""
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload("car")
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in synth.make_state_dict(w["arch"], 3, "KITTI", seed=7).items()}
    eng = FrustumEngine(w["arch"], 3, "KITTI", cfg.DATA.HEIGHT_HALF, 12, sd, "cpu", precision=1)
    eng.use_tma = False
    plan = _Plan(eng, 32, 1024, (280, 140, 70, 35))
    descs = plan.mega_descs()
    map_keys, rows, jobs, nflags = mega.build_tables(descs)
    loads = [k for k in map_keys if k[0] == "load"]
    stores = [k for k in map_keys if k[0] == "store"]
    assert len(jobs) == 648 and len(loads) == 17 and len(stores) == 13 and nflags == sum(d.m_tiles for d in descs)
    names = [descs[j["layer"]].name for j in jobs]
    first_d2, last_a3 = names.index("block2_deconv"), len(names) - 1 - names[::-1].index("block3_conv1")
    assert first_d2 < last_a3 and names.index("block3_conv1") < len(names) - 1 - names[::-1].index("block2_deconv")
    heads = [j for j in jobs if descs[j["layer"]].name == "heads"]
    assert len(heads) == 36 and all(len(j["deps"]) == 3 for j in heads)
    assert all(j["deps"] == [] for j in jobs if descs[j["layer"]].name == "block1_conv1")


def test_wide_tile_rule_is_by_tile_count():
    """FCN_MEGA_NT256=auto: 256-wide tiles only when every main-chain layer keeps >= 24 tiles."""
    from frustum_convnet_b200 import config, synth
    cfg, w = config.load_workload("car")
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=7)
    tsd = {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}
    eng = FrustumEngine(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, cfg.DATA.HEIGHT_HALF, 12, tsd, "cpu", precision=1)
    eng.use_tma = False
    eng.mega_nt256 = "auto"
    small = _Plan(eng, 32, 1024, (280, 140, 70, 35)).mega_descs()
    big = _Plan(eng, 128, 1024, (280, 140, 70, 35)).mega_descs()
    assert max(d.NT for d in small) == 128 and max(d.NT for d in big) == 256
    for d in big:
        assert d.k_atoms == (1 if d.NT == 256 else 2) and d.K_pad % (32 * d.k_atoms) == 0


@pytest.mark.parametrize("wl,NH,one_tile", [("car", 12, True), ("car", 24, True), ("car", 1, True), ("car", 64, False),
                                           ("people", 64, False), ("sunrgbd", 24, True), ("sunrgbd", 48, False)])
def test_planner_runs_wide_heads_on_the_per_layer_path(wl, NH, one_tile, monkeypatch):
    """The persistent kernel's heads epilogue decodes whole rows, so it takes the heads layer as ONE N tile: a logit
    row of 192 columns (KITTI with 64 heading bins, SUN-RGBD with 48) makes three 64-column tiles, and the planner
    must build no persistent-kernel tables for it (the per-layer GEMMs and fcn_decode_eval run instead)."""
    from frustum_convnet_b200 import _lib, config, synth
    calls = []
    monkeypatch.setattr(_lib, "call", lambda name, *a: calls.append(name))   # tensor-map encodes need a driver
    monkeypatch.setenv("FCN_MEGA", "1")
    cfg, w = config.load_workload(wl)
    sd = synth.make_state_dict(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, seed=7, num_bins=NH)
    eng = FrustumEngine(w["arch"], w["num_vec"], cfg.DATA.DATASET_NAME, cfg.DATA.HEIGHT_HALF, NH,
                        {k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, "cpu", precision=1)
    assert eng.use_mega and eng.use_tma
    T = (280, 140, 70, 35) if w["arch"].num_scales == 4 else (280, 140, 70, 35, 18)
    plan = _Plan(eng, 32, 1024, T)
    heads = [d for d in plan.mega_descs() if d.kind == "heads"]
    assert len(heads) == 1 and (eng.ld_logit == 192) == (not one_tile)
    assert heads[0].n_tiles == (1 if one_tile else 3)
    assert plan.heads_one_tile() == one_tile
    assert (plan.mega_args is not None) == one_tile
    assert ("fcn_encode_store_map" in calls) == one_tile        # only the persistent kernel's tables encode stores
