"""The ConvFeatNet + heads graph of ``config.fcn_layers`` against the drop-in ``nn.Module``s, on the CPU.

The eval weight pack, the persistent kernel's tables, the training layer table and the seeded state dicts are all
built from ``fcn_layers``; the modules of det_base.py / det_base_sunrgbd.py are the independent statement of the
same network (they fix the state-dict names and shapes a checkpoint must have)."""
import pytest
import torch.nn as nn

from frustum_convnet_b200 import config


@pytest.mark.parametrize("wl,module", [("car", "det_base"), ("sunrgbd", "det_base_sunrgbd")])
def test_fcn_layer_table_matches_the_modules(wl, module):
    import importlib
    cfg, w = config.load_workload(wl)
    mod = importlib.import_module("frustum_convnet_b200." + module)
    V = w["num_vec"]
    model = mod.PointNetDet(3, num_vec=V)
    arch = model.ARCH
    layers = config.fcn_layers(arch, V)
    children = dict(model.conv_net.named_children())
    body = [L for L in layers if L.kind != "heads"]
    assert [L.kind for L in layers].count("heads") == 1 and layers[-1].kind == "heads"
    # every conv_net child once, nothing else (SUN-RGBD registers its deconvs in reverse order: compare sets)
    assert len({L.name for L in body}) == len(body) and {L.name for L in body} == set(children)
    produced = {"feat%d" % (s + 1) for s in range(arch.num_scales)}
    for L in body:
        blk = children[L.name][0]
        ci = sum(c for _, c in L.srcs)
        assert all(src in produced for src, _ in L.srcs), L.name          # sources come before their consumers
        produced.add(L.name)
        if L.kind == "deconv":
            assert isinstance(blk, nn.ConvTranspose1d), L.name
            assert tuple(blk.weight.shape) == (ci, L.Cout, L.k) and blk.padding == (0,), L.name
        else:
            assert isinstance(blk, nn.Conv1d) and L.kind in ("conv", "merge"), L.name
            assert tuple(blk.weight.shape) == (L.Cout, ci, L.k) and blk.padding == (L.k // 2,), L.name
        assert blk.kernel_size == (L.k,) and blk.stride == (L.stride,), L.name
        assert children[L.name][1].num_features == L.Cout, L.name
        if L.kind == "merge":
            c3 = getattr(model.feat_net, "pointnet%d" % (L.level + 1)).conv3[0].weight.shape[0]
            assert L.srcs[1] == ("feat%d" % (L.level + 1), c3 + V), L.name
    # heads: the transposed convs in concat order, each at the column offset where the previous one ends
    heads = layers[-1]
    deconvs = {L.name: L for L in body if L.kind == "deconv"}
    assert [src for src, _ in heads.srcs] == sorted(deconvs, key=lambda n: deconvs[n].c_off)
    off = 0
    for src, c in heads.srcs:
        assert deconvs[src].c_off == off and deconvs[src].Cout == c == arch.deconv_out
        off += c
    assert off == arch.reg_in == model.reg_out.weight.shape[1] == model.cls_out.weight.shape[1]
