"""CPU: the float64 training-layer reference (tests/train_ref.py) against PyTorch modules with autograd in
float64 (outputs, every parameter gradient, input gradients, running statistics: 1e-12 relative), the restated
Adam against torch.optim.Adam, and the argument validation of the five training entry points, which all check
their arguments before any CUDA call."""
import ctypes as C

import pytest
import torch

import train_ref as tr

F64 = torch.float64
REL = 1e-12


def _close(got, exp, what):
    got, exp = got.double(), exp.double()
    err = float((got - exp).abs().max()) if got.numel() else 0.0
    assert err <= REL * max(1.0, float(exp.abs().max())), (what, err)


def _pm(t):
    """(B, C, T) -> position-major (B*T, C)."""
    return t.permute(0, 2, 1).reshape(-1, t.shape[1])


def _bn(c, g):
    bn = torch.nn.BatchNorm1d(c, eps=tr.EPS).double()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g, dtype=F64) + 0.5)
        bn.bias.copy_(torch.rand(c, generator=g, dtype=F64) - 0.5)
        bn.running_mean.copy_(torch.randn(c, generator=g, dtype=F64))
        bn.running_var.copy_(torch.rand(c, generator=g, dtype=F64) + 0.5)
    bn.initial = (bn.running_mean.clone(), bn.running_var.clone())     # the forward updates the buffers
    return bn


def _set_bn(case, bn):
    case.gamma.copy_(bn.weight.detach())
    case.beta.copy_(bn.bias.detach())
    case.run_mean.copy_(bn.initial[0])
    case.run_var.copy_(bn.initial[1])


def _as_bn_source(case, i, producer):
    """Source i of `case` is the raw output of `producer` (a BN layer case)."""
    b = case.src[i]
    b["raw"].copy_(producer.Y)
    b["sums"].copy_(producer.sums)
    b["gamma"].copy_(producer.gamma)
    b["beta"].copy_(producer.beta)


def _run_forward(case):
    L = case.layer()
    Y, _ = tr.forward_ref(L, case.mem)
    case.Y.copy_(Y)
    if case.d.has_bn:
        case.sums.copy_(tr.stats_ref(L, Y)[0])
    return L


def _run_backward(case, L, grads=True):
    """dsums, dW, dgamma / dbeta / dbias and the dX of every segment into the source gradients (accumulated)."""
    ds, _, _ = tr.reduce_ref(L, case.mem)
    case.dsums[:ds.numel()].copy_(ds)
    dy = tr.dy_ref(L, case.mem)                 # the BN backward reads the reduction (Sum dz, Sum dz*xh)
    for j in range(L.n_seg):
        widx, v, _, _ = tr.dw_ref(L, j, case.mem, dy)
        case.dW.index_add_(0, widx.reshape(-1), v.reshape(-1))
        src = case.src[case.d.segs[j].src]
        if grads and src["grad"] is not None:
            idx, v, _, _ = tr.dx_ref(L, j, case.mem, dy)
            src["grad"].view(-1).index_add_(0, idx.reshape(-1), v.reshape(-1))
    if case.d.has_bn:
        case.dbeta += ds[:case.d.Cout]
        case.dgamma += ds[case.d.Cout:]
    elif case.dbias is not None:
        case.dbias += ds


def _running(case):
    return tr.finalize_running_ref(case.sums, tr.bn_count(case.layer()), case.run_mean, case.run_var, case.d.Cout)


@pytest.mark.parametrize("k,stride,T", [(3, 1, 9), (3, 1, 10), (3, 2, 9), (3, 2, 10), (1, 1, 7)])
def test_conv_bn_relu_chain_matches_autograd(k, stride, T):
    """x -> Conv1d(1x1) -> BN -> ReLU -> Conv1d(k, stride, pad k//2) -> BN -> ReLU: the second layer reads the
    first one's RAW output through its statistics (a BN source), so the source-side activation and its backward
    (gradient w.r.t. the post-activation values) are covered as well."""
    g = torch.Generator().manual_seed(100 * k + 10 * stride + T)
    B, ci, c1, c2 = 3, 5, 6, 7
    x = torch.randn(B, ci, T, generator=g, dtype=F64, requires_grad=True)
    conv_a = torch.nn.Conv1d(ci, c1, 1, bias=False).double()
    conv_b = torch.nn.Conv1d(c1, c2, k, stride=stride, padding=k // 2, bias=False).double()
    bn_a, bn_b = _bn(c1, g), _bn(c2, g)
    h = torch.relu(bn_a(conv_a(x)))
    h.retain_grad()
    out = torch.relu(bn_b(conv_b(h)))
    G = torch.randn(out.shape, generator=g, dtype=F64)
    (out * G).sum().backward()

    da = tr.conv1d_layer(B, T, [tr.SrcDesc(T, ci)], ci, c1, 1, has_bn=1, relu=1)
    ca = tr.LayerCase(da, "cpu", F64)
    ca.src[0]["raw"].copy_(_pm(x.detach()))
    ca.W.copy_(conv_a.weight.detach().reshape(-1))
    _set_bn(ca, bn_a)
    La = _run_forward(ca)
    _close(ca.Y, _pm(conv_a(x).detach()), "Y_a")

    db = tr.conv1d_layer(B, T, [tr.SrcDesc(T, c1, stats=True, Cstat=c1)], c1, c2, k, stride=stride, has_bn=1, relu=1)
    assert db.T_out == out.shape[2]
    cb = tr.LayerCase(db, "cpu", F64)
    _as_bn_source(cb, 0, ca)
    cb.W.copy_(conv_b.weight.detach().reshape(-1))
    _set_bn(cb, bn_b)
    Lb = _run_forward(cb)
    _close(cb.Y, _pm(conv_b(h).detach()), "Y_b")

    cb.dA.copy_(_pm(G))
    _run_backward(cb, Lb)
    _close(cb.dW.view_as(conv_b.weight), conv_b.weight.grad, "dW_b")
    _close(cb.dgamma, bn_b.weight.grad, "dgamma_b")
    _close(cb.dbeta, bn_b.bias.grad, "dbeta_b")
    _close(cb.src[0]["grad"], _pm(h.grad), "dX_b (gradient of the post-activation source)")
    ca.dA.copy_(cb.src[0]["grad"])
    _run_backward(ca, La)
    _close(ca.dW.view_as(conv_a.weight), conv_a.weight.grad, "dW_a")
    _close(ca.dgamma, bn_a.weight.grad, "dgamma_a")
    _close(ca.dbeta, bn_a.bias.grad, "dbeta_a")
    _close(ca.src[0]["grad"], _pm(x.grad), "dX_a")
    for case, bn in ((ca, bn_a), (cb, bn_b)):
        rm, rv = _running(case)
        _close(rm, bn.running_mean, "running_mean")
        _close(rv, bn.running_var, "running_var")


@pytest.mark.parametrize("k", [2, 4, 8])
def test_transposed_conv_crop_and_concat_head_match_autograd(k):
    """ConvTranspose1d(kernel = stride = k) -> BN -> ReLU -> crop to T2, concatenated with a plain source, -> 1x1
    head with bias: the pixel shuffle (N = k*Cout columns folded onto Cout BN channels over B*T*k samples), the
    crop (T2 < T*k), two segments and the plain-layer bias."""
    g = torch.Generator().manual_seed(7 + k)
    B, T, ci, co, c2, n = 2, 5, 6, 4, 3, 5
    T2 = T * k - 3
    x = torch.randn(B, ci, T, generator=g, dtype=F64, requires_grad=True)
    x2 = torch.randn(B, c2, T2, generator=g, dtype=F64, requires_grad=True)
    dec = torch.nn.ConvTranspose1d(ci, co, k, stride=k, bias=False).double()
    bn = _bn(co, g)
    head = torch.nn.Conv1d(co + c2, n, 1).double()
    h = torch.relu(bn(dec(x)))
    h.retain_grad()
    out = head(torch.cat([h[:, :, :T2], x2], 1))
    G = torch.randn(out.shape, generator=g, dtype=F64)
    (out * G).sum().backward()

    dd = tr.deconv_layer(B, T, [tr.SrcDesc(T, ci)], ci, co, k, has_bn=1, relu=1)
    cd = tr.LayerCase(dd, "cpu", F64)
    cd.src[0]["raw"].copy_(_pm(x.detach()))
    cd.W.copy_(dec.weight.detach().reshape(-1))
    _set_bn(cd, bn)
    Ld = _run_forward(cd)
    _close(cd.Y.view(B, T, k, co).reshape(B, T * k, co), dec(x).detach().permute(0, 2, 1), "Y (un-shuffled)")

    srcs = [tr.SrcDesc(T, k * co, up=k, cup=co, stats=True, Cstat=co), tr.SrcDesc(T2, c2)]
    dh = tr.concat_layer(B, T2, srcs, [co, c2], n, bias=True)
    ch = tr.LayerCase(dh, "cpu", F64)
    _as_bn_source(ch, 0, cd)
    ch.src[1]["raw"].copy_(_pm(x2.detach()))
    ch.W.copy_(head.weight.detach().reshape(-1))
    ch.bias.copy_(head.bias.detach())
    Lh = _run_forward(ch)
    _close(ch.Y, _pm(out.detach()), "head output")
    ch.dA.copy_(_pm(G))
    _run_backward(ch, Lh)
    _close(ch.dW.view_as(head.weight), head.weight.grad, "dW head")
    _close(ch.dbias, head.bias.grad, "dbias head")
    _close(ch.src[1]["grad"], _pm(x2.grad), "dX plain source")
    hg = h.grad.permute(0, 2, 1).reshape(B, T, k * co)       # gradient of the post-activation, un-shuffled
    _close(ch.src[0]["grad"].view(B, T, k * co), hg, "dX through the crop and the pixel shuffle")
    cd.dA.copy_(ch.src[0]["grad"])
    _run_backward(cd, Ld)
    _close(cd.dW.view_as(dec.weight), dec.weight.grad, "dW transposed conv")
    _close(cd.dgamma, bn.weight.grad, "dgamma")
    _close(cd.dbeta, bn.bias.grad, "dbeta")
    _close(cd.src[0]["grad"], _pm(x.grad), "dX_a")
    rm, rv = _running(cd)
    _close(rm, bn.running_mean, "running_mean")
    _close(rv, bn.running_var, "running_var")


@pytest.mark.parametrize("V", [0, 3])
def test_pool_mask_max_and_one_hot_match_autograd(V):
    """Conv2d(1x1) -> BatchNorm2d -> ReLU -> x * (cnt > 0) -> max over K, one-hot columns appended
    (det_base.py:100-101,134-157): pooled features, the argmax scatter of the backward and the layer's
    gradients; rows with cnt = 0 are zero and get no gradient."""
    from frustum_convnet_b200 import _lib
    g = torch.Generator().manual_seed(40 + V)
    B, T, K, ci, Cc = 2, 3, 5, 4, 6
    x = torch.randn(B, ci, T, K, generator=g, dtype=F64, requires_grad=True)
    conv = torch.nn.Conv2d(ci, Cc, 1, bias=False).double()
    bn2 = torch.nn.BatchNorm2d(Cc, eps=tr.EPS).double()
    b1 = _bn(Cc, g)
    with torch.no_grad():
        for a in ("weight", "bias", "running_mean", "running_var"):
            getattr(bn2, a).copy_(getattr(b1, a))
    cnt = torch.tensor([[3, 0, 5], [1, 2, 0]], dtype=torch.int32)
    one_hot = torch.randn(B, max(V, 1), generator=g, dtype=F64)[:, :V]
    z = torch.relu(bn2(conv(x)))
    z.retain_grad()
    zm = z * (cnt > 0).double()[:, None, :, None]
    feat = torch.cat([zm.max(3).values, one_hot[:, :, None].expand(B, V, T)], 1)     # (B, C+V, T)
    G = torch.randn(feat.shape, generator=g, dtype=F64)
    (feat * G).sum().backward()

    rows = x.detach().permute(0, 2, 3, 1).reshape(B * T * K, ci)
    d = tr.conv1d_layer(B, T * K, [tr.SrcDesc(T * K, ci, grad=False)], ci, Cc, 1, has_bn=1, relu=1)
    case = tr.LayerCase(d, "cpu", F64)
    case.src[0]["raw"].copy_(rows)
    case.W.copy_(conv.weight.detach().reshape(-1))
    _set_bn(case, b1)
    L = _run_forward(case)
    featbuf = torch.zeros(B * T, Cc + V, dtype=F64)
    dfeat = G.permute(0, 2, 1).reshape(B * T, Cc + V).contiguous()
    argmax = torch.zeros(B * T, Cc, dtype=torch.int32)
    oh = one_hot.contiguous()
    cnt_f = cnt.reshape(-1).contiguous()
    mem = case.mem
    for t in (featbuf, dfeat, argmax, oh, cnt_f):
        mem.add(t)
    P = _lib.TrainPool()
    P.B, P.T, P.K, P.C, P.V, P.ld_feat = B, T, K, Cc, V, Cc + V
    P.Y, P.cnt, P.sums, P.gamma, P.beta = case.Y.data_ptr(), cnt_f.data_ptr(), case.sums.data_ptr(), \
        case.gamma.data_ptr(), case.beta.data_ptr()
    P.one_hot, P.feat, P.argmax = oh.data_ptr() if V else None, featbuf.data_ptr(), argmax.data_ptr()
    P.dfeat, P.dA = dfeat.data_ptr(), case.dA.data_ptr()
    pooled, _, _, zref = tr.pool_ref(P, mem)
    _close(pooled, _pm(feat.detach()[:, :Cc]), "pooled features")
    am = zref.argmax(1).int()
    case.dA.copy_(tr.pool_bwd_ref(P, mem, am))
    _close(case.dA, z.grad.permute(0, 2, 3, 1).reshape(-1, Cc), "pool backward (gradient of the post-activation)")
    _run_backward(case, L, grads=False)
    _close(case.dW.view_as(conv.weight), conv.weight.grad, "dW")
    _close(case.dgamma, bn2.weight.grad, "dgamma")
    _close(case.dbeta, bn2.bias.grad, "dbeta")
    rm, rv = _running(case)
    _close(rm, bn2.running_mean, "running_mean")
    _close(rv, bn2.running_var, "running_var")


def test_adam_restatement_matches_torch_adam_over_50_steps():
    """Hyper-parameters that are fp32 numbers (the kernel's rounding of them is then the identity)."""
    g = torch.Generator().manual_seed(3)
    n = 1000
    lr, b1, b2, eps, wd = 2.0 ** -10, 0.875, 1 - 2.0 ** -11, 2.0 ** -27, 2.0 ** -13
    p0 = torch.randn(n, generator=g, dtype=F64)
    pt = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([pt], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd)
    p, m, v = p0.clone(), torch.zeros(n, dtype=F64), torch.zeros(n, dtype=F64)
    for step in range(1, 51):
        grad = torch.randn(n, generator=g, dtype=F64)
        grad[:10] = 0.0
        pt.grad = grad.clone()
        opt.step()
        p, m, v, _ = tr.adam_ref(p, grad * 8.0, m, v, lr, b1, b2, eps, wd, step, 0.125)
        _close(p, pt.detach(), "param at step %d" % step)
    st = opt.state[pt]
    _close(m, st["exp_avg"], "exp_avg")
    _close(v, st["exp_avg_sq"], "exp_avg_sq")


# ============================================================================ argument validation (no GPU needed)
def _lib_handle():
    from frustum_convnet_b200 import _lib
    return _lib, _lib.load()


def _valid_layer():
    d = tr.concat_layer(2, 5, [tr.SrcDesc(5, 8, stats=True, Cstat=8)], [8], 4, has_bn=1, relu=1)
    case = tr.LayerCase(d, "cpu")
    return case, case.layer()


def _rejects(fn, L, what, *args):
    _lib, lib = _lib_handle()
    rc = getattr(lib, fn)(C.byref(L), *args)
    assert rc != 0, "%s accepted %s" % (fn, what)
    return lib.fcn_last_error().decode()


@pytest.mark.parametrize("bad", ["n_seg0", "n_seg5", "W", "Y", "bn_stats", "seg_raw", "seg_C", "seg_stride",
                                 "src_stats", "src_count", "shape"])
def test_train_forward_and_backward_reject_bad_layers(bad):
    case, L = _valid_layer()
    if bad == "n_seg0":
        L.n_seg = 0
    elif bad == "n_seg5":
        L.n_seg = 5
    elif bad == "W":
        L.W = None
    elif bad == "Y":
        L.Y = None
    elif bad == "bn_stats":
        L.sums = None
    elif bad == "seg_raw":
        L.seg[0].src.raw = None
    elif bad == "seg_C":
        L.seg[0].C = 0
    elif bad == "seg_stride":
        L.seg[0].stride = 0
    elif bad == "src_stats":
        L.seg[0].src.gamma = None
    elif bad == "src_count":
        L.seg[0].src.count = 0.0
    elif bad == "shape":
        L.T_out = 0
    msg = _rejects("fcn_train_forward", L, bad, None, 0, None)
    assert msg
    assert _rejects("fcn_train_backward", L, bad, 1, None) == msg


@pytest.mark.parametrize("missing", ["dA", "dW", "dsums"])
def test_train_backward_rejects_null_gradient_buffers(missing):
    case, L = _valid_layer()
    setattr(L, missing, None)
    assert "gradient" in _rejects("fcn_train_backward", L, missing, 1, None)


@pytest.mark.parametrize("backward,missing", [(0, "Y"), (0, "cnt"), (0, "argmax"), (0, "sums"), (0, "gamma"),
                                              (0, "beta"), (0, "feat"), (0, "one_hot"), (1, "dA"), (1, "dfeat"),
                                              (0, "shape")])
def test_train_pool_rejects_null_pointers(backward, missing):
    _lib, lib = _lib_handle()
    buf = torch.zeros(64)
    P = _lib.TrainPool()
    P.B, P.T, P.K, P.C, P.V, P.ld_feat = 1, 2, 3, 4, 2, 6
    for f in ("Y", "cnt", "sums", "gamma", "beta", "one_hot", "feat", "argmax", "dfeat", "dA"):
        setattr(P, f, buf.data_ptr())
    if missing == "shape":
        P.K = 0
    else:
        setattr(P, missing, None)
    assert lib.fcn_train_pool(C.byref(P), backward, None) != 0
    assert lib.fcn_last_error()


def test_train_finalize_and_adam_reject_bad_arguments():
    _lib, lib = _lib_handle()
    assert lib.fcn_train_finalize(None, 1, 1, None) != 0
    buf = torch.zeros(16)
    p = buf.data_ptr()
    assert lib.fcn_train_finalize(p, 0, 1, None) != 0
    assert lib.fcn_adam_step(p, p, p, p, 4, 1e-3, 0.9, 0.999, 1e-8, 0.0, 0, 1.0, None) != 0      # step 0
    assert lib.fcn_adam_step(None, p, p, p, 4, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None) != 0
    assert lib.fcn_adam_step(p, p, p, p, -1, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None) != 0
    assert lib.fcn_adam_step(p, p, p, p, 0, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 1.0, None) == 0      # no-op
    assert torch.equal(buf, torch.zeros(16))


def _expected_workspace(L):
    """slices * M * N of the launcher's K split (csrc/train.cu fwd_slices), 0 without a split."""
    cdiv = lambda a, b: -(-a // b)
    M = L.B * L.T_out
    tiles = sum(cdiv(L.seg[i].C, 16) for i in range(L.n_seg))
    want = min(cdiv(2 * 148, cdiv(M, 64) * cdiv(L.N, 64)), tiles // 2)
    if want < 2:
        return 0
    tps = cdiv(tiles, want)
    return cdiv(tiles, tps) * M * L.N


@pytest.mark.parametrize("B,T,Ci,N", [(4, 40, 768, 128), (32, 140, 64, 512), (1, 1, 16, 2), (2, 8, 40, 39),
                                      (2, 70, 1024, 512)])
def test_train_workspace_floats(B, T, Ci, N):
    _lib, lib = _lib_handle()
    d = tr.concat_layer(B, T, [tr.SrcDesc(T, Ci)], [Ci], N)
    L = tr.LayerCase(d, "cpu").layer()
    exp = _expected_workspace(L)
    assert lib.fcn_train_workspace_floats(C.byref(L)) == exp
    assert lib.fcn_train_workspace_floats(None) == 0
    if (B, T) == (32, 140):
        assert exp == 0                                     # enough CTAs: no split
    if (B, T, Ci) == (4, 40, 768):
        assert exp > 0 and exp % (B * T * N) == 0
