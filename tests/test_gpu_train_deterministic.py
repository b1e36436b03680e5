"""GPU: the deterministic training mode (fcn_train_forward_deterministic / fcn_train_backward_deterministic,
fcn_det_loss_deterministic, TrainStep(deterministic=...), PointNetDet.deterministic).

Bit-reproducibility is checked with torch.equal on the raw bits: per layer across streams and workspace contents,
for whole TrainSteps across fresh objects, allocator states and processes, and for the fused loss across calls and
streams.  Accuracy reuses the float64 bounds of test_gpu_train_layers.py and test_gpu_det_loss.py."""
import ctypes as C
import hashlib
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import loss_ref as lr
import train_ref as tr
from conftest import ROOT
from test_gpu_det_loss import Call, check
from test_gpu_train_layers import _assert_within, _engine_mem, _seg_K

pytestmark = pytest.mark.gpu


def _lib():
    from frustum_convnet_b200 import _lib
    return _lib


def _data(wl, B, seed):
    from frustum_convnet_b200 import synth
    d = synth.make_frustums(wl, B, seed=seed, with_labels=True, max_depth=(17.5 if wl == "car" else None))
    return {k: torch.from_numpy(v).cuda() for k, v in d.items()}


def _bits(t):
    return t.detach().reshape(-1).contiguous().view(torch.uint8).clone()


@pytest.fixture
def torch_deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


# ============================================================================ per layer
def _layer_run(eng, mem, li, stream, fill):
    """Zero the layer's accumulating outputs, fill the workspace, run its deterministic forward and backward on
    `stream`; -> the raw bits of Y, sums, dsums, the flat gradient bucket and every source gradient."""
    L = eng.layers[li]
    M = L.B * L.T_out
    lib = _lib()
    with torch.cuda.stream(stream):
        fill(eng.workspace)
        eng.flat.grad.zero_()
        if L.has_bn:
            mem.get(L.sums, 2 * L.Cout).zero_()
        dsums = mem.get(L.dsums, 2 * L.Cout if L.has_bn else L.N)
        dsums.zero_()
        grads = []
        for j in range(L.n_seg):
            s = L.seg[j].src
            if s.grad:
                g = mem.get(s.grad, L.B * s.T * s.ld)
                g.zero_()
                grads.append(g)
        st = stream.cuda_stream
        lib.call("fcn_train_forward_deterministic", C.byref(L), eng.workspace.data_ptr(), eng.workspace.numel(), st)
        fill(eng.workspace)
        lib.call("fcn_train_backward_deterministic", C.byref(L), eng.dx_mask[li], eng.workspace.data_ptr(),
                 eng.workspace.numel(), st)
        out = [_bits(mem.get(L.Y, M * L.N)), _bits(dsums), _bits(eng.flat.grad)] + [_bits(g) for g in grads]
        if L.has_bn:
            out.append(_bits(mem.get(L.sums, 2 * L.Cout)))
    stream.synchronize()
    return out


@pytest.mark.parametrize("wl,B", [("car", 2), ("refine_car", 4)])
def test_every_layer_is_bit_identical_across_streams_and_workspace_contents(wl, B):
    from frustum_convnet_b200.train_engine import TrainStep
    model = tr.make_model(wl, seed=B + 3)
    data = _data(wl, B, 60 + B)
    ts = TrainStep(model, deterministic=True)
    ts.forward_backward(data)
    torch.cuda.synchronize()
    eng = next(iter(ts.engines.values()))
    assert eng.deterministic
    mem = _engine_mem(eng, model)
    # accuracy: the deterministic step's own results within the float64 bounds of test_gpu_train_layers.py
    grad_exp, grad_S, dA_targets = {}, {}, {}
    for li, L in enumerate(eng.layers):
        nm, M = eng.names[li], L.B * L.T_out
        Y, S = tr.forward_ref(L, mem)
        got = mem.get(L.Y, M * L.N).view(M, L.N)
        _assert_within(got, Y, tr.contraction_tol(_seg_K(L), S), "%s %s Y" % (wl, nm))
        if L.has_bn:
            exp, sc = tr.stats_ref(L, got)
            _assert_within(mem.get(L.sums, 2 * L.Cout), exp, tr.sum_tol(sc), "%s %s sums" % (wl, nm))
        dy = tr.dy_ref(L, mem)
        ds, dss, amb = tr.reduce_ref(L, mem, dy)
        _assert_within(mem.get(L.dsums, ds.numel()), ds, tr.sum_tol(dss) + amb, "%s %s dsums" % (wl, nm))
        dWv, dWs, dWi = [], [], []
        for j in range(L.n_seg):
            widx, v, a, am = tr.dw_ref(L, j, mem, dy)
            dWi.append(widx.reshape(-1))
            dWv.append(v.reshape(-1))
            dWs.append((tr.contraction_tol(M, a) + am).reshape(-1))
        widx = torch.cat(dWi)
        nW = int(widx.max()) + 1
        ev, es = tr.scatter(nW, widx, torch.cat(dWv), torch.cat(dWs))
        off = (L.dW - eng.flat.grad.data_ptr()) // 4
        _assert_within(eng.flat.grad[off:off + nW], ev, es, "%s %s dW" % (wl, nm))
        # dX (train_dx_kernel<true> + train_dx_sum_kernel, or train_dx_plain_kernel): summed over every consumer
        for j in range(L.n_seg):
            s = L.seg[j].src
            if not ((eng.dx_mask[li] >> j) & 1) or not s.grad:
                continue
            idx, v, a, am = tr.dx_ref(L, j, mem, dy)
            n_src = L.B * s.T * s.ld
            tv, ts_ = tr.scatter(n_src, idx, v, tr.contraction_tol(L.N, a) + am)
            grad_exp[s.grad] = grad_exp.get(s.grad, 0) + tv
            grad_S[s.grad] = grad_S.get(s.grad, 0) + ts_
            dA_targets[s.grad] = n_src
        if L.has_bn:
            dsum = mem.get(L.dsums, 2 * L.Cout)
            assert torch.equal(mem.get(L.dbeta, L.Cout), dsum[:L.Cout].float()), "%s %s dbeta" % (wl, nm)
            assert torch.equal(mem.get(L.dgamma, L.Cout), dsum[L.Cout:].float()), "%s %s dgamma" % (wl, nm)
        elif L.dbias:
            assert torch.equal(mem.get(L.dbias, L.N), mem.get(L.dsums, L.N).float()), "%s %s dbias" % (wl, nm)
    # the pool backward's scatter into the last PointNet layer's dA
    for P in eng.pools:
        BT = P.B * P.T
        am = mem.get(P.argmax, BT * P.C).view(BT, P.C)
        exp_dA = tr.pool_bwd_ref(P, mem, am).reshape(-1)
        grad_exp[P.dA] = grad_exp.get(P.dA, 0) + exp_dA
        grad_S[P.dA] = grad_S.get(P.dA, 0) + torch.zeros_like(exp_dA)
        dA_targets[P.dA] = exp_dA.numel()
    assert dA_targets, "no source gradient was checked"
    for key, n in dA_targets.items():
        _assert_within(mem.get(key, n), grad_exp[key], grad_S[key],
                       "%s dA of the tensor at 0x%x (sum over consumers)" % (wl, key))
    # reproducibility: every layer twice, on two streams, with a NaN-filled and a random workspace
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for li in range(len(eng.layers)):
        r1 = _layer_run(eng, mem, li, s1, lambda w: w.fill_(math.nan))
        r2 = _layer_run(eng, mem, li, s2, lambda w: w.normal_())
        for k, (a, b) in enumerate(zip(r1, r2)):
            assert torch.equal(a, b), "%s %s: output %d differs between the two runs" % (wl, eng.names[li], k)


def test_workspace_errors_raise():
    from frustum_convnet_b200.train_engine import TrainStep
    model = tr.make_model("refine_car", seed=3)
    ts = TrainStep(model, deterministic=True)
    ts.forward_backward(_data("refine_car", 2, 5))
    eng = next(iter(ts.engines.values()))
    L = eng.layers[-3]
    need = int(_lib().load().fcn_train_deterministic_workspace_floats(C.byref(L)))
    assert need > 0
    st = torch.cuda.current_stream().cuda_stream
    for ptr, n in ((None, need), (eng.workspace.data_ptr(), need - 1)):
        with pytest.raises(RuntimeError, match="workspace"):
            _lib().call("fcn_train_forward_deterministic", C.byref(L), ptr, n, st)
        with pytest.raises(RuntimeError, match="workspace"):
            _lib().call("fcn_train_backward_deterministic", C.byref(L), 0, ptr, n, st)


# ============================================================================ whole step
def _steps(wl, B, optimizer, disturb=False):
    from frustum_convnet_b200.train_engine import TrainStep
    junk = [torch.empty(int(n), device="cuda") for n in (12345, 1 << 20, 77777)] if disturb else []
    model = tr.make_model(wl, seed=21)
    ts = TrainStep(model, lr=1e-3, optimizer=optimizer, momentum=0.9, deterministic=True)
    for i in range(3):
        ts.step(_data(wl, B, 100 + i))
        if disturb:
            junk.append(torch.randn(4096 * (i + 1), device="cuda"))
            del junk[0]
    torch.cuda.synchronize()
    opt = ts.optimizer
    state = [opt.exp_avg, opt.exp_avg_sq] if optimizer == "adam" else [opt.momentum_buffer]
    return dict(param=ts.flat.param.clone(), state=[t.clone() for t in state],
                buffers={n: b.clone() for n, b in model.named_buffers()},
                rows=ts.states.per_step(full=True).view(np.uint32), final=ts.states.finalize())


def _equal(r1, r2, what):
    assert torch.equal(r1["param"], r2["param"]), what + ": parameters"
    for a, b in zip(r1["state"], r2["state"]):
        assert torch.equal(a, b), what + ": optimizer state"
    for n in r1["buffers"]:
        assert torch.equal(r1["buffers"][n], r2["buffers"][n]), what + ": buffer " + n
    assert np.array_equal(r1["rows"], r2["rows"]), what + ": states rows"
    f1, f2 = r1["final"], r2["final"]
    assert f1.keys() == f2.keys()
    for k in f1:
        assert np.array_equal(np.asarray(f1[k], dtype=np.float64), np.asarray(f2[k], dtype=np.float64),
                              equal_nan=True), what + ": finalize " + k


@pytest.mark.parametrize("optimizer", ["adam", "sgd"])
@pytest.mark.parametrize("wl,B", [("refine_car", 32), ("car", 4), ("people", 4), ("sunrgbd", 4)])
def test_whole_steps_are_bit_identical(wl, B, optimizer):
    r1 = _steps(wl, B, optimizer)
    r2 = _steps(wl, B, optimizer, disturb=True)
    _equal(r1, r2, "%s B=%d %s" % (wl, B, optimizer))
    assert bool(torch.isfinite(r1["param"]).all())


def test_a_second_process_gives_the_same_parameters():
    code = ("import sys, hashlib; sys.path[:0] = [%r, %r]\n"
            "from test_gpu_train_deterministic import _steps\n"
            "r = _steps('refine_car', 32, 'adam')\n"
            "print('DIGEST', hashlib.sha256(r['param'].cpu().numpy().tobytes()).hexdigest())\n"
            % (ROOT, os.path.join(ROOT, "tests")))
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT)
    assert p.returncode == 0, p.stdout + p.stderr
    got = [ln.split()[1] for ln in p.stdout.splitlines() if ln.startswith("DIGEST")][0]
    r = _steps("refine_car", 32, "adam")
    assert got == hashlib.sha256(r["param"].cpu().numpy().tobytes()).hexdigest()


# ============================================================================ fused loss
class DetCall(Call):
    """A fcn_det_loss_deterministic call on the same inputs (scratch of the deterministic size, NaN-filled)."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        n = int(_lib().load().fcn_det_loss_deterministic_scratch_floats(self.N))
        self.scratch = torch.full((n,), math.nan, device="cuda")
        self.args.scratch = self.scratch.data_ptr()

    def run(self, stream=None):
        s = stream if stream is not None else torch.cuda.current_stream()
        _lib().call("fcn_det_loss_deterministic", C.byref(self.args), s.cuda_stream)
        s.synchronize()
        return self.out.clone(), self.dcls[:self.N].clone(), self.dreg[:self.N].clone()


@pytest.mark.parametrize("B,T2,NH,NS,seed", [(32, 280, 12, 3, 8), (3, 140, 12, 8, 2), (1, 1, 4, 1, 5)])
def test_deterministic_loss_bits_and_bounds(B, T2, NH, NS, seed):
    case = lr.make_case(B, T2, NH, NS, seed=seed)
    det = DetCall(case, NH, NS)
    o1, c1, r1 = det.run()
    o2, c2, r2 = det.run(torch.cuda.Stream())
    det.scratch.normal_()
    o3, _, _ = det.run()
    for o in (o2, o3):
        assert torch.equal(o.view(torch.int32), o1.view(torch.int32))
    assert torch.equal(c2.view(torch.int32), c1.view(torch.int32)) and torch.equal(r2.view(torch.int32),
                                                                                   r1.view(torch.int32))
    _, c0, r0 = Call(case, NH, NS).run()
    assert torch.equal(c0.view(torch.int32), c1.view(torch.int32)), "dcls differs from fcn_det_loss's"
    assert torch.equal(r0.view(torch.int32), r1.view(torch.int32)), "dreg differs from fcn_det_loss's"
    check(det, o1, c1, r1)


# ============================================================================ torch's flag
def test_dropin_loop_under_torch_flag_gives_identical_grads(torch_deterministic):
    torch.use_deterministic_algorithms(True, warn_only=True)
    model = tr.make_model("refine_car", seed=9)
    model.train()
    data = _data("refine_car", 8, 31)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    grads = []
    for _ in range(2):
        model.load_state_dict(state)
        model.zero_grad(set_to_none=True)
        losses, _ = model(data)
        losses["total_loss"].backward()
        grads.append([p.grad.clone() for p in model.parameters()])
    engines = [e for e in model.__dict__["_train_engines"].values()]
    assert engines and all(e.deterministic for e in engines)
    for a, b in zip(*grads):
        assert torch.equal(a, b)


def test_trainstep_follows_the_torch_flag_both_ways(torch_deterministic):
    from frustum_convnet_b200.train_engine import TrainStep
    model = tr.make_model("refine_car", seed=4)
    ts = TrainStep(model)
    assert ts.deterministic is None
    data = _data("refine_car", 4, 8)
    torch.use_deterministic_algorithms(True, warn_only=True)
    ts.step(data)
    torch.use_deterministic_algorithms(False)
    ts.step(data)
    modes = sorted(e.deterministic for e in ts.engines.values())
    assert modes == [False, True]
    ts.deterministic = False
    torch.use_deterministic_algorithms(True, warn_only=True)
    ts.step(data)
    assert len(ts.engines) == 2
