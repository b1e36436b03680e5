"""Float32 restatement of the eval decode ``decode_row`` (csrc/decode.cuh): the softmax / argmax / box decode of
the model's eval branch (models/det_base.py:376-411 of the original code) with ``angle_decode`` and
``size_decode`` (models/box_transform.py:5-12,28-41).  ``decode`` takes head-logit rows in the kernel's layout
[cls0, cls1, centre(3), heading scores(NH), heading res(NH), size scores(NS), size res(NS*3)] and returns, per row:

  * the three probability vectors as a float64 softmax of the float32 logits, each with a per-element bound;
  * the label SETS of the two arg-maxes (every index a float32 softmax within the bound could pick);
  * the centre, and the heading / size decode of any given label, bit-exactly in float32.

``check`` compares the six outputs of one kernel call with it.

Probability bound.  With u = 2^-24, one row x of n float32 logits, m = max x, d_j = |x_j - m| and p64 the float64
softmax, the kernel computes q_j = expf(fl(x_j - m)), s = sum_j q_j (in index order) and p_j = q_j / s.

  * fl(x_j - m) = (x_j - m)(1 + a), |a| <= u, i.e. an absolute error <= u d_j in the exponent: exp of it has
    relative error <= u d_j (first order).  CUDA's expf is within 2 ulp, i.e. 4u relative.  So
    q_j = exp(x_j - m)(1 + eps_j) with |eps_j| <= e_j = u (d_j + 4).
  * The n - 1 additions of non-negative terms add at most (n - 1) u relative: s = S (1 + sigma) with
    |sigma| <= sum_j e_j p64_j + (n - 1) u, where S = sum_j exp(x_j - m).  The weighted sum is at most max_j e_j,
    and it ignores terms that are zero in both (an exponent below the float32 range, an entry of -inf).
  * The division adds u.  p_j = p64_j (1 + eps_j)(1 + u') / (1 + sigma): to first order
    |p_j - p64_j| <= p64_j (e_j + sum_k e_k p64_k + n u); the factor 2 covers the second-order terms.
  * A q_j in the subnormal range has an absolute error of a few 2^-149, and s >= 1 (the maximum contributes
    exp(0) = 1): 2^-140 covers it.

    bound_j = 2 p64_j (e_j + sum_k e_k p64_k + n u) + 2^-140

Labels.  The kernel takes the FIRST maximum of its float32 probabilities.  Index k can be that maximum only if
p_k >= p_i for the index i of the largest p64, so L = {k : p64_k >= p64_max - (bound_k + bound_max)} holds every
possible label.  ``check`` reads the label from the kernel's own probabilities (numpy's argmax takes the first
maximum too) and requires it to lie in L and the heading / size to be the bit-exact decode of THAT label: a tie
rule other than the first maximum, or an argmax over logits instead of probabilities, changes the decode of rows
whose probabilities tie.

Decode (the model's float32 tensor arithmetic; the python-double constants enter each float32 operation as
float32 scalars, so 2 pi / NH and pi / NH are rounded once each):

    centre  = f32(off_c + center_ref[(b*3 + c)*T + t])
    heading = f32(f32(hl * f32(2 pi / NH)) + f32(res * f32(2 pi / NH / 2))), minus f32(2 pi) once if > f32(pi)
    size    = f32(f32(sr * ex) + ex),  ex = mean_size[sl, c]

Non-finite rows (NaN or +inf anywhere, or every entry -inf) give NaN probabilities and label 0, as torch's softmax
and argmax do (the kernel's m = fmaxf(...) skips NaN, but s and every p_j are then NaN, and no NaN is ``> best``).
"""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -140
F32 = np.float32
PI32 = F32(np.pi)
TWO_PI32 = F32(2 * np.pi)


def row_width(NH, NS):
    return 5 + 2 * NH + 4 * NS


def softmax_bound(x):
    """x (R, n) float32 -> (p64 (R, n), bound (R, n), finite (R,)).  Non-finite rows: NaN p64, NaN bound."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    R, n = x.shape
    finite = ~np.isnan(x).any(1) & ~np.isposinf(x).any(1) & ~np.isneginf(x).all(1)
    p64 = np.full((R, n), np.nan)
    bound = np.full((R, n), np.nan)
    if finite.any():
        xf = x[finite]
        m = xf.max(1, keepdims=True)
        with np.errstate(invalid="ignore", over="ignore"):
            d = m - xf                                   # >= 0, +inf for -inf entries
            q = np.exp(-d)
            p = q / q.sum(1, keepdims=True)
            e = U * (d + 4.0)
            pe = np.where(p > 0, e * p, 0.0)             # terms that are zero in both arithmetics add nothing
        b = 2.0 * p * (np.where(p > 0, e, 0.0) + pe.sum(1, keepdims=True) + n * U) + TINY
        p64[finite], bound[finite] = p, b
    return p64, bound, finite


def label_sets(p64, bound, finite):
    """(R, n) bool: every index a float32 first-maximum within the bound could pick; {0} for non-finite rows."""
    L = np.zeros(p64.shape, dtype=bool)
    L[~finite, 0] = True
    if finite.any():
        p, b = p64[finite], bound[finite]
        i = p.argmax(1)
        r = np.arange(len(p))
        L[finite] = p >= (p[r, i] - b[r, i])[:, None] - b
    return L


def heading_decode(hl, res, NH):
    """f32 angle of bin hl (int array) with normalised residual res (float32 array)."""
    apc = F32(2 * np.pi / NH)
    half = F32(2 * np.pi / NH / 2)
    ang = ((np.asarray(hl).astype(np.float32) * apc).astype(np.float32) +
           (np.asarray(res, np.float32) * half).astype(np.float32)).astype(np.float32)
    return np.where(ang > PI32, (ang - TWO_PI32).astype(np.float32), ang).astype(np.float32)


def size_decode(sl, sr, mean_size):
    """f32 (R, 3) size of cluster sl (int array) from its residuals sr (R, 3) float32."""
    ex = np.asarray(mean_size, np.float32)[np.asarray(sl)]
    return ((np.asarray(sr, np.float32) * ex).astype(np.float32) + ex).astype(np.float32)


def decode(rows, B, T, NH, NS, center_ref, mean_size):
    """rows (B*T, >= 5 + 2 NH + 4 NS) float32 logit rows (row r = b*T + t); center_ref (B, 3, T); mean_size (NS, 3)."""
    rows = np.asarray(rows, dtype=np.float32)
    R = B * T
    assert rows.shape[0] == R and rows.shape[1] >= row_width(NH, NS)
    cr = np.asarray(center_ref, np.float32).reshape(B, 3, T).transpose(0, 2, 1).reshape(R, 3)
    hs, hr = rows[:, 5:5 + NH], rows[:, 5 + NH:5 + 2 * NH]
    ss, sr = rows[:, 5 + 2 * NH:5 + 2 * NH + NS], rows[:, 5 + 2 * NH + NS:5 + 2 * NH + 4 * NS].reshape(R, NS, 3)
    o = SimpleNamespace(B=B, T=T, NH=NH, NS=NS, hr=hr, sr=sr, mean_size=np.asarray(mean_size, np.float32))
    o.cls = softmax_bound(rows[:, 0:2])
    o.hp = softmax_bound(hs)
    o.sp = softmax_bound(ss)
    o.hL = label_sets(*o.hp)
    o.sL = label_sets(*o.sp)
    o.center = (rows[:, 2:5] + cr).astype(np.float32)
    return o


def heading_of(o, hl):
    return heading_decode(hl, o.hr[np.arange(len(hl)), hl], o.NH)


def size_of(o, sl):
    return size_decode(sl, o.sr[np.arange(len(sl)), sl], o.mean_size)


def first_max(p):
    """The kernel's label from its own float32 probabilities: the first maximum, 0 for an all-NaN row."""
    p = np.asarray(p, np.float32)
    return np.where(np.isnan(p).all(1), 0, np.nanargmax(np.where(np.isnan(p), -np.inf, p), 1))


def _probs_ok(got, ref, what):
    p64, bound, finite = ref
    got = np.asarray(got, np.float64)
    assert np.isnan(got[~finite]).all(), "%s: a non-finite row gave a number" % what
    g, p, b = got[finite], p64[finite], bound[finite]
    err = np.abs(g - p)
    bad = ~(err <= b)
    if bad.any():
        r, j = np.argwhere(bad)[0]
        raise AssertionError("%s: %d probabilities out of bound; first row %d col %d: got %.9g want %.17g bound %.3g"
                             % (what, int(bad.sum()), r, j, g[r, j], p[r, j], b[r, j]))
    # exact zeros stay zeros (-inf entries, exponents below the float32 range), and no probability passes 1
    assert (g[p == 0] == 0).all() and (g <= 1).all(), what


def _bits_equal(got, want, what):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    same = got.view(np.int32) == want.view(np.int32)
    if not same.all():
        i = np.argwhere(~same)[0]
        raise AssertionError("%s: %d values differ bit-wise; first at %s: got %r want %r"
                             % (what, int((~same).sum()), tuple(i), got[tuple(i)], want[tuple(i)]))


def check(o, cls_probs, center, heading, size, heading_probs, size_probs, what=""):
    """The six outputs of one decode against the restatement.  Returns (heading labels, size labels)."""
    R = o.B * o.T
    cls_probs, center = np.asarray(cls_probs).reshape(R, 2), np.asarray(center).reshape(R, 3)
    heading, size = np.asarray(heading).reshape(R), np.asarray(size).reshape(R, 3)
    heading_probs, size_probs = np.asarray(heading_probs).reshape(R, o.NH), np.asarray(size_probs).reshape(R, o.NS)
    _probs_ok(cls_probs, o.cls, what + " cls_probs")
    _probs_ok(heading_probs, o.hp, what + " heading_probs")
    _probs_ok(size_probs, o.sp, what + " size_probs")
    _bits_equal(center, o.center, what + " center")
    hl, sl = first_max(heading_probs), first_max(size_probs)
    r = np.arange(R)
    assert o.hL[r, hl].all(), "%s: heading label outside the label set at rows %s" % (what, np.nonzero(~o.hL[r, hl])[0][:8])
    assert o.sL[r, sl].all(), "%s: size label outside the label set at rows %s" % (what, np.nonzero(~o.sL[r, sl])[0][:8])
    _bits_equal(heading, heading_of(o, hl), what + " heading")
    _bits_equal(size, size_of(o, sl), what + " size")
    return hl, sl


# ------------------------------------------------------------------ crafted rows
def _pre_wrap(hl, res, NH):
    apc, half = F32(2 * np.pi / NH), F32(2 * np.pi / NH / 2)
    return (F32(hl) * apc + np.asarray(res, np.float32) * half).astype(np.float32)


def residuals_at_pi(NH):
    """(hl, res_eq, res_up): residuals of bin hl whose decoded angle before the wrap is exactly f32(pi) and the
    smallest float above it that the decode reaches (its next float up wherever some bin reaches that; with NH = 1
    the product res * f32(pi) moves in steps of two ulp), found by a search over neighbouring float32 residuals."""
    up = np.nextafter(PI32, F32(np.inf))
    half = F32(2 * np.pi / NH / 2)
    best = None
    for hl in sorted(range(NH), key=lambda h: abs(h - (NH - 1) / 2.0)):
        start = np.float64(F32(hl) * F32(2 * np.pi / NH))
        found = []
        for target in (PI32, up):
            r0 = F32((np.float64(target) - start) / np.float64(half))
            cand = r0 + np.arange(-256, 257, dtype=np.float32) * np.spacing(r0)
            a = _pre_wrap(hl, cand, NH)
            found.append(cand[a == PI32] if target == PI32 else cand[a > PI32])
        eq, hi = found
        if len(eq) and len(hi):
            if _pre_wrap(hl, hi[0], NH) == up:
                return hl, F32(eq[0]), F32(hi[0])
            best = best or (hl, F32(eq[0]), F32(hi[0]))
    assert best is not None, "no residual lands on f32(pi) for NH=%d" % NH
    return best


def crafted_rows(NH, NS, seed=0, n_random=64, mean_size=None):
    """Logit rows at the decode's edges plus random rows.  Returns (rows (R, W) float32, families): families maps a
    name to (row indices, expected heading label or None, expected size label or None); 'cls_exact' rows carry
    their exact class probabilities in families['cls_want'].  With ``mean_size`` the 'fma_sensitive' rows get size
    residuals whose decode changes under a fused multiply-add; their heading residuals do so for a bin hl > 0."""
    rng = np.random.default_rng(seed)
    W = row_width(NH, NS)
    h0, r0, s0, q0 = 5, 5 + NH, 5 + 2 * NH, 5 + 2 * NH + NS
    rows, fam = [], {}

    def base():
        r = np.empty(W, np.float32)
        r[0:2] = rng.normal(0, 2, 2)
        r[2:5] = rng.normal(0, 5, 3)
        r[h0:h0 + NH] = rng.normal(0, 2, NH)
        r[r0:r0 + NH] = rng.uniform(-1.2, 1.2, NH)             # distinct residuals: a wrong label shows
        r[s0:s0 + NS] = rng.normal(0, 2, NS)
        r[q0:q0 + 3 * NS] = rng.uniform(-0.8, 0.8, 3 * NS)
        return r

    def add(name, r, hl=None, sl=None):
        idx, hls, sls = fam.setdefault(name, ([], [], []))
        idx.append(len(rows))
        hls.append(hl)
        sls.append(sl)
        rows.append(r)

    def clear_heading(r, hl, v=8.0):                            # bin hl the clear maximum
        r[h0:h0 + NH] = rng.uniform(-2, 0, NH)
        r[h0 + hl] = v

    # exact ties: the first maximum wins
    for k in range(4):
        r = base()
        if NH >= 2:
            i, j = sorted(rng.choice(NH, 2, replace=False))
            r[h0:h0 + NH] = rng.uniform(-3, 0, NH)
            r[h0 + i] = r[h0 + j] = F32(1.25 + k)
        else:
            i = 0
        if NS >= 2:
            a, b = sorted(rng.choice(NS, 2, replace=False))
            r[s0:s0 + NS] = rng.uniform(-3, 0, NS)
            r[s0 + a] = r[s0 + b] = F32(0.5 + k)
        else:
            a = 0
        add("tie_first", r, i, a)
    r = base()
    r[h0:h0 + NH] = F32(0.3)
    r[s0:s0 + NS] = F32(-2.0)
    add("tie_first", r, 0, 0)                                   # every score equal
    # distinct logits whose float32 probabilities tie: label 0, not the larger logit
    if NH >= 2 and NS >= 2:
        r = base()
        x = F32(1e-30)
        r[h0:h0 + NH] = F32(-1e4)
        r[h0], r[h0 + 1] = x, np.nextafter(x, F32(1))
        r[s0:s0 + NS] = F32(-1e4)
        r[s0], r[s0 + 1] = F32(-2e-9), np.nextafter(F32(-2e-9), F32(0))
        add("prob_tie", r, 0, 0)
    # 1-ulp near ties: any label of the set
    for k in range(6):
        r = base()
        if NH >= 2:
            i, j = rng.choice(NH, 2, replace=False)
            x = F32(rng.uniform(-4, 4))
            r[h0 + i], r[h0 + j] = x, np.nextafter(x, F32(np.inf) if k % 2 else F32(-np.inf))
            r[h0:h0 + NH] = np.minimum(r[h0:h0 + NH], x)
        if NS >= 2:
            a, b = rng.choice(NS, 2, replace=False)
            x = F32(rng.uniform(-4, 4))
            r[s0 + a], r[s0 + b] = x, np.nextafter(x, F32(np.inf))
            r[s0:s0 + NS] = np.minimum(r[s0:s0 + NS], np.nextafter(x, F32(np.inf)))
        add("near_tie", r)
    # class scores: equal, saturated either way, -inf
    cls_want = []
    for c, want in (([0.0, 0.0], [0.5, 0.5]), ([3.5, 3.5], [0.5, 0.5]), ([0.0, 200.0], [0.0, 1.0]),
                    ([200.0, 0.0], [1.0, 0.0]), ([-np.inf, 1.0], [0.0, 1.0]), ([1e30, -1e30], [1.0, 0.0])):
        r = base()
        r[0:2] = c
        add("cls_exact", r)
        cls_want.append(want)
    # -inf entries: probability exactly 0
    r = base()
    clear_heading(r, NH - 1)
    if NH >= 2:
        r[h0] = -np.inf
    if NS >= 2:
        r[s0 + NS - 1] = -np.inf
        r[s0] = F32(9.0)
    add("neg_inf", r, NH - 1, 0)
    # non-finite rows: NaN probabilities, label 0
    for where in ("nan_h", "inf_h", "ninf_h", "nan_s", "inf_s", "ninf_s", "nan_cls", "inf_cls"):
        r = base()
        if where.endswith("_h"):
            j = int(rng.integers(NH))
            r[h0 + j] = {"nan": np.nan, "inf": np.inf}.get(where[:-2], 0.0)
            if where == "ninf_h":
                r[h0:h0 + NH] = -np.inf
        elif where.endswith("_s"):
            j = int(rng.integers(NS))
            r[s0 + j] = {"nan": np.nan, "inf": np.inf}.get(where[:-2], 0.0)
            if where == "ninf_s":
                r[s0:s0 + NS] = -np.inf
        else:
            r[int(rng.integers(2))] = np.nan if where == "nan_cls" else np.inf
        add("non_finite", r, 0 if where.endswith("_h") else None, 0 if where.endswith("_s") else None)
    # heading wrap: last bin, residual +1
    r = base()
    clear_heading(r, NH - 1)
    r[r0 + NH - 1] = 1.0
    add("wrap_last_bin", r, NH - 1)
    # exactly f32(pi) (kept) and the next float up (wrapped)
    hl, req, rup = residuals_at_pi(NH)
    for res, name in ((req, "at_pi"), (rup, "above_pi")):
        r = base()
        clear_heading(r, hl)
        r[r0 + hl] = res
        add(name, r, hl)
    # bin 0, residual -1: negative angle, no wrap
    r = base()
    clear_heading(r, 0)
    r[r0] = -1.0
    add("negative", r, 0)
    # large residuals: one subtraction only
    for res in (5.0, -5.0, 1e3, -1e3):
        r = base()
        clear_heading(r, NH - 1)
        r[r0 + NH - 1] = res
        add("large_res", r, NH - 1)
    # last size cluster, residual -1: exactly 0
    r = base()
    r[s0:s0 + NS] = rng.uniform(-2, 0, NS)
    r[s0 + NS - 1] = 7.0
    r[q0 + 3 * (NS - 1):q0 + 3 * NS] = -1.0
    add("size_zero", r, None, NS - 1)
    # rows whose heading and size change when a product is fused with the addition (a contracted decode shows)
    apc, half = F32(2 * np.pi / NH), F32(2 * np.pi / NH / 2)
    for k in range(8):
        r = base()
        hl, sl = int(rng.integers(NH)), int(rng.integers(NS))
        clear_heading(r, hl)
        r[s0:s0 + NS] = rng.uniform(-2, 0, NS)
        r[s0 + sl] = 6.0
        p1 = F32(F32(hl) * apc)
        while hl > 0:
            res = F32(rng.uniform(-1.2, 1.2))
            if _fma32(res, half, p1) != F32(F32(res * half) + p1):
                r[r0 + hl] = res
                break
        ex = np.asarray(mean_size, np.float32)[sl] if mean_size is not None else None
        for c in range(3):
            while ex is not None:
                v = F32(rng.uniform(-0.8, 0.8))
                if _fma32(v, ex[c], ex[c]) != F32(F32(v * ex[c]) + ex[c]):
                    r[q0 + 3 * sl + c] = v
                    break
        add("fma_sensitive", r, hl, sl)
    for _ in range(n_random):
        add("random", base())
    out = {k: (np.array(v[0]), v[1], v[2]) for k, v in fam.items()}
    out["cls_want"] = np.array(cls_want, np.float32)
    return np.stack(rows).astype(np.float32), out


def _fma32(a, b, c):
    """float32 fused multiply-add via float64 (the product of two float32 is exact in float64)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(np.float32)


def contraction_sensitive(o, hl, sl):
    """Rows whose heading / size change when either product of the decode is fused with the addition."""
    r = np.arange(len(hl))
    apc, half = F32(2 * np.pi / o.NH), F32(2 * np.pi / o.NH / 2)
    res = o.hr[r, hl]
    p1 = (hl.astype(np.float32) * apc).astype(np.float32)
    p2 = (res * half).astype(np.float32)
    two = (p1 + p2).astype(np.float32)
    h = (_fma32(hl.astype(np.float32), apc, p2) != two) | (_fma32(res, half, p1) != two)
    ex = o.mean_size[sl]
    sr = o.sr[r, sl]
    s = (_fma32(sr, ex, ex) != ((sr * ex).astype(np.float32) + ex).astype(np.float32)).any(1)
    return h, s
