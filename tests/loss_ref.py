"""Float64 statement of the fused detection loss of include/frustum_b200.h section 7b (csrc/loss.cu, fcn_det_loss).

``det_loss_ref`` takes one call's own inputs (the kernel's layout: logits ``cls`` (N, 2) and ``reg`` (N, W) with
N = B*T2 and W = 3 + 2*NH + 4*NS, ``cls_label`` (B, T2), ``center_ref2`` (B, 3, T2), the GT boxes, ``size_class``,
``mean_size`` (NS, 3), the four loss weights, NH and NS) and returns the eight losses, the six metrics and
d(total)/d(logits), the gradient by float64 autograd.

Discrete decisions follow the float32 arithmetic of the model's train branch (models/det_base.py:414-525 of the
original code): the heading class and normalised residual of ``angle_encode`` are computed with the same float32
tensor operations, and the bin start ``class * angle_per_class`` of the decode is the float32 product.  Everything
continuous is float64: offsets, norms, softmaxes, Huber terms, corners, the decoded angle and the pi wrap (the wrap
does not change a corner).  Arg-maxes take the first maximum, as ``torch.argmax`` does.

Corner loss at an exact tie ``dg == df``: the loss takes the GT box (``dg <= df``) and its whole gradient goes to
the GT side.  ``torch.min`` would send half to each side; at a tie both one-sided gradients are valid, but only the
GT one is the gradient of the branch whose value the loss reports, and the half split can cancel to zero (a box
of zero width half-way between two opposite corner sets gets a zero size gradient from ``torch.min`` and a
non-zero one here).  csrc/loss.cu implements this choice; tests/test_det_loss_cpu.py and
tests/test_gpu_det_loss.py pin it.

Rounding companions.  Next to each value the reference returns a magnitude built from absolute values of the terms
the kernel rounds (``mag_*``).  With u = 2^-24 the kernel's error is bounded by ``c * u * mag`` for a small
constant c; the GPU test states the bounds.  Rows whose discrete decision is within rounding in float32 (flip
choice, arg-max) are flagged (``amb_*``); for the flip choice the gradient of the other choice is returned too.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import torch

U = 2.0 ** -24                       # unit round-off of fp32
EPS14 = float(np.float32(1e-14))     # the focal loss's 1e-14, as the fp32 arithmetic sees it
F64 = torch.float64
SX = torch.tensor([1, 1, -1, -1, 1, 1, -1, -1], dtype=F64)
SY = torch.tensor([1, 1, 1, 1, -1, -1, -1, -1], dtype=F64)
SZ = torch.tensor([1, -1, -1, 1, 1, -1, -1, 1], dtype=F64)
AMB_ARG = 2.0 ** -18                 # relative logit gap below which an fp32 arg-max is undecidable
AMB_FLIP = 64 * U                    # |dg - df| below this * (coordinate scale): flip choice undecidable


def angle_encode_f32(heading, NH):
    """Heading class (int64) and normalised residual (float32) with the float32 operations of angle_encode
    (box_transform.py:34-47): the python-double constants enter each float32 tensor operation as float32."""
    two_pi = 2 * np.pi
    apc = two_pi / float(NH)
    g = heading.float() % two_pi
    assert bool(((g >= 0) & (g <= two_pi)).all())
    shifted = (g + apc / 2) % two_pi
    # just above the last boundary, shifted / apc can round up to NH: the model's gather then fails (an index
    # error, no value to match); the kernel clamps to the last bin, whose residual (~ +1) names the same angle
    hc = torch.clamp(torch.floor(shifted / apc).long(), max=NH - 1)
    res = (shifted - (hc.float() * apc + apc / 2)) / (apc / 2)
    return hc, res, shifted


def bin_start_f32(cls_id, NH):
    """``class.float() * angle_per_class`` of angle_decode, in float32, returned as float64."""
    return (cls_id.float() * (2 * np.pi / float(NH))).double()


def half_bin(NH):
    """The float32 constant ``angle_per_class / 2`` as float64."""
    return float(np.float32(2 * np.pi / float(NH) / 2))


def total_f32(means, weights):
    """The total loss of det_base.py:468-474 as float32 tensors compute it from the seven float32 means
    [cls, center, head_cls, head_res, size_cls, size_res, corners] and the four loss weights (w_box, w_head_reg,
    w_size_reg, w_corner): Python's evaluation order, each Python-float weight entering as float32, every product and
    sum rounded on its own.  Returns a numpy float32."""
    f = np.float32
    cls, center, hcls, hres, scls, sres, corner = (f(m) for m in means)
    w_box, w_hr, w_sr, w_c = (f(w) for w in weights)
    box = f(f(center + hcls) + scls)
    box = f(box + f(w_hr * hres))
    box = f(box + f(w_sr * sres))
    box = f(box + f(w_c * corner))
    return f(cls + f(w_box * box))


def accuracy_f32(correct, n):
    """get_accuracy (utils/utils.py:28-48) of `correct` hits over n >= 1 rows: the float32 count times the Python
    double 1.0 / n, which enters the float32 multiply rounded to float32.  Returns a numpy float32."""
    return np.float32(np.float32(correct) * np.float32(1.0 / n))


def corners(ctr, heading, size):
    """(n, 8, 3) float64 corners of model_util.py:48-72 (x: +-l/2, y: +-h/2, z: +-w/2; rotation about y)."""
    x = SX * size[:, :1] * 0.5
    y = SY * size[:, 2:3] * 0.5
    z = SZ * size[:, 1:2] * 0.5
    c, s = torch.cos(heading)[:, None], torch.sin(heading)[:, None]
    return torch.stack([c * x + s * z + ctr[:, :1], y + ctr[:, 1:2], -s * x + c * z + ctr[:, 2:3]], -1)


def _safe_norm(v):
    """Euclidean norm over the last axis with gradient 0 at 0 (the kernel skips zero-length corner terms)."""
    n2 = (v * v).sum(-1)
    pos = n2 > 0
    return torch.where(pos, torch.sqrt(torch.where(pos, n2, torch.ones_like(n2))), torch.zeros_like(n2))


def _huber(a_abs, delta):
    q = torch.clamp(a_abs, max=delta)
    return 0.5 * q * q + delta * (a_abs - q)


def _first_argmax(x):
    """Arg-max with the first maximum on ties, and whether the top two are within fp32 rounding (not equal)."""
    arg = torch.argmax(x, -1)
    top = x.gather(-1, arg[:, None])[:, 0]
    other = x.clone()
    other.scatter_(-1, arg[:, None], -math.inf)
    gap = top - other.max(-1).values if x.shape[-1] > 1 else torch.full_like(top, math.inf)
    amb = (gap > 0) & (gap <= AMB_ARG * torch.clamp(top.abs(), min=1.0))
    return arg, amb


def det_loss_ref(cls, reg, cls_label, center_ref2, box3d_center, box3d_heading, box3d_size, size_class, mean_size,
                 weights, NH, NS, iou_thresh=0.7, with_iou=True):
    """See the module docstring.  Tensors on any device; everything is computed on the CPU."""
    from oracle import box_iou as obox
    w_box, w_hr, w_sr, w_c = (float(w) for w in weights)
    cls, reg = cls.detach().cpu().float(), reg.detach().cpu().float()
    B, _, T2 = center_ref2.shape
    N, W = B * T2, 3 + 2 * NH + 4 * NS
    assert cls.shape == (N, 2) and reg.shape == (N, W)
    lab = cls_label.detach().cpu().reshape(-1).long()
    cref = center_ref2.detach().cpu().float()
    cgt_b = box3d_center.detach().cpu().float().reshape(B, 3)
    hgt_b = box3d_heading.detach().cpu().float().reshape(B)
    sgt_b = box3d_size.detach().cpu().float().reshape(B, 3)
    sc_b = size_class.detach().cpu().reshape(B).long()
    ms = mean_size.detach().cpu().float().reshape(NS, 3)

    keep, fg = lab != -1, lab == 1
    nfg = int(fg.sum())
    nfg_c = float(max(nfg, 1))
    fgi = torch.nonzero(fg).reshape(-1)
    b_of, t_of = fgi // T2, fgi % T2
    n = len(fgi)

    def run(flip_override=None):
        c64 = cls.double().requires_grad_(True)
        r64 = reg.double().requires_grad_(True)
        # ---- focal loss over the rows with label != -1
        p = torch.softmax(c64, -1)
        tl = (lab >= 1).long()
        pt = p.gather(1, tl[:, None])[:, 0]
        alpha = torch.where(tl == 0, 0.75, 0.25).double()
        lg = torch.log(pt + EPS14)
        focal = torch.where(keep, -alpha * (1 - pt) ** 2 * lg, torch.zeros_like(pt))
        l_cls = focal.sum() / (nfg + EPS14)
        # ---- foreground rows
        o = r64[fgi]
        ctr, hs, hr = o[:, :3], o[:, 3:3 + NH], o[:, 3 + NH:3 + 2 * NH]
        ss, sr = o[:, 3 + 2 * NH:3 + 2 * NH + NS], o[:, 3 + 2 * NH + NS:].reshape(n, NS, 3)
        cgt, ref = cgt_b[b_of].double(), cref[b_of, :, t_of].double()
        hgt, sgt, sc = hgt_b[b_of], sgt_b[b_of].double(), sc_b[b_of]
        ex = ms[sc].double()
        hc, hres_lab, shifted = angle_encode_f32(hgt, NH)
        dv_c = (cgt - ref) - ctr
        d_c = _safe_norm(dv_c)
        t_center = _huber(d_c, 3.0)
        t_hcls = -torch.log_softmax(hs, -1).gather(1, hc[:, None])[:, 0]
        e_h = hr.gather(1, hc[:, None])[:, 0] - hres_lab.double()
        t_hres = _huber(e_h.abs(), 1.0)
        t_scls = -torch.log_softmax(ss, -1).gather(1, sc[:, None])[:, 0]
        sr_sel = sr[torch.arange(n), sc]
        dv_s = (sgt - ex) / ex - sr_sel
        d_s = _safe_norm(dv_s)
        t_sres = _huber(d_s, 1.0)
        cp = ref + ctr
        ang = bin_start_f32(hc, NH) + hr.gather(1, hc[:, None])[:, 0] * half_bin(NH)
        ang = torch.where(ang > math.pi, ang - 2 * math.pi, ang)
        sz = sr_sel * ex + ex
        P = corners(cp, ang, sz)
        G = corners(cgt, hgt.double(), sgt)
        Fl = corners(cgt, hgt.double() + math.pi, sgt)
        dg = _safe_norm(P - G).mean(-1)
        df = _safe_norm(P - Fl).mean(-1)
        use_g = dg <= df
        if flip_override is not None:
            use_g = flip_override
        D = torch.where(use_g, dg, df)
        t_corner = _huber(D, 1.0)
        terms = [t_center, t_hcls, t_hres, t_scls, t_sres, t_corner]
        means = [t.sum() / nfg_c for t in terms]
        total = l_cls + w_box * (means[0] + means[1] + means[3] + w_hr * means[2] + w_sr * means[4] + w_c * means[5])
        total.backward()
        ns = SimpleNamespace(
            losses=torch.stack([total, l_cls] + means).detach(), dcls=c64.grad, dreg=r64.grad,
            p=p.detach(), pt=pt.detach(), lg=lg.detach(), focal=focal.detach(), alpha=alpha,
            hc=hc, hres_lab=hres_lab, shifted=shifted, use_g=use_g, dg=dg.detach(), df=df.detach(),
            d_c=d_c.detach(), d_s=d_s.detach(), e_h=e_h.detach(), D=D.detach(), ang=ang.detach(),
            cp=cp.detach(), sz=sz.detach(), ex=ex, cgt=cgt, ref=ref, hgt=hgt.double(), sgt=sgt, sc=sc,
            terms=[t.detach() for t in terms], G=G.detach())
        return ns

    r = run()
    # ---- flip decisions within rounding: the gradient of the other choice
    coord = (r.cp.abs().sum(-1) + r.cgt.abs().sum(-1) + r.sz.abs().sum(-1) + r.sgt.abs().sum(-1)
             + (r.sz.abs().sum(-1) + r.sgt.abs().sum(-1)) * (2 * math.pi + r.ang.abs() + r.hgt.abs()))
    amb_flip = (r.dg - r.df).abs() <= AMB_FLIP * coord
    dreg_alt = r.dreg
    if bool(amb_flip.any()):
        dreg_alt = run(torch.where(amb_flip, ~r.use_g, r.use_g)).dreg

    # ---- metrics (no gradient)
    cls_arg, amb_cls = _first_argmax(cls.double())
    o = reg.double()[fgi]
    h_arg, amb_h = _first_argmax(o[:, 3:3 + NH])
    s_arg, amb_s = _first_argmax(o[:, 3 + 2 * NH:3 + 2 * NH + NS])
    cls_acc = float((cls_arg[keep] == lab[keep]).double().sum()) / max(int(keep.sum()), 1)
    head_acc = float((h_arg == r.hc).double().sum()) / nfg_c
    size_acc = float((s_arg == r.sc).double().sum()) / nfg_c
    iou = np.zeros((n, 2))
    if n:
        hr = o[:, 3 + NH:3 + 2 * NH]
        srp = o[:, 3 + 2 * NH + NS:].reshape(n, NS, 3)[torch.arange(n), s_arg]
        angp = bin_start_f32(h_arg, NH) + hr.gather(1, h_arg[:, None])[:, 0] * half_bin(NH)
        angp = torch.where(angp > math.pi, angp - 2 * math.pi, angp)
        msp = ms[s_arg].double()
        Pp = corners(r.cp, angp, srp * msp + msp)
        iou = obox.rbbox_iou_3d_pair(Pp.numpy(), r.G.numpy())
    if with_iou:
        iou_m = [float(iou[:, 0].sum()) / nfg_c, float(iou[:, 1].sum()) / nfg_c,
                 float((iou[:, 1] >= iou_thresh).sum()) / nfg_c]
    else:
        iou_m = [math.nan] * 3
    metrics = torch.tensor([cls_acc, head_acc, size_acc] + iou_m, dtype=F64)

    mag = _companions(r, cls, reg, lab, keep, fgi, NH, NS, nfg, nfg_c, (w_box, w_hr, w_sr, w_c))
    return SimpleNamespace(
        losses=r.losses, metrics=metrics, dcls=r.dcls, dreg=r.dreg, dreg_alt=dreg_alt, nfg=nfg,
        nkeep=int(keep.sum()), fg_rows=fgi, hc=r.hc, hres_lab=r.hres_lab, use_g=r.use_g, h_arg=h_arg, s_arg=s_arg,
        cls_arg=cls_arg, amb_flip=amb_flip, amb_cls=amb_cls & keep, amb_h=amb_h, amb_s=amb_s, iou=iou,
        dg=r.dg, df=r.df, d_c=r.d_c, d_s=r.d_s, e_h=r.e_h, D=r.D, ang=r.ang, pt=r.pt, **mag)


def _companions(r, cls, reg, lab, keep, fgi, NH, NS, nfg, nfg_c, weights):
    """Absolute-value magnitudes of what the kernel rounds: ``mag_dcls`` (N, 2), ``mag_dreg`` (N, W) and
    ``mag_loss`` (8,), each such that the kernel's fp32 error is at most a small multiple of u times it."""
    w_box, w_hr, w_sr, w_c = weights
    N, W = reg.shape
    n = len(fgi)
    u = U
    # ---- focal rows: pt from expf and one division (<= 4u relative), 1 - pt (<= 4u absolute), log(pt + eps)
    # (<= 4u absolute); scale = dpt / nfg; d = scale * pt * (delta - p)
    pt, lg, alpha = r.pt, r.lg, r.alpha
    q = 1 - pt
    inv = 1.0 / (nfg + EPS14)
    dpt_abs = alpha * (2 * q * lg.abs() + q * q / (pt + EPS14))
    # sensitivity of dpt to the errors of (1 - pt), log and 1/(pt + eps), in units of u
    ddpt = alpha * (8 * (lg.abs() + q) + 8 * q / (pt + EPS14) + 8 * q * q / (pt + EPS14))
    mag_focal_g = inv * pt * (dpt_abs * 8 + ddpt * (q + pt + 4 * u)) + inv * dpt_abs * 2.0 ** -125
    mag_dcls = torch.where(keep[:, None], mag_focal_g[:, None].expand(N, 2), torch.zeros(N, 2, dtype=F64)).clone()
    mag_focal_v = torch.where(keep, 16 * r.focal.abs() + 8 * alpha * (q * (lg.abs() + 1) + q * q), torch.zeros_like(pt))

    mag_dreg = torch.zeros(N, W, dtype=F64)
    mag_terms = [torch.zeros(0, dtype=F64)] * 6
    if n:
        o = reg.double()[fgi]
        ctr, hs, hr = o[:, :3], o[:, 3:3 + NH], o[:, 3 + NH:3 + 2 * NH]
        ss, sr = o[:, 3 + 2 * NH:3 + 2 * NH + NS], o[:, 3 + 2 * NH + NS:].reshape(n, NS, 3)
        ar = torch.arange(n)
        wb = w_box / nfg_c
        m = torch.zeros(n, W, dtype=F64)
        # centre: dv = (cgt - ref) - ctr, error <= 2u * A; gradient wb * min(d,3)/d * dv
        A = r.cgt.abs() + r.ref.abs() + ctr.abs()
        gmag = torch.where(r.d_c < 3, torch.ones_like(r.d_c), 3 / r.d_c.clamp(min=3))
        m[:, :3] += 8 * wb * gmag[:, None] * (A + A.sum(-1, keepdim=True))
        t_c = 8 * r.terms[0] + 8 * torch.clamp(r.d_c, max=3) * A.sum(-1)
        # heading / size cross-entropy: p_i = expf(s_i - mx) / sum over K terms
        def ce(s, lab_idx, K, off, w):
            mx = s.max(-1, keepdim=True).values
            p = torch.softmax(s, -1)
            onehot = torch.zeros_like(s).scatter_(1, lab_idx[:, None], 1.0)
            m[:, off:off + K] += 4 * w * (p * ((s - mx).abs() + K + 4) + onehot)
            return s.gather(1, lab_idx[:, None])[:, 0].abs() + mx[:, 0].abs() + torch.log(
                torch.exp(s - mx).sum(-1)).abs() + K + 4
        t_hc = 4 * ce(hs, r.hc, NH, 3, wb)
        t_sc = 4 * ce(ss, r.sc, NS, 3 + 2 * NH, wb)
        # heading residual: the label's fp32 evaluation (fused or not) moves e by <= 4u (shifted + bin end) / half
        half = half_bin(NH)
        e_err = 4 * (hr.gather(1, r.hc[:, None])[:, 0].abs() + r.hres_lab.double().abs()
                     + (r.shifted.double() + bin_start_f32(r.hc, NH) + 2 * half) / half)
        col_h = 3 + NH + r.hc
        m[ar, col_h] += 4 * wb * w_hr * (torch.clamp(r.e_h.abs(), max=1) + e_err)
        t_hr = 8 * r.terms[2] + 4 * torch.clamp(r.e_h.abs(), max=1) * e_err
        # size residual: dv = (sgt - ex) / ex - sr, error <= 4u * A
        A_s = (r.sgt.abs() + r.ex.abs()) / r.ex.abs() + sr[ar, r.sc].abs()
        gmag_s = torch.where(r.d_s < 1, torch.ones_like(r.d_s), 1 / r.d_s.clamp(min=1))
        col_s = 3 + 2 * NH + NS + 3 * r.sc
        for i in range(3):
            m[ar, col_s + i] += 8 * wb * w_sr * gmag_s * (A_s[:, i] + A_s.sum(-1))
        t_sr = 8 * r.terms[4] + 8 * torch.clamp(r.d_s, max=1) * A_s.sum(-1)
        # corners: every coordinate of P, G and F to <= eps (units of u): cosf / sinf within 2 ulp, the products and
        # sums of centre and half extents (<= 3 roundings of the largest coordinate), and the fp32 rounding of the
        # two angles that are computed: the decoded angle (one rounding of bin start + residual * half bin, and for a
        # wrapped angle the fp32 2 pi and the subtraction: <= u (|start| + |res| half + 2 pi wrapped + 1)) and
        # hgt + pi of the flipped box (<= u (|hgt| + pi + 1)); hgt itself is an exact input.  The unit vector of
        # corner j is then within 4 eps / |.|_j + 8, D within 2 eps + 4 D.
        ext_p, ext_g = r.sz.abs().sum(-1), r.sgt.abs().sum(-1)
        hr_sel = hr.gather(1, r.hc[:, None])[:, 0]
        wrapped = (bin_start_f32(r.hc, NH) + hr_sel * half) > math.pi
        ang_err = bin_start_f32(r.hc, NH) + hr_sel.abs() * half + 2 * math.pi * wrapped + 1
        flip_err = torch.where(r.use_g, torch.zeros_like(ang_err), r.hgt.abs() + math.pi + 1)
        eps = (3 * (r.cp.abs().max(-1).values + r.cgt.abs().max(-1).values + ext_p + ext_g) + ctr.abs().max(-1).values
               + r.ref.abs().max(-1).values + ext_p * ang_err + ext_g * flip_err)
        Pn = torch.where(r.use_g, r.dg, r.df)
        nrm_min = torch.where(r.use_g[:, None], (corners(r.cp, r.ang, r.sz) - r.G).norm(dim=-1),
                              (corners(r.cp, r.ang, r.sz) - corners(r.cgt, r.hgt + math.pi, r.sgt)).norm(dim=-1))
        unit_err = (4 * eps[:, None] / nrm_min.clamp(min=1e-30) + 8).clamp(max=1e30).sum(-1)
        gD = wb * w_c * torch.clamp(Pn, max=1) * 0.125
        gD_err = wb * w_c * 0.125 * torch.where(Pn < 1, 2 * eps + 4 * Pn, torch.full_like(Pn, 4.0))
        base = gD * unit_err + 8 * gD_err          # sum over the eight corners of the error of gD * unit vector
        L = r.sz[:, 0].abs() + r.sz[:, 1].abs()    # |d corner / d heading| <= (l + w) / 2 per coordinate pair
        m[:, :3] += base[:, None]
        m[ar, col_h] += (base + 8 * gD) * L * half
        for i in range(3):
            m[ar, col_s + i] += (base + 8 * gD) * 0.5 * r.ex[:, i].abs()
        t_co = 8 * r.terms[5] + 8 * torch.clamp(Pn, max=1) * 2 * eps
        mag_dreg[fgi] = m
        mag_terms = [t_c, t_hc, t_hr, t_sc, t_sr, t_co]
    mag_loss = torch.stack([mag_focal_v.sum()] + [t.sum() for t in mag_terms])
    return {"mag_dcls": mag_dcls, "mag_dreg": mag_dreg, "mag_loss_rows": mag_loss}


# ============================================================================ crafted inputs at the branch points
HEADING_KINDS = ("centre", "boundary", "boundary+ulp", "boundary-ulp", "zero", "+pi", "-pi", "2pi-ulp", "2pi",
                 "below-2pi", "above2pi", "near-pi", "random")


def _heading_of_kind(kind, k, NH, rng):
    """A float32 GT heading of one of HEADING_KINDS; k is the bin for the bin-relative kinds."""
    f32 = np.float32
    apc, half = f32(2 * np.pi / NH), f32(np.float32(2 * np.pi / NH) / f32(2))
    bd = f32(f32(k * apc) + half)                       # start of bin k + 1 in the shifted angle
    two_pi = f32(2 * np.pi)
    return {"centre": f32(k * apc), "boundary": bd, "boundary+ulp": np.nextafter(bd, f32(10)),
            "boundary-ulp": np.nextafter(bd, f32(-10)), "zero": f32(0), "+pi": f32(np.pi), "-pi": f32(-np.pi),
            "2pi-ulp": np.nextafter(two_pi, f32(0)), "2pi": two_pi, "below-2pi": f32(-7.3 - rng.uniform(0, 6)),
            "above2pi": f32(6.4 + rng.uniform(0, 6)), "near-pi": f32(np.pi + rng.uniform(-0.2, 0.2)),
            "random": f32(rng.uniform(-np.pi, np.pi))}[kind]


def heading_kinds(hgt, NH):
    """The HEADING_KINDS (other than "random" / "near-pi") that the float32 headings `hgt` contain."""
    f32 = np.float32
    hgt = np.asarray(hgt, f32)
    apc, half = f32(2 * np.pi / NH), f32(np.float32(2 * np.pi / NH) / f32(2))
    centres = np.array([f32(k * apc) for k in range(NH)], f32)
    bds = np.array([f32(f32(k * apc) + half) for k in range(NH)], f32)
    two_pi = f32(2 * np.pi)
    found = set()
    for h in hgt:
        if h in bds:
            found.add("boundary")
        if h in np.nextafter(bds, f32(10)):
            found.add("boundary+ulp")
        if h in np.nextafter(bds, f32(-10)):
            found.add("boundary-ulp")
        if h in centres:
            found.add("centre")
        for name, v in (("zero", f32(0)), ("+pi", f32(np.pi)), ("-pi", f32(-np.pi)),
                        ("2pi-ulp", np.nextafter(two_pi, f32(0))), ("2pi", two_pi)):
            if h == v:
                found.add(name)
        if h < -two_pi:
            found.add("below-2pi")
        if h > two_pi:
            found.add("above2pi")
    return found


def make_case(B, T2, NH, NS, seed, fg_frac=0.35, empty_frustums=True, mean_size=None):
    """Inputs of one fcn_det_loss call (numpy, the kernel's layout) whose foreground rows visit every branch point
    of the loss: focal pt -> 0 / -> 1 / 1/2, centre distance 0, < 3, 3 +- ulp, >> 3, headings at bin centres and
    boundaries +- 1 ulp, 0, +-pi, 2 pi - ulp, below -2 pi and above 2 pi, heading residuals across +-1, decoded
    angles on both sides of the pi wrap, size classes 0 and NS - 1, size residual norms 0 and across 1, rows where
    the flipped GT box is the nearer one, exact arg-max ties in the heading / size / class scores."""
    f32 = np.float32
    rng = np.random.default_rng(seed)
    N, W = B * T2, 3 + 2 * NH + 4 * NS
    if mean_size is None:
        mean_size = rng.uniform(0.5, 4.0, (NS, 3)).astype(f32)
    lab = rng.choice(np.array([-1, 0, 1]), size=(B, T2), p=[0.2, 1 - 0.2 - fg_frac, fg_frac]).astype(np.int64)
    for b in range(B):
        if not (lab[b] == 1).any():
            lab[b, (7 * b) % T2] = 1                           # every GT box is seen by a foreground row ...
    if empty_frustums and B > 2:
        lab[1] = np.where(lab[1] == 1, 0, lab[1])            # ... but one: a frustum without foreground
    # GT headings: frustum 1 (the one without foreground in a batch of more than two) takes "random", the others
    # HEADING_KINDS in turn from an offset given by the seed, so B >= len(HEADING_KINDS) + 1 visits every kind
    k = rng.integers(0, max(NH - 1, 1), B)     # not the last boundary, where the model itself fails (see above)
    heads = []
    for b in range(B):
        kind = "random" if b == 1 else HEADING_KINDS[(b - (b > 1) + seed) % len(HEADING_KINDS)]
        heads.append(_heading_of_kind(kind, int(k[b]), NH, rng))
    hgt = np.asarray(heads, f32)
    sc = rng.integers(0, NS, B).astype(np.int64)
    sc[0], sc[-1] = 0, NS - 1
    cgt = rng.normal(0, 3, (B, 3)).astype(f32)
    sgt = (mean_size[sc] * rng.uniform(0.6, 1.4, (B, 3))).astype(f32)
    cref = (cgt[:, :, None] + rng.normal(0, 1.0, (B, 3, T2))).astype(f32)

    cls = rng.normal(0, 2, (N, 2)).astype(f32)
    reg = rng.normal(0, 1, (N, W)).astype(f32)
    hc_t, hres_t, _ = angle_encode_f32(torch.from_numpy(hgt), NH)
    hc_b, hres_b = hc_t.numpy(), hres_t.numpy()
    lab_f = lab.reshape(-1)
    for r in range(N):
        b, t = divmod(r, T2)
        j = r * 7 + seed
        if lab_f[r] != -1:
            gap = [0.0, 30.0, -30.0, 100.0, -100.0, None, None, None][j % 8]
            if gap is not None:
                cls[r, 1] = f32(cls[r, 0] + gap)
        if lab_f[r] != 1:
            continue
        o = reg[r]
        # centre distance regime
        dgt = (cgt[b] - cref[b, :, t]).astype(f32)
        dirn = rng.normal(0, 1, 3)
        dirn /= np.linalg.norm(dirn)
        dist = [0.0, 0.4, 2.5, 3 * (1 - 2 ** -23), 3 * (1 + 2 ** -23), 3.7, 12.0, 1.1][j % 8]
        o[:3] = (dgt - dirn * dist).astype(f32)
        # heading scores with exact ties, residual across +-1, the flipped box
        hs = o[3:3 + NH]
        if j % 5 == 0 and NH > 1:
            m = int(np.argmax(hs))
            hs[(m + 1 + j) % NH] = hs[m]                         # exact tie, before or after the first maximum
        hc, hl = int(hc_b[b]), hres_b[b]
        if j % 4 == 0:
            hs[hc] = hs.max() + 1                                # predicted class = label
        e = [0.0, 0.3, -0.3, 0.999, -1.001, 1.5, -2.5, 0.01][(j // 3) % 8]
        o[3 + NH + hc] = f32(hl + e)
        if j % 6 == 5:
            o[3 + NH + hc] = f32(hl + NH + [0.1, -0.05][j % 2])  # decoded heading ~ GT + pi: flipped box nearer
        # size scores with ties, size residual norm 0 / < 1 / > 1
        ss = o[3 + 2 * NH:3 + 2 * NH + NS]
        if j % 3 == 1 and NS > 1:
            m = int(np.argmax(ss))
            ss[(m + 1 + j) % NS] = ss[m]
        if j % 4 == 1:
            ss[sc[b]] = ss.max() + 1
        ex = mean_size[sc[b]]
        lbl = ((sgt[b] - ex) / ex).astype(f32)
        sdir = rng.normal(0, 1, 3)
        sdir /= np.linalg.norm(sdir)
        sdist = [0.0, 0.3, 0.95, 1.6][(j // 2) % 4]
        base = 3 + 2 * NH + NS + 3 * sc[b]
        o[base:base + 3] = (lbl - sdir * sdist).astype(f32)
    reg = reg.astype(f32)
    return {"cls": cls, "reg": reg, "cls_label": lab, "center_ref2": cref, "box3d_center": cgt,
            "box3d_heading": hgt, "box3d_size": sgt, "size_class": sc, "mean_size": mean_size.astype(f32)}
