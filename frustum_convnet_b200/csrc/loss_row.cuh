// Body of the fused loss's row kernels (csrc/loss.cu), included inside det_loss_rows_kernel and
// det_loss_rows_det_kernel: with a, counts, N, NH, NS, W, r and the zeroed float v[A_N] in scope, row r's loss terms
// go to v and its logit gradients to a.dcls / a.dreg.  One body for both kernels; an inlined function would change
// the register allocation, and so the code, of the default kernel.
    if (r < N) {
        const int b = r / a.T2, t = r - b * a.T2;
        const long long lab = a.cls_label[r];
        const float nfg = fmaxf(counts[0], 1.f), inv_fg = 1.f / nfg;
        const float *cl = a.cls + (size_t)r * 2, *o = a.reg + (size_t)r * W;
        float *dc = a.dcls + (size_t)r * 2, *dr = a.dreg + (size_t)r * W;
        for (int i = 0; i < W; ++i) dr[i] = 0.f;
        // ---------------- focal classification loss (all rows with label != -1), common.py:217-232
        float p0, p1;
        softmax2(cl, p0, p1);
        float d0 = 0.f, d1 = 0.f;
        if (lab != -1) {
            const int tl = lab >= 1 ? 1 : 0;
            const float alpha = tl == 0 ? 0.75f : 0.25f;
            const float pt = tl == 0 ? p0 : p1;
            float lg;
            v[A_CLS] = focal_term(pt, alpha, lg);
            // d/dpt [ -alpha (1-pt)^2 log(pt+eps) ]
            const float dpt = -alpha * (-2.f * (1.f - pt) * lg + (1.f - pt) * (1.f - pt) / (pt + 1e-14f));
            const float scale = dpt / (counts[0] + 1e-14f);           // loss.sum() / (num_fg + 1e-14)
            // dpt/dc_k = pt (delta_kt - p_k)
            d0 = scale * pt * ((tl == 0 ? 1.f : 0.f) - p0);
            d1 = scale * pt * ((tl == 1 ? 1.f : 0.f) - p1);
            v[A_CLSACC] = ((p1 > p0 ? 1 : 0) == (int)lab) ? 1.f : 0.f;   // argmax: first maximum on ties
        }
        dc[0] = d0; dc[1] = d1;
        if (lab == 1) {
            // ---------------- labels of this frustum, box_transform.py:15-25
            const float cgt[3] = {a.box3d_center[b * 3], a.box3d_center[b * 3 + 1], a.box3d_center[b * 3 + 2]};
            const float ref[3] = {a.center_ref2[((size_t)b * 3 + 0) * a.T2 + t], a.center_ref2[((size_t)b * 3 + 1) * a.T2 + t],
                                  a.center_ref2[((size_t)b * 3 + 2) * a.T2 + t]};
            const float hgt = a.box3d_heading[b];
            const float sgt[3] = {a.box3d_size[b * 3], a.box3d_size[b * 3 + 1], a.box3d_size[b * 3 + 2]};
            const int sc = (int)a.size_class[b];
            const float apc = heading_bin_width(NH);
            float hres_lab;
            const int hc = angle_encode(hgt, NH, hres_lab);
            const float *ctr = o, *hs = o + 3, *hr = hs + NH, *ss = hr + NH, *sr = ss + NS;
            float ex[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) ex[i] = a.mean_size[sc * 3 + i];
            const float wb = a.w_box * inv_fg;                         // weight of a box term of ONE fg row in the total
            // ---------------- centre Huber loss (delta 3) on the distance
            {
                float dv[3], d2 = 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i) { dv[i] = (cgt[i] - ref[i]) - ctr[i]; d2 += dv[i] * dv[i]; }
                const float d = sqrtf(d2);
                v[A_CENTER] = huber(d, 3.f);
                const float gd = d > 0.f ? fminf(d, 3.f) / d : 0.f;   // dh/dd * 1/d
#pragma unroll
                for (int i = 0; i < 3; ++i) dr[i] += wb * gd * (-dv[i]);
            }
            // ---------------- heading class CE + residual Huber (delta 1)
            int h_arg = 0;
            {
                float mx;
                const float sum = softmax_denom(hs, NH, mx);
                v[A_HCLS] = -(hs[hc] - mx - logf(sum));
                float best = -1.f;
                for (int i = 0; i < NH; ++i) {
                    const float p = expf(hs[i] - mx) / sum;
                    dr[3 + i] += wb * (p - (i == hc ? 1.f : 0.f));
                    if (p > best) { best = p; h_arg = i; }
                }
                v[A_HACC] = h_arg == hc ? 1.f : 0.f;
                const float e = hr[hc] - hres_lab;
                v[A_HRES] = huber(fabsf(e), 1.f);
                dr[3 + NH + hc] += wb * a.w_head_reg * fmaxf(-1.f, fminf(1.f, e));
            }
            // ---------------- size class CE + residual Huber (delta 1) on the norm
            int s_arg = 0;
            {
                float mx;
                const float sum = softmax_denom(ss, NS, mx);
                v[A_SCLS] = -(ss[sc] - mx - logf(sum));
                float best = -1.f;
                for (int i = 0; i < NS; ++i) {
                    const float p = expf(ss[i] - mx) / sum;
                    dr[3 + 2 * NH + i] += wb * (p - (i == sc ? 1.f : 0.f));
                    if (p > best) { best = p; s_arg = i; }
                }
                v[A_SACC] = s_arg == sc ? 1.f : 0.f;
                float dv[3], d2 = 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i) { dv[i] = (sgt[i] - ex[i]) / ex[i] - sr[sc * 3 + i]; d2 += dv[i] * dv[i]; }
                const float d = sqrtf(d2);
                v[A_SRES] = huber(d, 1.f);
                const float gd = d > 0.f ? fminf(d, 1.f) / d : 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i) dr[3 + 2 * NH + NS + sc * 3 + i] += wb * a.w_size_reg * gd * (-dv[i]);
            }
            // ---------------- corner loss (det_base.py:449-461): predicted box with the GT class labels
            {
                const float cp[3] = {ref[0] + ctr[0], ref[1] + ctr[1], ref[2] + ctr[2]};
                const float ang = angle_decode(hc, hr[hc], apc);
                float sz[3];
#pragma unroll
                for (int i = 0; i < 3; ++i) sz[i] = sr[sc * 3 + i] * ex[i] + ex[i];
                float P[24], G[24], F[24];
                corners_of(cp, ang, sz, P);
                corners_of(cgt, hgt, sgt, G);
                corners_of(cgt, hgt + LOSS_PI, sgt, F);
                float dg = 0.f, df = 0.f, ng[8], nf[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float a2 = 0.f, b2 = 0.f;
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        const float x = P[3 * j + k] - G[3 * j + k], y = P[3 * j + k] - F[3 * j + k];
                        a2 += x * x; b2 += y * y;
                    }
                    ng[j] = sqrtf(a2); nf[j] = sqrtf(b2);
                    dg += ng[j]; df += nf[j];
                }
                dg *= 0.125f; df *= 0.125f;
                const bool use_g = dg <= df;
                const float D = use_g ? dg : df;
                v[A_CORNER] = huber(D, 1.f);
                const float gD = wb * a.w_corner * fminf(D, 1.f) * 0.125f;   // dL/dD * dD/d||.||_j
                const float cs = cosf(ang), sn = sinf(ang);
                const float sx[8] = {1, 1, -1, -1, 1, 1, -1, -1}, sy[8] = {1, 1, 1, 1, -1, -1, -1, -1},
                            szz[8] = {1, -1, -1, 1, 1, -1, -1, 1};
                float gc[3] = {0.f, 0.f, 0.f}, gth = 0.f, gl = 0.f, gw = 0.f, gh = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float nrm = use_g ? ng[j] : nf[j];
                    if (!(nrm > 0.f)) continue;
                    const float *Tg = use_g ? G : F;
                    const float gx = gD * (P[3 * j] - Tg[3 * j]) / nrm, gy = gD * (P[3 * j + 1] - Tg[3 * j + 1]) / nrm,
                                gz = gD * (P[3 * j + 2] - Tg[3 * j + 2]) / nrm;
                    gc[0] += gx; gc[1] += gy; gc[2] += gz;
                    const float x = sx[j] * sz[0] * 0.5f, z = szz[j] * sz[1] * 0.5f;
                    gth += gx * (-sn * x + cs * z) + gz * (-cs * x - sn * z);
                    gl += (gx * cs - gz * sn) * sx[j] * 0.5f;
                    gw += (gx * sn + gz * cs) * szz[j] * 0.5f;
                    gh += gy * sy[j] * 0.5f;
                }
#pragma unroll
                for (int i = 0; i < 3; ++i) dr[i] += gc[i];
                dr[3 + NH + hc] += gth * (apc * 0.5f);
                dr[3 + 2 * NH + NS + sc * 3 + 0] += gl * ex[0];
                dr[3 + 2 * NH + NS + sc * 3 + 1] += gw * ex[1];
                dr[3 + 2 * NH + NS + sc * 3 + 2] += gh * ex[2];
                // ---------------- IoU metrics: predicted box with the PREDICTED class labels (det_base.py:488-500)
                if (a.with_iou) {
                    const float angp = angle_decode(h_arg, hr[h_arg], apc);
                    float szp[3];
#pragma unroll
                    for (int i = 0; i < 3; ++i) szp[i] = sr[s_arg * 3 + i] * a.mean_size[s_arg * 3 + i] + a.mean_size[s_arg * 3 + i];
                    corners_of(cp, angp, szp, P);
                    float iou[2];
                    rbbox_iou_pair(P, G, iou);
                    v[A_IOU2] = iou[0];
                    v[A_IOU3] = iou[1];
                    v[A_IOUGT] = iou[1] >= a.iou_thresh ? 1.f : 0.f;
                }
            }
        }
    }
