/* taps.c -- CPU oracle of the jittered regulariser taps (TEST INFRASTRUCTURE, not product code).
 *
 * A plain-C restatement of the contract in nvdiffrecmc_b200/csrc/taps.cu, written independently of the kernels: the reference's
 * kd_grad / ks_grad / normal_grad / perturbed_nrm_grad of shade() (render/render.py:50-97, alpha appended as at :151-153,161-163), forward
 * and backward, texture path (tapped kd / ks, grad weight) and MLP path (kd_jitter / ks_jitter, no grad weight).  The tap is texture.c's
 * 'linear' / 'clamp' look-up (included below rather than copied), with the coordinate u * W - 0.5 of the contract.
 * Operands are contiguous: rast [B,H,W,4], jitter [B,H,W,2], kd / kd_jitter [B,H,W,Ckd], ks / ks_jitter / gb_normal / perturbed_nrm
 * [B,H,W,3]; outputs kd_grad [B,H,W,Ckd+1] and [B,H,W,4] for the others; gradients d kd [B,H,W,Ckd], d ks / d normal / d perturbed
 * [B,H,W,3], accumulated as a sequential scatter in pixel order (the pixel's direct terms, then its four tap terms per tapped image);
 * d kd_jitter / d ks_jitter overwritten (one writer).
 * `terms` (test-only, oracle.TERMS) applies to the scattered gradients: 0 sums the terms, 1 their absolute values, 2 counts the non-zero
 * ones.  Every component of a direct term is a term of its own there (kd's alpha gets up to five: -g_d, then the alpha gradient of each
 * buffer), so the statistics bound any order of summing them; mode 0 adds the direct term as the kernels form it, in the contract's order.
 * Two builds (oracle/taps.py), as texture.c: fp32 (compared bit for bit with the kernels' forward and terms) and fp64 (-DORACLE_F64;
 * checked by finite differences).  Compile with -ffp-contract=off.
 */
#include "texture.c"

#include <stdlib.h>

int taps_sizeof_real(void) { return (int)sizeof(real); }

#define SN_EPS ((real)1e-20f)

static real r_abs(real x) { return (real)fabs((double)x); }
static real sgn(real x) { return x > 0 ? (real)1 : (x < 0 ? (real)-1 : (real)0); }      /* torch.sign: 0 for +-0 and NaN */

/* texel offsets of the one-channel taps scaled to an image of C channels */
static taps_t scaled(const taps_t *t1, int C)
{
    taps_t t = *t1;
    for (int j = 0; j < 4; ++j) t.o[j] *= C;
    return t;
}

static real sn_len(const real *x, real *d)
{
    *d = (x[0] * x[0] + x[1] * x[1]) + x[2] * x[2];
    return R_SQRT(*d < SN_EPS ? SN_EPS : *d);
}

static void sn(const real *x, real *y)
{
    real d;
    const real l = sn_len(x, &d);
    for (int c = 0; c < 3; ++c) y[c] = x[c] / l;
}

static void sn_bwd(const real *x, const real *gy, real *gx)
{
    real d;
    const real l = sn_len(x, &d);
    real gl = -gy[0] * ((x[0] / l) / l);
    for (int c = 1; c < 3; ++c) gl = gl + -gy[c] * ((x[c] / l) / l);
    const real gd = d >= SN_EPS ? gl / ((real)2 * l) : (real)0;
    for (int c = 0; c < 3; ++c) gx[c] = gy[c] / l + (gd * x[c] + gd * x[c]);
}

/* a = sn(tp) + sn(pv); returns sn(a)_2 */
static real pert_z(const real *tp, const real *pv, real *a)
{
    real s0[3], s1[3], d;
    sn(tp, s0);
    sn(pv, s1);
    for (int c = 0; c < 3; ++c) a[c] = s0[c] + s1[c];
    return a[2] / sn_len(a, &d);
}

typedef struct {
    int B, H, W, Ckd;
    const real *rast, *jitter, *kd, *ks, *nrm, *pn, *kdj, *ksj;
    real *mask;
} args_t;

static args_t mk(int B, int H, int W, int Ckd, const real *rast, const real *jitter, const real *kd, const real *ks, const real *nrm,
                 const real *pn, const real *kdj, const real *ksj)
{
    args_t a = {B, H, W, Ckd, rast, jitter, kd, ks, nrm, pn, kdj, ksj, NULL};
    const int64_t n = (int64_t)B * H * W;
    a.mask = (real *)malloc(sizeof(real) * (size_t)(n ? n : 1));
    for (int64_t i = 0; i < n; ++i) a.mask[i] = rast[4 * i + 3] > 0 ? (real)1 : (real)0;
    return a;
}

/* one-channel taps of pixel i and its grad weight */
static taps_t pixel_tap(const args_t *a, int64_t i, real *gw)
{
    const int b = (int)(i / ((int64_t)a->H * a->W));
    const taps_t t = taps(1, a->H, a->W, (int64_t)a->H * a->W, b, a->jitter[2 * i], a->jitter[2 * i + 1], 1);
    *gw = a->mask[i] * bilerp(a->mask, &t, 0);
    return t;
}

void taps_fwd(int B, int H, int W, int Ckd, const real *rast, const real *jitter, const real *kd, const real *ks, const real *nrm, const real *pn,
              const real *kdj, const real *ksj, real *kd_grad, real *ks_grad, real *nrm_grad, real *pn_grad)
{
    args_t a = mk(B, H, W, Ckd, rast, jitter, kd, ks, nrm, pn, kdj, ksj);
    const int64_t n = (int64_t)B * H * W;
    for (int64_t i = 0; i < n; ++i) {
        real gw;
        const taps_t t1 = pixel_tap(&a, i, &gw);
        const taps_t tk = scaled(&t1, Ckd), t3 = scaled(&t1, 3);
        const real alpha = Ckd == 4 ? kd[4 * i + 3] : (real)1;
        for (int c = 0; c < Ckd; ++c) {
            const real v = kd[i * Ckd + c];
            kd_grad[i * (Ckd + 1) + c] = kdj ? r_abs(kdj[i * Ckd + c] - v) : r_abs(bilerp(kd, &tk, c) - v) * gw;
        }
        kd_grad[i * (Ckd + 1) + Ckd] = alpha;
        for (int c = 0; c < 3; ++c) {
            const real v = ks[3 * i + c], m = c == 0 ? (real)0 : (real)1;
            ks_grad[4 * i + c] = ksj ? r_abs(ksj[3 * i + c] - v) * m : (r_abs(bilerp(ks, &t3, c) - v) * m) * gw;
            nrm_grad[4 * i + c] = r_abs(bilerp(nrm, &t3, c) - nrm[3 * i + c]) * gw;
        }
        ks_grad[4 * i + 3] = nrm_grad[4 * i + 3] = alpha;
        if (pn) {
            real tp[3], av[3];
            for (int c = 0; c < 3; ++c) tp[c] = bilerp(pn, &t3, c);
            const real g = ((real)1 - pert_z(tp, pn + 3 * i, av)) * gw;
            for (int c = 0; c < 3; ++c) pn_grad[4 * i + c] = g;
            pn_grad[4 * i + 3] = alpha;
        }
    }
    free(a.mask);
}

/* dst += the direct term of n components (mode 0: their sum in order, one addition; else one term each) */
static void add_direct(real *dst, const real *comp, int n, int terms)
{
    if (terms == 0) {
        real s = comp[0];
        for (int k = 1; k < n; ++k) s = s + comp[k];
        *dst = *dst + s;
    } else {
        for (int k = 0; k < n; ++k) *dst = *dst + term_of(comp[k], terms);
    }
}

/* the four tap terms w_ij * g_c of C channels into img's gradient */
static void add_taps(real *d, const taps_t *t, int C, const real *g, int terms)
{
    const real ox = (real)1 - t->fx, oy = (real)1 - t->fy;
    const real w[4] = {oy * ox, oy * t->fx, t->fy * ox, t->fy * t->fx};
    for (int j = 0; j < 4; ++j)
        for (int c = 0; c < C; ++c) d[t->o[j] + c] = d[t->o[j] + c] + term_of(w[j] * g[c], terms);
}

void taps_bwd(int B, int H, int W, int Ckd, const real *rast, const real *jitter, const real *kd, const real *ks, const real *nrm, const real *pn,
              const real *kdj, const real *ksj, const real *g_kd, const real *g_ks, const real *g_n, const real *g_p, real *d_kd, real *d_ks,
              real *d_n, real *d_p, real *d_kdj, real *d_ksj, int terms)
{
    args_t a = mk(B, H, W, Ckd, rast, jitter, kd, ks, nrm, pn, kdj, ksj);
    const int64_t n = (int64_t)B * H * W;
    const int mlp = kdj != NULL;
    for (int64_t i = 0; i < n; ++i) {
        real gw;
        const taps_t t1 = pixel_tap(&a, i, &gw);
        const taps_t tk = scaled(&t1, Ckd), t3 = scaled(&t1, 3);
        const real *Gk = g_kd + i * (Ckd + 1), *Gs = g_ks + 4 * i, *Gn = g_n + 4 * i, *Gp = pn ? g_p + 4 * i : NULL;
        real tg[4], comp[5];
        /* kd */
        for (int c = 0; c < Ckd; ++c) {
            const real v = kd[i * Ckd + c];
            const real u = mlp ? kdj[i * Ckd + c] : bilerp(kd, &tk, c);
            tg[c] = (mlp ? Gk[c] : Gk[c] * gw) * sgn(u - v);
            int k = 0;
            comp[k++] = -tg[c];
            if (c == 3) {
                comp[k++] = Gk[4];
                comp[k++] = Gs[3];
                comp[k++] = Gn[3];
                if (pn) comp[k++] = Gp[3];
            }
            add_direct(d_kd + i * Ckd + c, comp, k, terms);
        }
        if (mlp) {
            for (int c = 0; c < Ckd; ++c) d_kdj[i * Ckd + c] = tg[c];
        } else {
            add_taps(d_kd, &tk, Ckd, tg, terms);
        }
        /* ks */
        for (int c = 0; c < 3; ++c) {
            const real v = ks[3 * i + c], m = c == 0 ? (real)0 : (real)1;
            const real u = mlp ? ksj[3 * i + c] : bilerp(ks, &t3, c);
            tg[c] = (mlp ? Gs[c] * m : (Gs[c] * gw) * m) * sgn(u - v);
            comp[0] = -tg[c];
            add_direct(d_ks + 3 * i + c, comp, 1, terms);
        }
        if (mlp) {
            for (int c = 0; c < 3; ++c) d_ksj[3 * i + c] = tg[c];
        } else {
            add_taps(d_ks, &t3, 3, tg, terms);
        }
        /* normal */
        for (int c = 0; c < 3; ++c) {
            tg[c] = (Gn[c] * gw) * sgn(bilerp(nrm, &t3, c) - nrm[3 * i + c]);
            comp[0] = -tg[c];
            add_direct(d_n + 3 * i + c, comp, 1, terms);
        }
        add_taps(d_n, &t3, 3, tg, terms);
        /* perturbed normal */
        if (pn) {
            real tp[3], av[3], ga[3], gt[3], gd[3];
            for (int c = 0; c < 3; ++c) tp[c] = bilerp(pn, &t3, c);
            pert_z(tp, pn + 3 * i, av);
            const real gy[3] = {0, 0, -((Gp[0] * gw + Gp[1] * gw) + Gp[2] * gw)};
            sn_bwd(av, gy, ga);
            sn_bwd(tp, ga, gt);
            sn_bwd(pn + 3 * i, ga, gd);
            for (int c = 0; c < 3; ++c) add_direct(d_p + 3 * i + c, gd + c, 1, terms);
            add_taps(d_p, &t3, 3, gt, terms);
        }
    }
    free(a.mask);
}
