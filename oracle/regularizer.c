/*
 * oracle/regularizer.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C, fp32 by default, fp64 with -DORACLE_F64) of the image-space regularisers of the reference,
 * render/regularizer.py:15-49 (luma :15-16, value :17-18, chroma_loss :20-24, shading_loss :27-38, material_smoothness_grad :44-49) and
 * render/util.py:95-99 (_rgb_to_srgb), forward and backward, in the operation order of nvdiffrecmc_b200/csrc/regularizer.cu (the contract
 * is stated there).  Operands are contiguous [n,4]; gradients are full [n,4].  The sums are carried in double in pixel order; each mean
 * is rounded to `real` once.
 *
 * PARITY PIN: the reference's own three functions, frozen in tests/golden/ref_regularizer.npz (tests/golden/make_regularizer_golden.py).
 * The per-pixel terms of material_smoothness_grad and chroma_loss use only + - * / max and abs, so with -ffp-contract=off the fp32 build
 * equals the kernels' explicitly rounded gradients bit for bit.  Only tests/ may load this library; the product never does.
 */
#include <math.h>
#include <stddef.h>

#ifdef ORACLE_F64
typedef double real;
#define R_POW(x, y) pow(x, y)
#define R_FABS(x) fabs(x)
#define R_LOG(x) log(x)
#else
typedef float real;
#define R_POW(x, y) powf(x, y)
#define R_FABS(x) fabsf(x)
#define R_LOG(x) logf(x)
#endif
#define RC(x) ((real)(x))

int reg_sizeof_real(void) { return (int)sizeof(real); }

#define REG_EPS RC(0.001f)
#define REG_SRGB_T RC(0.0031308f)
#ifdef ORACLE_F64
#define REG_SRGB_E (1.0 / 2.4)
#define REG_SRGB_EM1 (1.0 / 2.4 - 1.0)
#else
#define REG_SRGB_E ((float)(1.0 / 2.4))
#define REG_SRGB_EM1 ((float)(1.0 / 2.4 - 1.0))
#endif
static inline real reg_luma(const real *x) { return ((x[0] + x[1]) + x[2]) / RC(3); }                           /* regularizer.py:15-16 */
static inline int reg_argmax3(const real *x)     /* torch.max(dim) (regularizer.py:17-18): the first NaN, else the first maximal channel */
{
    int i = 0;
    real m = x[0];
    if (x[1] > m || (x[1] != x[1] && m == m)) { i = 1; m = x[1]; }
    if (x[2] > m || (x[2] != x[2] && m == m)) i = 2;
    return i;
}
static inline real reg_clamp_min(real x, real lo) { return x < lo ? lo : x; }                   /* torch.clamp / clip: NaN passes */
static inline real reg_clamp_lh(real x, real lo, real hi) { return x < lo ? lo : (x > hi ? hi : x); }
static inline real reg_sgn(real x) { return x > 0 ? RC(1) : (x < 0 ? RC(-1) : RC(0)); }           /* torch.sign: 0 for +-0 and NaN */
static inline real reg_srgb(real f)                                                                 /* util.py:95-96 */
{
    return f <= REG_SRGB_T ? f * RC(12.92f) : R_POW(reg_clamp_min(f, REG_SRGB_T), REG_SRGB_E) * RC(1.055f) - RC(0.055f);
}
static inline real reg_log_srgb(real x) { return reg_srgb(R_LOG(reg_clamp_lh(x, RC(0), RC(65535.0f)) + RC(1))); }   /* regularizer.py:33-34 */

/* shading_loss (regularizer.py:27-38): loss[0]; means = (mean(diffuse luma), mean(specular luma)), as the kernel saves them */
void reg_shading_loss_fwd(int n, const real *diffuse, const real *specular, const real *ref, real ld, real ls, real *loss, real *means)
{
    double se = 0, ss = 0, sd = 0;
    for (int i = 0; i < n; ++i) {
        const real *d = diffuse + 4 * (size_t)i, *s = specular + 4 * (size_t)i, *r = ref + 4 * (size_t)i;
        const real dl = reg_luma(d), sl = reg_luma(s), a = r[3], sum = dl + sl;
        const real img = reg_log_srgb(sum * a), tgt = reg_log_srgb(r[reg_argmax3(r)] * a);
        const real e = (R_FABS(img - tgt) * dl) / reg_clamp_min(sum, REG_EPS);
        se += e; ss += sl; sd += dl;
    }
    const real me = (real)(se / n), ms = (real)(ss / n), md = (real)(sd / n);     /* 3N copies: 3 sum / 3N */
    loss[0] = me * ld + (ms / reg_clamp_min(md, REG_EPS)) * ls;
    means[0] = md; means[1] = ms;
}
/* The adjoint of reg_shading_loss_fwd for the upstream gradient G of the loss, given its means */
void reg_shading_loss_bwd(int n, const real *diffuse, const real *specular, const real *ref, real ld, real ls, const real *means, real G,
                          real *d_diffuse, real *d_specular)
{
    const real n3 = (real)(3 * (long long)n);
    const real g_e = (G * ld) / n3;
    const real md = means[0], ms = means[1], cmd = reg_clamp_min(md, REG_EPS), gq = G * ls;
    const real g_ms = gq / cmd, g_cmd = -gq * ((ms / cmd) / cmd);       /* mean(sl) / clamp(mean(dl), eps) */
    const real g_md = md >= REG_EPS ? g_cmd : RC(0);
    const real g_slm = g_ms / n3, g_dlm = g_md / n3;
    for (int i = 0; i < n; ++i) {
        const real *d = diffuse + 4 * (size_t)i, *s = specular + 4 * (size_t)i, *r = ref + 4 * (size_t)i;
        const real dl = reg_luma(d), sl = reg_luma(s), a = r[3], sum = dl + sl, x = sum * a;
        const real u = reg_clamp_lh(x, RC(0), RC(65535.0f)), L = R_LOG(u + RC(1));
        const real img = reg_srgb(L), tgt = reg_log_srgb(r[reg_argmax3(r)] * a);
        const real diff = img - tgt, ad = R_FABS(diff), cs = reg_clamp_min(sum, REG_EPS), num = ad * dl;
        const real g_num = g_e / cs, g_cs = -g_e * ((num / cs) / cs);   /* e = num / cs */
        const real g_ad = g_num * dl, g_dl1 = g_num * ad;                 /* num = |img - tgt| * dl */
        const real g_s2 = sum >= REG_EPS ? g_cs : RC(0);                  /* cs = clamp(dl + sl, eps) */
        const real g_img = g_ad * reg_sgn(diff);
        real g_L;                                                         /* where(L <= T, L * 12.92, pow(clamp(L, T), E) * 1.055 - 0.055) */
        if (L <= REG_SRGB_T) g_L = g_img * RC(12.92f);
        else g_L = L >= REG_SRGB_T ? (g_img * RC(1.055f)) * (REG_SRGB_E * R_POW(L, REG_SRGB_EM1)) : RC(0);
        const real g_u = g_L / (u + RC(1));                               /* log(u + 1) */
        const real g_x = (x >= 0 && x <= RC(65535.0f)) ? g_u : RC(0);     /* clamp(x, 0, 65535) */
        const real g_s1 = g_x * a;                                        /* x = (dl + sl) * alpha */
        const real g_dl = ((g_dl1 + g_s2) + g_s1) + g_dlm, g_sl = (g_s2 + g_s1) + g_slm;
        const real gd = ((g_dl + g_dl) + g_dl) / RC(3), gs = ((g_sl + g_sl) + g_sl) / RC(3);     /* repeat: three copies; luma: / 3 */
        real *od = d_diffuse + 4 * (size_t)i, *os = d_specular + 4 * (size_t)i;
        od[0] = od[1] = od[2] = gd; od[3] = 0;
        os[0] = os[1] = os[2] = gs; os[3] = 0;
    }
}

/* material_smoothness_grad (regularizer.py:44-49) */
void reg_material_smoothness_grad_fwd(int n, const real *kd, const real *ks, const real *nrm, real lkd, real lks, real lnrm, real *loss)
{
    double s0 = 0, s1 = 0, s2 = 0;
    for (int i = 0; i < n; ++i) {
        const real *k = kd + 4 * (size_t)i, *s = ks + 4 * (size_t)i, *m = nrm + 4 * (size_t)i;
        s0 += (double)(reg_luma(k) * k[3]);
        s1 += ((double)(s[0] * s[3]) + (double)(s[1] * s[3])) + (double)(s[2] * s[3]);
        s2 += ((double)(m[0] * m[3]) + (double)(m[1] * m[3])) + (double)(m[2] * m[3]);
    }
    const real m0 = (real)(s0 / n), m1 = (real)(s1 / (3.0 * n)), m2 = (real)(s2 / (3.0 * n));
    loss[0] = (m0 * lkd + m1 * lks) + m2 * lnrm;
}
void reg_material_smoothness_grad_bwd(int n, const real *kd, const real *ks, const real *nrm, real lkd, real lks, real lnrm, real G,
                                      real *d_kd, real *d_ks, real *d_nrm)
{
    const real n1 = (real)n, n3 = (real)(3 * (long long)n);
    const real g1 = (G * lkd) / n1, g2 = (G * lks) / n3, g3 = (G * lnrm) / n3;
    for (int i = 0; i < n; ++i) {
        const real *k = kd + 4 * (size_t)i, *s = ks + 4 * (size_t)i, *m = nrm + 4 * (size_t)i;
        real *gk = d_kd + 4 * (size_t)i, *gs = d_ks + 4 * (size_t)i, *gm = d_nrm + 4 * (size_t)i;
        const real gl = (g1 * k[3]) / RC(3);                              /* (k0 + k1 + k2) / 3 * k3 */
        gk[0] = gk[1] = gk[2] = gl; gk[3] = g1 * reg_luma(k);
        gs[0] = gs[1] = gs[2] = g2 * s[3]; gs[3] = ((g2 * s[0]) + (g2 * s[1])) + (g2 * s[2]);     /* rgb * alpha, alpha broadcast */
        gm[0] = gm[1] = gm[2] = g3 * m[3]; gm[3] = ((g3 * m[0]) + (g3 * m[1])) + (g3 * m[2]);
    }
}

/* chroma_loss (regularizer.py:20-24) */
static inline void reg_chroma_t(const real *k, const real *r, real *t)
{
    const real ck = reg_clamp_min(k[reg_argmax3(k)], REG_EPS), cr = reg_clamp_min(r[reg_argmax3(r)], REG_EPS);
    for (int c = 0; c < 3; ++c) t[c] = (k[c] / ck - r[c] / cr) * r[3];
}
void reg_chroma_loss_fwd(int n, const real *kd, const real *ref, real lc, real *loss)
{
    double s = 0;
    for (int i = 0; i < n; ++i) {
        real t[3];
        reg_chroma_t(kd + 4 * (size_t)i, ref + 4 * (size_t)i, t);
        s += ((double)R_FABS(t[0]) + (double)R_FABS(t[1])) + (double)R_FABS(t[2]);
    }
    loss[0] = (real)(s / (3.0 * n)) * lc;
}
void reg_chroma_loss_bwd(int n, const real *kd, const real *ref, real lc, real G, real *d_kd)
{
    const real ge = (G * lc) / (real)(3 * (long long)n);
    for (int i = 0; i < n; ++i) {
        const real *k = kd + 4 * (size_t)i, *r = ref + 4 * (size_t)i;
        real *gk = d_kd + 4 * (size_t)i;
        const int ik = reg_argmax3(k);
        const real vk = k[ik], ck = reg_clamp_min(vk, REG_EPS);
        real t[3], gdir[3], gck = 0;
        reg_chroma_t(k, r, t);
        for (int c = 0; c < 3; ++c) {
            const real g_opt = (ge * reg_sgn(t[c])) * r[3];                 /* |.|, then * ref.w; the subtraction passes it on */
            gdir[c] = g_opt / ck;                                           /* kd_c / ck */
            const real gc = -g_opt * ((k[c] / ck) / ck);
            gck = c == 0 ? gc : gck + gc;                                   /* repeat: the three copies of value(kd) */
        }
        const real gv = vk >= REG_EPS ? gck : RC(0);                        /* clip(value, eps) */
        for (int c = 0; c < 3; ++c) gk[c] = gdir[c] + (c == ik ? gv : RC(0));   /* max: the selected channel */
        gk[3] = 0;
    }
}
