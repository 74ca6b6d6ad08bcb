/* mipchain.c -- CPU oracle of Texture2D's automatic mip chain (TEST INFRASTRUCTURE, not product code).
 *
 * A plain-C restatement of the chain contract in nvdiffrecmc_b200/csrc/texture.cu, written independently of the kernels:
 *   the chain forward (render/texture.py:20-23, avg_pool2d by 2 x 2), its backward folded over every level (texture.py:25-30: a quarter of
 *   the coarser gradient sampled bilinearly with clamped borders at the finer texels' centres, added to the finer level's own gradient),
 *   and Texture2D's in-place clamp_ / normalize_ (texture.py:89-100, util.safe_normalize).
 * Levels are dense [Bt, h[k], w[k], C]; a chain has h[k] = h[k-1] / 2, w alike.
 * Two builds of this file (oracle/mipchain.py): fp32 (`real` = float; compared bit for bit with the kernels) and fp64 (-DORACLE_F64).
 * Compile with -ffp-contract=off: every product and sum is one IEEE round-to-nearest operation, in the order the contract writes it.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#ifdef ORACLE_F64
typedef double real;
#define R_FLOOR floor
#define R_SQRT sqrt
#else
typedef float real;
#define R_FLOOR floorf
#define R_SQRT sqrtf
#endif

int mip_sizeof_real(void) { return (int)sizeof(real); }

/* the clamped taps of one axis at texel-space coordinate x of a level n texels wide, and the fraction */
static void clamped_axis(real x, int n, int64_t *i0, int64_t *i1, real *fr)
{
    const real f = R_FLOOR(x);
    *fr = x - f;
    const int64_t x0 = (int64_t)f, x1 = x0 + 1;
    *i0 = x0 < 0 ? 0 : (x0 > n - 1 ? n - 1 : x0);
    *i1 = x1 < 0 ? 0 : (x1 > n - 1 ? n - 1 : x1);
}

/* levels 1 .. n_levels-1 of level 0: the 2 x 2 average, summed from 0 in row-major order and divided by 4 (avg_pool2d) */
void mip_fwd(int n_levels, int C, int Bt, real *const *lv, const int *h, const int *w)
{
    for (int k = 1; k < n_levels; ++k)
        for (int b = 0; b < Bt; ++b) {
            const real *src = lv[k - 1] + (int64_t)b * h[k - 1] * w[k - 1] * C;
            real *dst = lv[k] + (int64_t)b * h[k] * w[k] * C;
            for (int y = 0; y < h[k]; ++y)
                for (int x = 0; x < w[k]; ++x)
                    for (int c = 0; c < C; ++c) {
                        real s = 0;
                        for (int dy = 0; dy < 2; ++dy)
                            for (int dx = 0; dx < 2; ++dx) s = s + src[((int64_t)(2 * y + dy) * w[k - 1] + 2 * x + dx) * C + c];
                        dst[((int64_t)y * w[k] + x) * C + c] = s / (real)4;
                    }
        }
}

/* the gradient of level 0 from the gradients g[k] of every level (null = none), in the reference's order: the coarsest level with a
 * gradient passes it down; each pool's backward samples a quarter of the coarser gradient bilinearly, clamped, at the finer texels'
 * centres (the exact coarse coordinate i / 2 - 0.25, where the reference's torch.linspace grid can be an ulp off for sides that
 * are not powers of two), and the result is added to the finer level's own gradient.  d0 [Bt, h[0], w[0], C]. */
void mip_fold(int n_levels, int C, int Bt, const real *const *g, const int *h, const int *w, real *d0)
{
    int top = n_levels - 1;
    while (top > 0 && !g[top]) --top;
    int64_t most = 0;
    for (int k = 0; k <= top; ++k) most = (int64_t)h[k] * w[k] * C > most ? (int64_t)h[k] * w[k] * C : most;
    real *cur = malloc(sizeof(real) * most), *up = malloc(sizeof(real) * most);
    for (int b = 0; b < Bt; ++b) {
        for (int k = top; k >= 0; --k) {
            const int64_t n = (int64_t)h[k] * w[k] * C;
            const real *gk = g[k] ? g[k] + (int64_t)b * n : NULL;
            real *out = k ? cur : d0 + (int64_t)b * n;
            for (int y = 0; y < h[k]; ++y)
                for (int x = 0; x < w[k]; ++x)
                    for (int c = 0; c < C; ++c) {
                        const int64_t i = ((int64_t)y * w[k] + x) * C + c;
                        real s = 0;
                        if (k < top) {
                            int64_t x0, x1, y0, y1;
                            real fx, fy;
                            clamped_axis((real)x * (real)0.5 - (real)0.25, w[k + 1], &x0, &x1, &fx);
                            clamped_axis((real)y * (real)0.5 - (real)0.25, h[k + 1], &y0, &y1, &fy);
                            const real q = (real)0.25;
                            const real t00 = q * up[(y0 * w[k + 1] + x0) * C + c], t10 = q * up[(y0 * w[k + 1] + x1) * C + c];
                            const real t01 = q * up[(y1 * w[k + 1] + x0) * C + c], t11 = q * up[(y1 * w[k + 1] + x1) * C + c];
                            const real ox = (real)1 - fx, oy = (real)1 - fy;
                            s = oy * (ox * t00 + fx * t10) + fy * (ox * t01 + fx * t11);
                        }
                        out[i] = !gk ? s : (k < top ? gk[i] + s : gk[i]);
                    }
            if (k) { real *t = up; up = cur; cur = t; }
        }
    }
    free(cur);
    free(up);
}

/* torch.clamp(x, lo[c], hi[c]) with tensor bounds: a NaN texel stays, else a NaN bound is returned, else min(max(x, lo), hi) */
void mip_clamp(int n_levels, int C, int Bt, real *const *lv, const int *h, const int *w, const real *lo, const real *hi)
{
    for (int k = 0; k < n_levels; ++k)
        for (int64_t i = 0; i < (int64_t)Bt * h[k] * w[k] * C; ++i) {
            const real x = lv[k][i], l = lo[i % C], u = hi[i % C];
            if (x != x) continue;
            if (l != l) { lv[k][i] = l; continue; }
            if (u != u) { lv[k][i] = u; continue; }
            const real m = x < l ? l : x;
            lv[k][i] = u < m ? u : m;
        }
}

/* util.safe_normalize on 3 channels: x / sqrt(max(x0 x0 + x1 x1 + x2 x2, 1e-20)), a NaN dot kept */
void mip_normalize(int n_levels, int Bt, real *const *lv, const int *h, const int *w)
{
    for (int k = 0; k < n_levels; ++k)
        for (int64_t i = 0; i < (int64_t)Bt * h[k] * w[k]; ++i) {
            real *p = lv[k] + 3 * i;
            const real d = p[0] * p[0] + p[1] * p[1] + p[2] * p[2];
            const real eps = (real)1e-20;
            const real l = R_SQRT(d != d || d > eps ? d : eps);
            p[0] = p[0] / l; p[1] = p[1] / l; p[2] = p[2] / l;
        }
}
