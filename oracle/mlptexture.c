/* mlptexture.c -- CPU oracle of the fused MLP texture (TEST INFRASTRUCTURE, not product code).
 *
 * A plain-C restatement of the contract in nvdiffrecmc_b200/csrc/mlptexture.cu, written independently of the kernels: normalise into the
 * AABB, clamp, encode (hashgrid.c's hg_fwd, included below rather than copied), a bias-free ReLU MLP of `hidden` 32-wide layers and C
 * outputs, the fixed exp and the sigmoid scaled into min_max; the backward's d W as chunk partials (fma chains over MLPTEX_CHUNK
 * consecutive points) summed in chunk order, d params and d x through hashgrid.c's hg_bwd.  Weights are one flat array: layer l < hidden
 * at l * 1024 ([32,32], [out, in] row-major), the output layer at hidden * 1024 ([C,32]).
 * Two builds (oracle/mlptexture.py), as hashgrid.c: fp32 (`real` = float, compared bit for bit with the CUDA output, encoding, d texc and
 * d W) and fp64 (-DORACLE_F64, libm exp; checked by finite differences).  Compile with -ffp-contract=off.
 */
#include "hashgrid.c"

#include <stdlib.h>
#define MLPTEX_CHUNK 1024          /* MCS_MLPTEX_CHUNK */

/* Cephes expf: range reduction by ln 2 in two parts, a degree-5 polynomial, and 2^n applied as two normal powers of two (one rounding) */
static float det_expf(float x)
{
    if (x != x) return x;
    if (x > 88.72283935546875f) return INFINITY;
    if (x < -103.27892990343185f) return 0.0f;
    const float z = floorf(1.44269504088896341f * x + 0.5f);
    const int n = (int)z;
    float r = x - z * 0.693359375f;
    r = r - z * -2.12194440e-4f;
    const float rr = r * r;
    float p = 1.9875691500e-4f;
    p = p * r + 1.3981999507e-3f;
    p = p * r + 8.3334519073e-3f;
    p = p * r + 4.1665795894e-2f;
    p = p * r + 1.6666665459e-1f;
    p = p * r + 5.0000001201e-1f;
    p = p * rr + r + 1.0f;
    const int n1 = n / 2, n2 = n - n1;
    union { uint32_t u; float f; } s1, s2;
    s1.u = (uint32_t)(n1 + 127) << 23;
    s2.u = (uint32_t)(n2 + 127) << 23;
    return (p * s1.f) * s2.f;
}

static real mt_exp(real x)
{
#ifdef ORACLE_F64
    return exp(x);
#else
    return det_expf(x);
#endif
}

/* the contract's exp (fp32 build; libm exp in the fp64 build) */
void mlt_exp(const real *x, int64_t n, real *y)
{
    for (int64_t i = 0; i < n; ++i) y[i] = mt_exp(x[i]);
}

/* xn = (t - a0) / (a1 - a0), xc = clamp(xn, 0, 1) with NaN kept */
static void mt_normalise(const real *t, int64_t n, const real *aabb, real *xn, real *xc)
{
    for (int64_t i = 0; i < 3 * n; ++i) {
        const int d = (int)(i % 3);
        xn[i] = (t[i] - aabb[d]) / (aabb[3 + d] - aabb[d]);
        xc[i] = xn[i] < 0 ? (real)0 : (xn[i] > 1 ? (real)1 : xn[i]);
    }
}

/* acts [(hidden + 1) * 32]: the input of every layer (acts[0..31] = e); s [C]: the sigmoid */
static void mt_point_fwd(const real *e, int hidden, int C, const real *w, real *acts, real *s)
{
    memcpy(acts, e, 32 * sizeof(real));
    for (int l = 0; l < hidden; ++l)
        for (int j = 0; j < 32; ++j) {
            real acc = 0;
            for (int k = 0; k < 32; ++k) acc = R_FMA(w[l * 1024 + j * 32 + k], acts[l * 32 + k], acc);
            acts[(l + 1) * 32 + j] = acc <= 0 ? (real)0 : acc;
        }
    for (int c = 0; c < C; ++c) {
        real acc = 0;
        for (int k = 0; k < 32; ++k) acc = R_FMA(w[hidden * 1024 + c * 32 + k], acts[hidden * 32 + k], acc);
        s[c] = (real)1 / ((real)1 + mt_exp(-acc));
    }
}

/* t [n,3], aabb [2,3], min_max [2,C]; out [n,C]; enc [n,32] (may be null).  L must be 16. */
void mlt_fwd(const real *t, int64_t n, const real *aabb, const real *min_max, const real *params, int L, const uint64_t *offset,
                   const uint32_t *res, const float *scale, uint32_t dense_mask, int hidden, int C, const real *w, real *out, real *enc)
{
    real *xn = malloc(sizeof(real) * 3 * (size_t)n + 1), *xc = malloc(sizeof(real) * 3 * (size_t)n + 1);
    real *e = malloc(sizeof(real) * 32 * (size_t)n + 1);
    mt_normalise(t, n, aabb, xn, xc);
    hg_fwd(xc, n, params, L, offset, res, scale, dense_mask, e);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        real acts[5 * 32], s[8];
        mt_point_fwd(e + 32 * i, hidden, C, w, acts, s);
        for (int c = 0; c < C; ++c) out[i * C + c] = s[c] * (min_max[C + c] - min_max[c]) + min_max[c];
    }
    if (enc) memcpy(enc, e, sizeof(real) * 32 * (size_t)n);
    free(xn); free(xc); free(e);
}

/* d_out [n,C]; d_params (may be null) accumulates; d_t [n,3] and d_w [hidden * 1024 + 32 C] (each may be null) are overwritten. */
void mlt_bwd(const real *t, int64_t n, const real *aabb, const real *min_max, const real *params, int L, const uint64_t *offset,
                   const uint32_t *res, const float *scale, uint32_t dense_mask, int hidden, int C, const real *w, const real *d_out,
                   real *d_params, real *d_t, real *d_w)
{
    const int nA = (hidden + 1) * 32, nD = hidden * 32 + C, nW = hidden * 1024 + C * 32;
    real *xn = malloc(sizeof(real) * 3 * (size_t)n + 1), *xc = malloc(sizeof(real) * 3 * (size_t)n + 1);
    real *e = malloc(sizeof(real) * 32 * (size_t)n + 1), *de = malloc(sizeof(real) * 32 * (size_t)n + 1);
    real *A = malloc(sizeof(real) * nA * (size_t)n + 1), *D = malloc(sizeof(real) * nD * (size_t)n + 1);
    mt_normalise(t, n, aabb, xn, xc);
    hg_fwd(xc, n, params, L, offset, res, scale, dense_mask, e);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        real s[8], dh[32], dv[32];
        real *acts = A + nA * i, *dd = D + nD * i;
        mt_point_fwd(e + 32 * i, hidden, C, w, acts, s);
        for (int k = 0; k < 32; ++k) dh[k] = 0;
        for (int c = 0; c < C; ++c) {
            const real gs = d_out[i * C + c] * (min_max[C + c] - min_max[c]);
            const real dz = gs * (((real)1 - s[c]) * s[c]);
            dd[hidden * 32 + c] = dz;
            for (int k = 0; k < 32; ++k) dh[k] = R_FMA(dz, w[hidden * 1024 + c * 32 + k], dh[k]);
        }
        for (int l = hidden - 1; l >= 0; --l) {
            for (int j = 0; j < 32; ++j) dd[l * 32 + j] = acts[(l + 1) * 32 + j] > 0 ? dh[j] : (real)0;
            for (int k = 0; k < 32; ++k) dv[k] = 0;
            for (int j = 0; j < 32; ++j)
                for (int k = 0; k < 32; ++k) dv[k] = R_FMA(dd[l * 32 + j], w[l * 1024 + j * 32 + k], dv[k]);
            memcpy(dh, dv, sizeof dh);
        }
        memcpy(de + 32 * i, dh, sizeof dh);
    }
    if (d_w) {
        real *part = malloc(sizeof(real) * nW);
        for (int q = 0; q < nW; ++q) d_w[q] = 0;
        for (int64_t c0 = 0; c0 < n; c0 += MLPTEX_CHUNK) {
            const int64_t c1 = c0 + MLPTEX_CHUNK < n ? c0 + MLPTEX_CHUNK : n;
#pragma omp parallel for schedule(static)
            for (int q = 0; q < nW; ++q) {
                const int l = q / 1024 < hidden ? q / 1024 : hidden, r = q - l * 1024, row = r / 32, k = r % 32;
                real p = 0;
                for (int64_t i = c0; i < c1; ++i) p = R_FMA(D[nD * i + l * 32 + row], A[nA * i + l * 32 + k], p);
                part[q] = p;
            }
            for (int q = 0; q < nW; ++q) d_w[q] = d_w[q] + part[q];
        }
        free(part);
    }
    if (d_params || d_t) {
        real *dxc = d_t ? malloc(sizeof(real) * 3 * (size_t)n + 1) : NULL;
        hg_bwd(xc, n, params, L, offset, res, scale, dense_mask, de, d_params, dxc);
        if (d_t) {
            for (int64_t i = 0; i < 3 * n; ++i) {
                const int d = (int)(i % 3);
                const real g = (xn[i] >= 0 && xn[i] <= 1) ? dxc[i] : (real)0;
                d_t[i] = g / (aabb[3 + d] - aabb[d]);
            }
            free(dxc);
        }
    }
    free(xn); free(xc); free(e); free(de); free(A); free(D);
}
