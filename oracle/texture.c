/* texture.c -- CPU oracle of the filtered, mip-mapped texture look-up (TEST INFRASTRUCTURE, not product code).
 *
 * A plain-C restatement of the contract in nvdiffrecmc_b200/csrc/texture.cu, written independently of the kernels:
 *   bilinear sample of a level (x = u * W - 0.5, taps (x0, x0+1) x (y0, y0+1), wrap = index mod size, clamp = index clamped),
 *   level of detail from the major axis of the pixel footprint, lam = 0.5 * log2(M) clamped to [0, L], trilinear blend of levels
 *   floor(lam) and floor(lam) + 1 (level l1 not read when the blend fraction is 0), and the three adjoints:
 *   d tex (a sequential scatter in pixel, channel-group, level, tap order), d uv and d uv_da (one writer per pixel).
 * Two builds of this file (oracle/texture.py): fp32 (`real` = float; log2 is the fixed algorithm of the contract, so the forward, d uv and
 * d uv_da equal the kernels' bit for bit) and fp64 (-DORACLE_F64, libm log2; checked by finite differences and the adjoint identity).
 * Compile with -ffp-contract=off: every product and sum is one IEEE round-to-nearest operation, in the order the contract writes it.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#ifdef ORACLE_F64
typedef double real;
#define R_FLOOR floor
#define R_SQRT sqrt
#define TWO_LN2 1.3862943611198906
#else
typedef float real;
#define R_FLOOR floorf
#define R_SQRT sqrtf
#define TWO_LN2 1.38629436f
#endif

int tex_sizeof_real(void) { return (int)sizeof(real); }

/* The contract's log2 (fp32): exponent extraction, Cephes' single-precision logf polynomial on the mantissa, fixed order. */
float tex_log2f(float x)
{
    if (!(x > 0.0f)) return x == 0.0f ? -INFINITY : NAN;
    if (isinf(x)) return x;
    int e = 0;
    if (x < 1.17549435e-38f) { x = x * 8388608.0f; e = -23; }
    uint32_t bits;
    memcpy(&bits, &x, 4);
    e += (int)((bits >> 23) & 0xffu) - 126;
    bits = (bits & 0x7fffffu) | 0x3f000000u;
    float m;
    memcpy(&m, &bits, 4);
    float z;
    if (m < 0.707106781186547524f) { e -= 1; z = (m + m) - 1.0f; } else { z = m - 1.0f; }
    const float zz = z * z;
    static const float P[9] = {7.0376836292e-2f, -1.1514610310e-1f, 1.1676998740e-1f, -1.2420140846e-1f, 1.4249322787e-1f,
                               -1.6668057665e-1f, 2.0000714765e-1f, -2.4999993993e-1f, 3.3333331174e-1f};
    float p = P[0];
    for (int i = 1; i < 9; ++i) p = p * z + P[i];
    float y = (p * z) * zz;
    y = y - 0.5f * zz;
    const float L2EA = 0.44269504088896340736f;
    float r = y * L2EA;
    r = r + z * L2EA;
    r = r + y;
    r = r + z;
    return r + (float)e;
}

#ifdef ORACLE_F64
static real lg2(real x) { return log2(x); }
#else
static real lg2(real x) { return tex_log2f(x); }
#endif

/* floor of x as cvt.rmi.s32 does it: saturating, NaN -> 0 */
static int32_t floor_s32(real x)
{
    const real f = R_FLOOR(x);
    if (f != f) return 0;
    if (f >= (real)2147483648.0) return INT32_MAX;
    if (f <= (real)-2147483648.0) return INT32_MIN;
    return (int32_t)f;
}

static void axis(real u, int n, int clamp, int64_t *i0, int64_t *i1, real *fr)
{
    const real x = u * (real)n - (real)0.5;
    *fr = x - R_FLOOR(x);
    const int64_t x0 = floor_s32(x), x1 = x0 + 1;
    if (clamp) {
        *i0 = x0 < 0 ? 0 : (x0 > n - 1 ? n - 1 : x0);
        *i1 = x1 < 0 ? 0 : (x1 > n - 1 ? n - 1 : x1);
    } else {
        *i0 = ((x0 % n) + n) % n;
        *i1 = ((x1 % n) + n) % n;
    }
}

typedef struct {
    int64_t o[4];       /* element offsets of t00, t10, t01, t11 */
    real fx, fy;
} taps_t;

static taps_t taps(int C, int h, int w, int64_t bstride, int b, real u, real v, int clamp)
{
    taps_t t;
    int64_t x0, x1, y0, y1;
    axis(u, w, clamp, &x0, &x1, &t.fx);
    axis(v, h, clamp, &y0, &y1, &t.fy);
    const int64_t base = (int64_t)b * bstride;
    t.o[0] = base + (y0 * w + x0) * C;
    t.o[1] = base + (y0 * w + x1) * C;
    t.o[2] = base + (y1 * w + x0) * C;
    t.o[3] = base + (y1 * w + x1) * C;
    return t;
}

static real bilerp(const real *p, const taps_t *t, int c)
{
    const real ox = (real)1 - t->fx, oy = (real)1 - t->fy;
    const real top = ox * p[t->o[0] + c] + t->fx * p[t->o[1] + c];
    const real bot = ox * p[t->o[2] + c] + t->fx * p[t->o[3] + c];
    return oy * top + t->fy * bot;
}

typedef struct {
    int l0, l1;
    real f, lam_raw, a, b, c, d, C, h, q, M;
} lod_t;

static lod_t lod(const real *da, real W0, real H0, int L)
{
    lod_t o;
    o.a = da[0] * W0; o.b = da[1] * W0; o.c = da[2] * H0; o.d = da[3] * H0;
    const real A = o.a * o.a + o.c * o.c, B = o.b * o.b + o.d * o.d;
    o.C = o.a * o.b + o.c * o.d;
    o.h = (A - B) * (real)0.5;
    o.q = R_SQRT(o.h * o.h + o.C * o.C);
    o.M = (A + B) * (real)0.5 + o.q;
    o.lam_raw = (real)0.5 * lg2(o.M);
    real lam = o.lam_raw > (real)0 ? o.lam_raw : (real)0;       /* NaN -> 0 */
    if (lam > (real)L) lam = (real)L;
    const real fl = R_FLOOR(lam);
    o.l0 = (int)fl;
    o.f = lam - fl;
    o.l1 = o.l0 + 1 < L ? o.l0 + 1 : L;
    return o;
}

/* level k: ptr[k] [Bt, h[k], w[k], C] with minibatch stride bstride[k] (0 = shared); uv [B,H,W,2], uv_da [B,H,W,4] (mip only). */
void tex_fwd(int n_levels, int C, const real *const *ptr, const int *h, const int *w, const int64_t *bstride, const real *uv, const real *uv_da,
             int B, int H, int W, int mip, int clamp, real *out)
{
    const int64_t n = (int64_t)B * H * W;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        const int b = (int)(i / ((int64_t)H * W));
        lod_t d;
        memset(&d, 0, sizeof d);
        if (mip) d = lod(uv_da + 4 * i, (real)w[0], (real)h[0], n_levels - 1);
        const taps_t t0 = taps(C, h[d.l0], w[d.l0], bstride[d.l0], b, uv[2 * i], uv[2 * i + 1], clamp);
        const taps_t t1 = taps(C, h[d.l1], w[d.l1], bstride[d.l1], b, uv[2 * i], uv[2 * i + 1], clamp);
        for (int c = 0; c < C; ++c) {
            real r = bilerp(ptr[d.l0], &t0, c);
            if (d.f != 0) r = ((real)1 - d.f) * r + d.f * bilerp(ptr[d.l1], &t1, c);
            out[i * C + c] = r;
        }
    }
}

/* d_tex: n_levels pointers (null entries skipped) accumulated; d_uv [B,H,W,2], d_uv_da [B,H,W,4] overwritten (each may be null). */
void tex_bwd(int n_levels, int C, const real *const *ptr, const int *h, const int *w, const int64_t *bstride, const real *uv, const real *uv_da,
             int B, int H, int W, int mip, int clamp, const real *d_out, real *const *d_tex, real *d_uv, real *d_uv_da)
{
    const int64_t n = (int64_t)B * H * W;
    const int L = mip ? n_levels - 1 : 0;
    for (int64_t i = 0; i < n; ++i) {
        const int b = (int)(i / ((int64_t)H * W));
        lod_t d;
        memset(&d, 0, sizeof d);
        if (mip) d = lod(uv_da + 4 * i, (real)w[0], (real)h[0], L);
        const real u = uv[2 * i], v = uv[2 * i + 1];
        const taps_t t[2] = {taps(C, h[d.l0], w[d.l0], bstride[d.l0], b, u, v, clamp), taps(C, h[d.l1], w[d.l1], bstride[d.l1], b, u, v, clamp)};
        const int lv[2] = {d.l0, d.l1};
        const real wl[2] = {(real)1 - d.f, d.f};
        const int two = d.f != 0;
        const int want_da = mip && d.lam_raw > 0 && d.lam_raw < (real)L && two;
        real su[2] = {0, 0}, sv[2] = {0, 0}, gl = 0;
        const real *g = d_out + i * C;
        for (int c = 0; c < C; ++c) {
            for (int s = 0; s < 1 + two; ++s) {
                const real *p = ptr[lv[s]];
                const real *o00 = p + t[s].o[0] + c, *o10 = p + t[s].o[1] + c, *o01 = p + t[s].o[2] + c, *o11 = p + t[s].o[3] + c;
                const real ox = (real)1 - t[s].fx, oy = (real)1 - t[s].fy;
                const real du = oy * (*o10 - *o00) + t[s].fy * (*o11 - *o01);
                const real dv = ox * (*o01 - *o00) + t[s].fx * (*o11 - *o10);
                su[s] = su[s] + g[c] * du;
                sv[s] = sv[s] + g[c] * dv;
            }
            if (want_da) gl = gl + g[c] * (bilerp(ptr[d.l1], &t[1], c) - bilerp(ptr[d.l0], &t[0], c));
        }
        if (d_tex) {
            /* channel groups of the kernels' vector width make no difference here: a group with an all-zero gradient adds only zeros */
            for (int s = 0; s < 1 + two; ++s) {
                real *dt = d_tex[lv[s]];
                if (!dt) continue;
                const real ox = (real)1 - t[s].fx, oy = (real)1 - t[s].fy;
                const real wt[4] = {wl[s] * (oy * ox), wl[s] * (oy * t[s].fx), wl[s] * (t[s].fy * ox), wl[s] * (t[s].fy * t[s].fx)};
                for (int c = 0; c < C; ++c) {
                    if (g[c] == 0) continue;
                    for (int j = 0; j < 4; ++j) dt[t[s].o[j] + c] = dt[t[s].o[j] + c] + wt[j] * g[c];
                }
            }
        }
        if (d_uv) {
            real du = wl[0] * ((real)w[d.l0] * su[0]), dv = wl[0] * ((real)h[d.l0] * sv[0]);
            if (two) {
                du = du + wl[1] * ((real)w[d.l1] * su[1]);
                dv = dv + wl[1] * ((real)h[d.l1] * sv[1]);
            }
            d_uv[2 * i] = du;
            d_uv[2 * i + 1] = dv;
        }
        if (d_uv_da && mip) {
            real r[4] = {0, 0, 0, 0};
            if (want_da) {
                const real gM = gl / (d.M * TWO_LN2);
                real gA, gB, gC;
                if (d.q > 0) {
                    const real rr = d.h / d.q, e = d.C / d.q;
                    gA = gM * ((real)0.5 + (real)0.5 * rr);
                    gB = gM * ((real)0.5 - (real)0.5 * rr);
                    gC = gM * e;
                } else {
                    gA = gB = gM * (real)0.5;
                    gC = 0;
                }
                const real W0 = (real)w[0], H0 = (real)h[0];
                r[0] = ((d.a + d.a) * gA + d.b * gC) * W0;
                r[1] = ((d.b + d.b) * gB + d.a * gC) * W0;
                r[2] = ((d.c + d.c) * gA + d.d * gC) * H0;
                r[3] = ((d.d + d.d) * gB + d.c * gC) * H0;
            }
            memcpy(d_uv_da + 4 * i, r, sizeof r);
        }
    }
}
