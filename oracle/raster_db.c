/*
 * oracle/raster_db.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C, fp32 by default, fp64 with -DORACLE_F64 for finite-difference checks of the hand-derived adjoints) of the
 * G-buffer producer's screen-space derivatives: rast_db, interpolate's attribute derivatives out_da, their adjoints (d attr, d rast_db,
 * d rast_db -> d pos), and interpolate's forward in the kernel's operation order.  No reference code exists for them (nvdiffrast is
 * absent); the semantics are those stated in nvdiffrecmc_b200/csrc/raster.cu.  Compile with -ffp-contract=off.  The pixel-centre,
 * triangle-id and barycentric terms are evaluated exactly as oracle/geometry.c evaluates them for the rasterize backward.  Loaded by
 * oracle/raster_db.py.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#ifdef ORACLE_F64
typedef double real;
#define R_FMA(a, b, c) fma(a, b, c)
#else
typedef float real;
#define R_FMA(a, b, c) fmaf(a, b, c)
#endif
#define RC(x) ((real)(x))

int db_sizeof_real(void) { return (int)sizeof(real); }

/* NDC coordinate of pixel centre i of n (row iy -> NDC y = (iy + 0.5) / H * 2 - 1, no flip), as the kernels */
static inline real px_ndc(int i, int n) { return ((real)i + RC(0.5f)) / (real)n * RC(2.0f) - RC(1.0f); }

/* triangle id of a rast pixel (id + 1 in channel 3), -1 for background and ids >= T */
static inline int rast_tid(const real *r, int T)
{
    const int id = (int)r[3] - 1;
    return id < T ? id : -1;
}

/* a_i = (x_i - px w_i, y_i - py w_i), s_i = a_{i+1} x a_{i+2}, S = (s0 + s1) + s2; returns 0 when S == 0 */
static int bary_terms(const real *P, const int32_t *tri, real px, real py, real ax[3], real ay[3], real s[3], real *S)
{
    for (int k = 0; k < 3; ++k) {
        const real *q = P + 4 * (size_t)tri[k];
        ax[k] = q[0] - px * q[3]; ay[k] = q[1] - py * q[3];
    }
    s[0] = ax[1] * ay[2] - ay[1] * ax[2];
    s[1] = ax[2] * ay[0] - ay[2] * ax[0];
    s[2] = ax[0] * ay[1] - ay[0] * ax[1];
    *S = s[0] + s[1] + s[2];
    return *S != RC(0);
}

/* ================================================================================================================================
 * Screen-space derivatives (nvdiffrecmc_b200/csrc/raster.cu: k_rast_db, k_interpolate_da, k_rasterize_bwd<true>), restated:
 *   rast_db[b,y,x] = (du/dX, du/dY, dv/dX, dv/dY), X the column and Y the row index in pixels, for the triangle id in rast (0 for
 *   background, ids >= T and S == 0).  With a_k = (x_k - px w_k, y_k - py w_k), s_i = a_{i+1} x a_{i+2}, S = sum s_i, u = s0 / S,
 *   v = s1 / S, each s_i is affine in (px, py):  ds_i/dpx = y_{i+1} w_{i+2} - w_{i+1} y_{i+2},  ds_i/dpy = w_{i+1} x_{i+2} - x_{i+1} w_{i+2};
 *   du/dpx = (ds0/dpx - u dS/dpx) / S (likewise py, and v with s1);  d/dX = (2/W) d/dpx,  d/dY = (2/H) d/dpy.
 *   out_da[b,y,x,2k:2k+2] = (db.x (A0 - A2) + db.z (A1 - A2), db.y (A0 - A2) + db.w (A1 - A2)) for the k-th selected attribute.
 * The fp32 build evaluates rast_db, out_da and d rast_db in the kernels' explicitly rounded order (this file is compiled with
 * -ffp-contract=off), so they agree bit for bit.  interpolate's forward uses the kernel's fused multiply-adds.
 * ================================================================================================================================ */

/* out = fma(w0, A0, fma(w1, A1, w2 A2)) with w2 = 1 - u - v, as k_interpolate<0> */
void orc_interpolate_fwd(int B, int H, int W, int C, int64_t attr_bs, const real *attr, int T, const int32_t *tris, const real *rast, real *out)
{
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int b = (int)(i / ((int64_t)W * H));
        const int id = rast_tid(rast + 4 * i, T);
        for (int c = 0; c < C; ++c) out[i * C + c] = 0;
        if (id < 0) continue;
        const real *A = attr + b * attr_bs;
        const int32_t *tri = tris + 3 * (size_t)id;
        const real w0 = rast[4 * i], w1 = rast[4 * i + 1], w2 = RC(1) - w0 - w1;
        for (int c = 0; c < C; ++c)
            out[i * C + c] = R_FMA(w0, A[(size_t)tri[0] * C + c], R_FMA(w1, A[(size_t)tri[1] * C + c], w2 * A[(size_t)tri[2] * C + c]));
    }
}

/* per-pixel terms of rast_db: vertex (x, y, w), ds_i/dpx, ds_i/dpy and their sums; 0 when the pixel has none */
typedef struct { real x[3], y[3], w[3], ax[3], ay[3], s[3], S, dx[3], dy[3], dSx, dSy, u, v, px, py; } DbTerms;

static int db_terms(const real *P, const int32_t *tri, int ix, int iy, int H, int W, DbTerms *d)
{
    d->px = px_ndc(ix, W); d->py = px_ndc(iy, H);
    if (!bary_terms(P, tri, d->px, d->py, d->ax, d->ay, d->s, &d->S)) return 0;
    for (int k = 0; k < 3; ++k) {
        const real *q = P + 4 * (size_t)tri[k];
        d->x[k] = q[0]; d->y[k] = q[1]; d->w[k] = q[3];
    }
    for (int k = 0; k < 3; ++k) {
        const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
        d->dx[k] = d->y[k1] * d->w[k2] - d->w[k1] * d->y[k2];
        d->dy[k] = d->w[k1] * d->x[k2] - d->x[k1] * d->w[k2];
    }
    d->dSx = d->dx[0] + d->dx[1] + d->dx[2]; d->dSy = d->dy[0] + d->dy[1] + d->dy[2];
    d->u = d->s[0] / d->S; d->v = d->s[1] / d->S;
    return 1;
}

void orc_rast_db(int B, int H, int W, int64_t pos_bs, const real *pos, int T, const int32_t *tris, const real *rast, real *db)
{
    const real sx = RC(2) / (real)W, sy = RC(2) / (real)H;
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int ix = (int)(i % W), iy = (int)((i / W) % H), b = (int)(i / ((int64_t)W * H));
        const int id = rast_tid(rast + 4 * i, T);
        real *o = db + 4 * i;
        DbTerms d;
        o[0] = o[1] = o[2] = o[3] = RC(0);
        if (id < 0 || !db_terms(pos + b * pos_bs, tris + 3 * (size_t)id, ix, iy, H, W, &d)) continue;
        o[0] = (d.dx[0] - d.u * d.dSx) / d.S * sx;
        o[1] = (d.dy[0] - d.u * d.dSy) / d.S * sy;
        o[2] = (d.dx[1] - d.v * d.dSx) / d.S * sx;
        o[3] = (d.dy[1] - d.v * d.dSy) / d.S * sy;
    }
}

/* d rast_db -> d pos (accumulated): L = sum_{c = u, v; p = px, py} h_cp (ds_c/dp - c dS/dp) / S, h = d rast_db scaled by 2/W, 2/H */
void orc_rast_db_bwd(int B, int H, int W, int64_t pos_bs, const real *pos, int T, const int32_t *tris, const real *rast, const real *d_db, real *d_pos)
{
    const real sx = RC(2) / (real)W, sy = RC(2) / (real)H;
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int ix = (int)(i % W), iy = (int)((i / W) % H), b = (int)(i / ((int64_t)W * H));
        const int id = rast_tid(rast + 4 * i, T);
        const int32_t *tri = tris + 3 * (size_t)id;
        DbTerms d;
        if (id < 0 || !db_terms(pos + b * pos_bs, tri, ix, iy, H, W, &d)) continue;
        const real *g = d_db + 4 * i, S = d.S, u = d.u, v = d.v;
        const real hxu = g[0] * sx, hyu = g[1] * sy, hxv = g[2] * sx, hyv = g[3] * sy;
        const real Kx = hxu * u + hxv * v, Ky = hyu * u + hyv * v;
        const real ex[3] = {(hxu - Kx) / S, (hxv - Kx) / S, -Kx / S};                 /* dL / d(ds_i/dpx) */
        const real ey[3] = {(hyu - Ky) / S, (hyv - Ky) / S, -Ky / S};                 /* dL / d(ds_i/dpy) */
        const real mu = -(hxu * d.dSx + hyu * d.dSy) / S, mv = -(hxv * d.dSx + hyv * d.dSy) / S;         /* dL/du, dL/dv */
        const real Ldb = (hxu * (d.dx[0] - u * d.dSx) + hyu * (d.dy[0] - u * d.dSy) + hxv * (d.dx[1] - v * d.dSx) + hyv * (d.dy[1] - v * d.dSy)) / S;
        const real GS = -(Ldb + mu * u + mv * v) / S;                                 /* dL/dS */
        const real gs[3] = {mu / S + GS, mv / S + GS, GS};                           /* dL/ds_i */
        for (int k = 0; k < 3; ++k) {
            const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
            const real dax = gs[k2] * d.ay[k1] - gs[k1] * d.ay[k2];
            const real day = gs[k1] * d.ax[k2] - gs[k2] * d.ax[k1];
            real *o = d_pos + b * pos_bs + 4 * (size_t)tri[k];
            o[0] += dax + ey[k1] * d.w[k2] - ey[k2] * d.w[k1];
            o[1] += day + ex[k2] * d.w[k1] - ex[k1] * d.w[k2];
            o[3] += -d.px * dax - d.py * day + ex[k1] * d.y[k2] - ex[k2] * d.y[k1] + ey[k2] * d.x[k1] - ey[k1] * d.x[k2];
        }
    }
}

/* out_da [B,H,W,2n]; idx = NULL selects every attribute in order (n = C) */
void orc_interpolate_da(int B, int H, int W, int C, int64_t attr_bs, const real *attr, int T, const int32_t *tris, const real *rast, const real *db,
                        int n, const int32_t *idx, real *out_da)
{
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int b = (int)(i / ((int64_t)W * H));
        const int id = rast_tid(rast + 4 * i, T);
        real *o = out_da + i * 2 * n;
        for (int k = 0; k < 2 * n; ++k) o[k] = RC(0);
        if (id < 0) continue;
        const real *A = attr + b * attr_bs, *g = db + 4 * i;
        const int32_t *tri = tris + 3 * (size_t)id;
        for (int k = 0; k < n; ++k) {
            const int c = idx ? idx[k] : k;
            const real a2 = A[(size_t)tri[2] * C + c], d0 = A[(size_t)tri[0] * C + c] - a2, d1 = A[(size_t)tri[1] * C + c] - a2;
            o[2 * k] = g[0] * d0 + g[2] * d1;
            o[2 * k + 1] = g[1] * d0 + g[3] * d1;
        }
    }
}

/* d attr (accumulated) and d rast_db (overwritten) of out_da */
void orc_interpolate_da_bwd(int B, int H, int W, int C, int64_t attr_bs, const real *attr, int T, const int32_t *tris, const real *rast, const real *db,
                            int n, const int32_t *idx, const real *d_out_da, real *d_attr, real *d_db)
{
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int b = (int)(i / ((int64_t)W * H));
        const int id = rast_tid(rast + 4 * i, T);
        real e[4] = {0, 0, 0, 0};
        if (id >= 0) {
            const real *A = attr + b * attr_bs, *g = db + 4 * i;
            real *D = d_attr + b * attr_bs;
            const int32_t *tri = tris + 3 * (size_t)id;
            for (int k = 0; k < n; ++k) {
                const int c = idx ? idx[k] : k;
                const real gX = d_out_da[(i * n + k) * 2], gY = d_out_da[(i * n + k) * 2 + 1];
                const real a2 = A[(size_t)tri[2] * C + c], d0 = A[(size_t)tri[0] * C + c] - a2, d1 = A[(size_t)tri[1] * C + c] - a2;
                const real a0 = gX * g[0] + gY * g[1], a1 = gX * g[2] + gY * g[3];
                D[(size_t)tri[0] * C + c] += a0; D[(size_t)tri[1] * C + c] += a1; D[(size_t)tri[2] * C + c] -= a0 + a1;
                e[0] = e[0] + gX * d0; e[1] = e[1] + gY * d0; e[2] = e[2] + gX * d1; e[3] = e[3] + gY * d1;
            }
        }
        for (int k = 0; k < 4; ++k) d_db[4 * i + k] = e[k];
    }
}
