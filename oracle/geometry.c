/*
 * oracle/geometry.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C, fp32 by default, fp64 with -DORACLE_F64 for finite-difference checks of the hand-derived adjoints) of the
 * G-buffer producer's geometry gradients: the barycentrics of the clip-space triangle and their adjoint (rasterize backward), the
 * adjoint of interpolate with respect to rast, edge adjacency, and pixel-pair analytic antialiasing.  No reference code exists for
 * them; the semantics are those stated in nvdiffrecmc_b200/csrc/raster.cu.  Compile with -ffp-contract=off: the antialias pair
 * decisions are evaluated in the same explicitly rounded operation order as the CUDA kernel.  Loaded by oracle/geometry.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef ORACLE_F64
typedef double real;
#define R_FABS(x) fabs(x)
#else
typedef float real;
#define R_FABS(x) fabsf(x)
#endif
#define RC(x) ((real)(x))

typedef struct { real x, y, z; } v3;

int geo_sizeof_real(void) { return (int)sizeof(real); }

/* ================================================================================================================================
 * Geometry gradients of the G-buffer producer (nvdiffrecmc_b200/csrc/raster.cu states the semantics and the derivation):
 * barycentrics of the clip-space triangle and their adjoint, the adjoint of interpolate with respect to rast, edge adjacency,
 * and pixel-pair analytic antialiasing (Laine et al. 2020).  rast is [B,H,W,4] (u, v, z/w, id + 1) in `real`; pos is [V,4]
 * (pos_bs = 0) or [B,V,4] (pos_bs = 4V).  The antialias pair decisions are evaluated in the same operation order as the CUDA kernel.
 * ================================================================================================================================ */
static inline real px_ndc(int i, int n) { return ((real)i + RC(0.5f)) / (real)n * RC(2.0f) - RC(1.0f); }

static inline int rast_tid(const real *r, int T)
{
    const int id = (int)r[3] - 1;
    return id < T ? id : -1;
}

/* u = s0 / S, v = s1 / S of a_i = (x_i - px w_i, y_i - py w_i); returns 0 when S == 0 */
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

void orc_raster_bary(int B, int H, int W, int64_t pos_bs, const real *pos, int T, const int32_t *tris, const real *rast, real *uv)
{
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int ix = (int)(i % W), iy = (int)((i / W) % H), b = (int)(i / ((int64_t)W * H));
        const int id = rast_tid(rast + 4 * i, T);
        real ax[3], ay[3], s[3], S;
        uv[2 * i] = uv[2 * i + 1] = RC(0);
        if (id < 0 || !bary_terms(pos + b * pos_bs, tris + 3 * (size_t)id, px_ndc(ix, W), px_ndc(iy, H), ax, ay, s, &S)) continue;
        uv[2 * i] = s[0] / S; uv[2 * i + 1] = s[1] / S;
    }
}

void orc_raster_bwd(int B, int H, int W, int64_t pos_bs, const real *pos, int T, const int32_t *tris, const real *rast, const real *d_rast, real *d_pos)
{
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int ix = (int)(i % W), iy = (int)((i / W) % H), b = (int)(i / ((int64_t)W * H));
        const int id = rast_tid(rast + 4 * i, T);
        const real px = px_ndc(ix, W), py = px_ndc(iy, H);
        const int32_t *tri = tris + 3 * (size_t)id;
        real ax[3], ay[3], s[3], S;
        if (id < 0 || !bary_terms(pos + b * pos_bs, tri, px, py, ax, ay, s, &S)) continue;
        const real du = d_rast[4 * i], dv = d_rast[4 * i + 1];
        const real G = du * (s[0] / S) + dv * (s[1] / S);
        const real gs[3] = {(du - G) / S, (dv - G) / S, -G / S};    /* dL/ds_i */
        for (int k = 0; k < 3; ++k) {
            const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;            /* s_{k2} = a_k x a_{k1}, s_{k1} = a_{k2} x a_k */
            const real dax = gs[k2] * ay[k1] - gs[k1] * ay[k2];
            const real day = gs[k1] * ax[k2] - gs[k2] * ax[k1];
            real *d = d_pos + b * pos_bs + 4 * (size_t)tri[k];
            d[0] += dax; d[1] += day; d[3] += -px * dax - py * day;
        }
    }
}

void orc_interpolate_bwd_rast(int B, int H, int W, int C, int64_t attr_bs, const real *attr, int T, const int32_t *tris, const real *rast,
                              const real *d_out, real *d_rast)
{
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int b = (int)(i / ((int64_t)W * H));
        const int id = rast_tid(rast + 4 * i, T);
        real du = 0, dv = 0;
        if (id >= 0) {
            const real *A = attr + b * attr_bs;
            const int32_t *tri = tris + 3 * (size_t)id;
            for (int c = 0; c < C; ++c) {
                const real g = d_out[i * C + c], a2 = A[(size_t)tri[2] * C + c];
                du += g * (A[(size_t)tri[0] * C + c] - a2);
                dv += g * (A[(size_t)tri[1] * C + c] - a2);
            }
        }
        d_rast[4 * i] = du; d_rast[4 * i + 1] = dv; d_rast[4 * i + 2] = 0; d_rast[4 * i + 3] = 0;
    }
}

/* edge adjacency by sorting the 3T (edge key, triangle) entries: a run of n equal keys is a boundary (n = 1), a shared edge (n = 2:
 * the other entry's triangle) or a non-manifold edge (n >= 3) */
typedef struct { uint64_t key; int32_t t, k; } EdgeEnt;
static int cmp_edge(const void *a, const void *b)
{
    const EdgeEnt *x = (const EdgeEnt *)a, *y = (const EdgeEnt *)b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    if (x->t != y->t) return x->t < y->t ? -1 : 1;
    return x->k - y->k;
}

void orc_aa_topology(int T, const int32_t *tris, int32_t *adj)
{
    const int64_t n = 3 * (int64_t)T;
    EdgeEnt *e = (EdgeEnt *)malloc(sizeof(EdgeEnt) * (size_t)n);
    for (int64_t i = 0; i < n; ++i) {
        const int t = (int)(i / 3), k = (int)(i % 3);
        const uint32_t a = (uint32_t)tris[3 * (size_t)t + k], c = (uint32_t)tris[3 * (size_t)t + (k + 1) % 3];
        e[i].key = ((uint64_t)(a < c ? a : c) << 32) | (a < c ? c : a);
        e[i].t = t; e[i].k = k;
    }
    qsort(e, (size_t)n, sizeof(EdgeEnt), cmp_edge);
    for (int64_t s = 0; s < n;) {
        int64_t r = s;
        while (r < n && e[r].key == e[s].key) ++r;
        for (int64_t j = s; j < r; ++j)
            adj[3 * (size_t)e[j].t + e[j].k] = r - s == 1 ? -1 : (r - s >= 3 ? -2 : e[j == s ? s + 1 : s].t);
        s = r;
    }
    free(e);
}

typedef struct {
    int B, H, W, C, V, T;
    int64_t pos_bs;
    const real *color, *rast, *pos;
    const int32_t *tris, *adj;
} OrcAA;

typedef struct { real t, ef, eo; int va, vb; v3 A, Bv; } AAEdge;      /* v3 (x, y, z) holds (x, y, w) */

static inline v3 aa_vert(const real *P, int v) { const real *q = P + 4 * (size_t)v; v3 r = {q[0], q[1], q[3]}; return r; }

static inline real aa_edge(v3 A, v3 B, real px, real py)
{
    const real ax = A.x - px * A.z, ay = A.y - py * A.z, bx = B.x - px * B.z, by = B.y - py * B.z;
    return ax * by - ay * bx;
}

static inline int aa_facing(v3 a, v3 b, v3 c)
{
    const real m0 = b.y * c.z - b.z * c.y, m1 = b.x * c.z - b.z * c.x, m2 = b.x * c.y - b.y * c.x;
    return a.x * m0 - a.y * m1 + a.z * m2 > RC(0);
}

/* rules 3-5: closest crossing candidate edge of front triangle F between pixel centres f and o */
static int aa_search(const OrcAA *p, const real *P, int F, int horiz, real fx, real fy, real ox, real oy, AAEdge *e)
{
    const int32_t *tri = p->tris + 3 * (size_t)F;
    v3 q[3];
    for (int k = 0; k < 3; ++k) q[k] = aa_vert(P, tri[k]);
    int found = 0;
    for (int k = 0; k < 3; ++k) {
        const int k1 = (k + 1) % 3;
        const v3 A = q[k], B = q[k1];
        if (!(A.z > RC(0) && B.z > RC(0))) continue;
        const int nb = p->adj[3 * (size_t)F + k];
        if (nb >= 0 && nb < p->T) {
            const int32_t *nt = p->tris + 3 * (size_t)nb;
            if (aa_facing(q[0], q[1], q[2]) == aa_facing(aa_vert(P, nt[0]), aa_vert(P, nt[1]), aa_vert(P, nt[2]))) continue;
        }
        const real dX = (B.x / B.z - A.x / A.z) * (real)p->W;
        const real dY = (B.y / B.z - A.y / A.z) * (real)p->H;
        if ((R_FABS(dY) >= R_FABS(dX)) != horiz) continue;
        const real ef = aa_edge(A, B, fx, fy), eo = aa_edge(A, B, ox, oy);
        if (!((ef > RC(0) && eo < RC(0)) || (ef < RC(0) && eo > RC(0)))) continue;
        const real t = ef / (ef - eo);
        if (!found || t < e->t) { found = 1; e->t = t; e->ef = ef; e->eo = eo; e->va = tri[k]; e->vb = tri[k1]; e->A = A; e->Bv = B; }
    }
    return found;
}

/* Pair of pixels i (first) and j: 1 when an edge crosses with a nonzero weight w; *gain = pixel that gains w (c_other - c_gain),
 * *front = front pixel; (fx, fy) / (ox, oy) = front / other pixel centres */
static int aa_pair(const OrcAA *p, int b, int64_t i, int ix, int iy, int64_t j, int jx, int jy, int horiz, real *w, int64_t *gain, int64_t *front,
                   AAEdge *e, real *fx, real *fy, real *ox, real *oy)
{
    const real *ri = p->rast + 4 * i, *rj = p->rast + 4 * j;
    const int ti = rast_tid(ri, p->T), tj = rast_tid(rj, p->T);
    if (ti == tj) return 0;
    int i_front;
    if (tj < 0) i_front = 1;
    else if (ti < 0) i_front = 0;
    else if (ri[2] < rj[2]) i_front = 1;
    else if (rj[2] < ri[2]) i_front = 0;
    else i_front = ti < tj;
    const real xi = px_ndc(ix, p->W), yi = px_ndc(iy, p->H), xj = px_ndc(jx, p->W), yj = px_ndc(jy, p->H);
    *fx = i_front ? xi : xj; *fy = i_front ? yi : yj; *ox = i_front ? xj : xi; *oy = i_front ? yj : yi;
    if (!aa_search(p, p->pos + b * p->pos_bs, i_front ? ti : tj, horiz, *fx, *fy, *ox, *oy, e)) return 0;
    int gain_front;
    if (e->t < RC(0.5f)) { *w = RC(0.5f) - e->t; gain_front = 1; }
    else if (e->t > RC(0.5f)) { *w = e->t - RC(0.5f); gain_front = 0; }
    else return 0;
    *front = i_front ? i : j;
    *gain = gain_front ? *front : (i_front ? j : i);
    return 1;
}

static OrcAA aa_make(int B, int H, int W, int C, const real *color, const real *rast, int64_t pos_bs, const real *pos, int T, const int32_t *tris,
                     const int32_t *adj)
{
    OrcAA p = {B, H, W, C, 0, T, pos_bs, color, rast, pos, tris, adj};
    return p;
}

/* forward: out_p = c_p + sum over the pairs p gains, in the order left, right, up, down, of w (c_q - c_p) */
void orc_antialias_fwd(int B, int H, int W, int C, const real *color, const real *rast, int64_t pos_bs, const real *pos, int T, const int32_t *tris,
                       const int32_t *adj, real *out)
{
    const OrcAA p = aa_make(B, H, W, C, color, rast, pos_bs, pos, T, tris, adj);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int ix = (int)(i % W), iy = (int)((i / W) % H), b = (int)(i / ((int64_t)W * H));
        const int nx[4] = {ix - 1, ix + 1, ix, ix}, ny[4] = {iy, iy, iy - 1, iy + 1};
        real wk[4]; int64_t jk[4]; int n = 0;
        for (int d = 0; d < 4; ++d) {
            if (nx[d] < 0 || nx[d] >= W || ny[d] < 0 || ny[d] >= H) continue;
            const int64_t j = ((int64_t)b * H + ny[d]) * W + nx[d];
            real w, fx, fy, ox, oy; int64_t gain, front; AAEdge e;
            if (aa_pair(&p, b, i, ix, iy, j, nx[d], ny[d], d < 2, &w, &gain, &front, &e, &fx, &fy, &ox, &oy) && gain == i) { wk[n] = w; jk[n] = j; ++n; }
        }
        for (int c = 0; c < C; ++c) {
            const real cs = color[i * C + c];
            real v = cs;
            for (int k = 0; k < n; ++k) v = v + wk[k] * (color[jk[k] * C + c] - cs);
            out[i * C + c] = v;
        }
    }
}

static void aa_edge_grad(const AAEdge *e, real px, real py, real s, real *dA, real *dB)
{
    const real ax = e->A.x - px * e->A.z, ay = e->A.y - py * e->A.z, bx = e->Bv.x - px * e->Bv.z, by = e->Bv.y - py * e->Bv.z;
    dA[0] += s * by; dA[1] -= s * bx; dA[3] += s * (py * bx - px * by);
    dB[0] -= s * ay; dB[1] += s * ax; dB[3] += s * (px * ay - py * ax);
}

/* backward, written as a scatter over the pairs (the kernel gathers): d_color (overwritten) and d_pos (accumulated) */
void orc_antialias_bwd(int B, int H, int W, int C, const real *color, const real *rast, int64_t pos_bs, const real *pos, int T, const int32_t *tris,
                       const int32_t *adj, const real *d_out, real *d_color, real *d_pos)
{
    const OrcAA p = aa_make(B, H, W, C, color, rast, pos_bs, pos, T, tris, adj);
    memcpy(d_color, d_out, sizeof(real) * (size_t)B * H * W * C);
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int ix = (int)(i % W), iy = (int)((i / W) % H), b = (int)(i / ((int64_t)W * H));
        for (int d = 0; d < 2; ++d) {                      /* the pairs (x, y)-(x+1, y) and (x, y)-(x, y+1) */
            const int jx = ix + (d == 0), jy = iy + (d == 1);
            if (jx >= W || jy >= H) continue;
            const int64_t j = ((int64_t)b * H + jy) * W + jx;
            real w, fx, fy, ox, oy; int64_t gain, front; AAEdge e;
            if (!aa_pair(&p, b, i, ix, iy, j, jx, jy, d == 0, &w, &gain, &front, &e, &fx, &fy, &ox, &oy)) continue;
            const int64_t other = gain == i ? j : i;
            real dLdt = 0;
            for (int c = 0; c < C; ++c) {
                const real g = d_out[gain * C + c];
                d_color[gain * C + c] -= w * g;
                d_color[other * C + c] += w * g;
                dLdt += g * (color[other * C + c] - color[gain * C + c]);
            }
            if (gain == front) dLdt = -dLdt;               /* f gains (1/2 - t)(c_o - c_f); o gains (t - 1/2)(c_f - c_o) */
            const real D = e.ef - e.eo;
            real *dA = d_pos + b * pos_bs + 4 * (size_t)e.va, *dB = d_pos + b * pos_bs + 4 * (size_t)e.vb;
            aa_edge_grad(&e, fx, fy, dLdt * (-e.eo / (D * D)), dA, dB);
            aa_edge_grad(&e, ox, oy, dLdt * (e.ef / (D * D)), dA, dB);
        }
    }
}
