/*
 * oracle/geometry.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C, fp32 by default, fp64 with -DORACLE_F64 for finite-difference checks of the hand-derived adjoints) of the
 * G-buffer producer's geometry gradients and screen-space derivatives: the barycentrics of the clip-space triangle and their adjoint
 * (rasterize backward), the adjoint of interpolate with respect to rast, edge adjacency, pixel-pair analytic antialiasing, rast_db,
 * interpolate's attribute derivatives out_da, their adjoints (d attr, d rast_db, d rast_db -> d pos), and interpolate's forward in the
 * kernel's operation order.  Every entry point that scatters (d pos of rasterize, rast_db and antialias, d attr of interpolate and
 * interpolate_da) takes a `terms` mode (test-only): 0 sums the per-pixel terms, 1 sums their absolute values, 2 counts the non-zero ones
 * (the bound on the rounding of summing them in another order); the one-writer outputs are the same in every mode.  No reference code
 * exists for them (nvdiffrast is absent); the semantics are those stated in nvdiffrecmc_b200/csrc/raster.cu.  Compile with
 * -ffp-contract=off: the antialias pair decisions, rast_db, out_da and d rast_db are evaluated in the same explicitly rounded operation
 * order as the CUDA kernels.  Loaded by oracle/geometry.py.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef ORACLE_F64
typedef double real;
#define R_FABS(x) fabs(x)
#define R_FMA(a, b, c) fma(a, b, c)
#else
typedef float real;
#define R_FABS(x) fabsf(x)
#define R_FMA(a, b, c) fmaf(a, b, c)
#endif
#define RC(x) ((real)(x))

typedef struct { real x, y, z; } v3;

int geo_sizeof_real(void) { return (int)sizeof(real); }

/* the term a scatter adds in mode `terms`: the term (0), its absolute value (1) or 1 when it is non-zero (2) */
static inline real term_of(real t, int terms) { return terms == 0 ? t : (terms == 1 ? R_FABS(t) : (real)(t != RC(0))); }

/* ================================================================================================================================
 * Geometry gradients of the G-buffer producer (nvdiffrecmc_b200/csrc/raster.cu states the semantics and the derivation):
 * barycentrics of the clip-space triangle and their adjoint, the adjoint of interpolate with respect to rast, edge adjacency,
 * and pixel-pair analytic antialiasing (Laine et al. 2020).  rast is [B,H,W,4] (u, v, z/w, id + 1) in `real`; pos is [V,4]
 * (pos_bs = 0) or [B,V,4] (pos_bs = 4V).  The antialias pair decisions are evaluated in the same operation order as the CUDA kernel.
 * ================================================================================================================================ */
static inline real px_ndc(int i, int n) { return ((real)i + RC(0.5f)) / (real)n * RC(2.0f) - RC(1.0f); }

/* triangle id of a rast pixel (id + 1 in channel 3), -1 for background and ids >= T */
static inline int rast_tid(const real *r, int T)
{
    const int id = (int)r[3] - 1;
    return id < T ? id : -1;
}

/* a_i = (x_i - px w_i, y_i - py w_i), s_i = a_{i+1} x a_{i+2}, S = (s0 + s1) + s2 (u = s0 / S, v = s1 / S); returns 0 when S == 0 */
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

void orc_raster_bwd(int B, int H, int W, int64_t pos_bs, const real *pos, int T, const int32_t *tris, const real *rast, const real *d_rast, real *d_pos,
                    int terms)
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
            d[0] += term_of(dax, terms); d[1] += term_of(day, terms); d[3] += term_of(-px * dax - py * day, terms);
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
            for (int c = 0; c < C; ++c) {             /* fused multiply-adds in channel order, as k_interpolate<2> */
                const real g = d_out[i * C + c], a2 = A[(size_t)tri[2] * C + c];
                du = R_FMA(g, A[(size_t)tri[0] * C + c] - a2, du);
                dv = R_FMA(g, A[(size_t)tri[1] * C + c] - a2, dv);
            }
        }
        d_rast[4 * i] = du; d_rast[4 * i + 1] = dv; d_rast[4 * i + 2] = 0; d_rast[4 * i + 3] = 0;
    }
}

/* d attr (accumulated) of interpolate: vertex k of the pixel's triangle gets w_k g, with (w0, w1, w2) = (u, v, (1 - u) - v), in pixel,
 * channel, vertex order (k_interpolate<1/2>'s terms) */
void orc_interpolate_bwd_attr(int B, int H, int W, int C, int64_t attr_bs, int T, const int32_t *tris, const real *rast, const real *d_out,
                              real *d_attr, int terms)
{
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int b = (int)(i / ((int64_t)W * H));
        const int id = rast_tid(rast + 4 * i, T);
        if (id < 0) continue;
        real *D = d_attr + b * attr_bs;
        const int32_t *tri = tris + 3 * (size_t)id;
        const real w[3] = {rast[4 * i], rast[4 * i + 1], RC(1) - rast[4 * i] - rast[4 * i + 1]};
        for (int c = 0; c < C; ++c) {
            const real g = d_out[i * C + c];
            for (int k = 0; k < 3; ++k) D[(size_t)tri[k] * C + c] += term_of(w[k] * g, terms);
        }
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

/* t of the crossing edge of each pixel's right (channel 0) and down (channel 1) pair, NaN where the pair has none; t = 1/2 means no
 * blend (rule 6).  Lets the tests check that a scene really produces the discrete cases it is built for. */
void orc_antialias_pair_t(int B, int H, int W, const real *rast, int64_t pos_bs, const real *pos, int T, const int32_t *tris, const int32_t *adj,
                          real *t_out)
{
    const OrcAA p = {B, H, W, 0, 0, T, pos_bs, NULL, rast, pos, tris, adj};
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int ix = (int)(i % W), iy = (int)((i / W) % H), b = (int)(i / ((int64_t)W * H));
        for (int d = 0; d < 2; ++d) {
            const int jx = ix + (d == 0), jy = iy + (d == 1);
            real w, fx, fy, ox, oy; int64_t gain, front; AAEdge e;
            e.t = (real)NAN;                              /* aa_pair leaves e.t unset without a crossing edge */
            if (jx < W && jy < H) aa_pair(&p, b, i, ix, iy, ((int64_t)b * H + jy) * W + jx, jx, jy, d == 0, &w, &gain, &front, &e, &fx, &fy, &ox, &oy);
            t_out[2 * i + d] = e.t;
        }
    }
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

static void aa_edge_grad(const AAEdge *e, real px, real py, real s, real *dA, real *dB, int terms)
{
    const real ax = e->A.x - px * e->A.z, ay = e->A.y - py * e->A.z, bx = e->Bv.x - px * e->Bv.z, by = e->Bv.y - py * e->Bv.z;
    dA[0] += term_of(s * by, terms); dA[1] += term_of(-(s * bx), terms); dA[3] += term_of(s * (py * bx - px * by), terms);
    dB[0] += term_of(-(s * ay), terms); dB[1] += term_of(s * ax, terms); dB[3] += term_of(s * (px * ay - py * ax), terms);
}

/* d_color (overwritten) as the kernel gathers it: start from g_p and walk p's pairs in the order left, right, up, down; a pair p gains
 * gives v = fma(-w, g_p, v), a pair the neighbour q gains v = fma(w, g_q, v) */
void orc_antialias_bwd_color(int B, int H, int W, int C, const real *color, const real *rast, int64_t pos_bs, const real *pos, int T,
                             const int32_t *tris, const int32_t *adj, const real *d_out, real *d_color)
{
    const OrcAA p = aa_make(B, H, W, C, color, rast, pos_bs, pos, T, tris, adj);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)B * H * W; ++i) {
        const int ix = (int)(i % W), iy = (int)((i / W) % H), b = (int)(i / ((int64_t)W * H));
        const int nx[4] = {ix - 1, ix + 1, ix, ix}, ny[4] = {iy, iy, iy - 1, iy + 1};
        real wk[4]; int64_t jk[4]; int self[4]; int n = 0;
        for (int d = 0; d < 4; ++d) {
            if (nx[d] < 0 || nx[d] >= W || ny[d] < 0 || ny[d] >= H) continue;
            const int64_t j = ((int64_t)b * H + ny[d]) * W + nx[d];
            real w, fx, fy, ox, oy; int64_t gain, front; AAEdge e;
            if (aa_pair(&p, b, i, ix, iy, j, nx[d], ny[d], d < 2, &w, &gain, &front, &e, &fx, &fy, &ox, &oy)) { wk[n] = w; jk[n] = j; self[n] = gain == i; ++n; }
        }
        for (int c = 0; c < C; ++c) {
            const real g = d_out[i * C + c];
            real v = g;
            for (int k = 0; k < n; ++k) v = self[k] ? R_FMA(-wk[k], g, v) : R_FMA(wk[k], d_out[jk[k] * C + c], v);
            d_color[i * C + c] = v;
        }
    }
}

/* backward, written as a scatter over the pairs: d_color (overwritten; orc_antialias_bwd_color gathers it in the kernel's order) and
 * d_pos (accumulated in the `terms` mode: two terms per pair and element, the front and the other pixel's) */
void orc_antialias_bwd(int B, int H, int W, int C, const real *color, const real *rast, int64_t pos_bs, const real *pos, int T, const int32_t *tris,
                       const int32_t *adj, const real *d_out, real *d_color, real *d_pos, int terms)
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
            aa_edge_grad(&e, fx, fy, dLdt * (-e.eo / (D * D)), dA, dB, terms);
            aa_edge_grad(&e, ox, oy, dLdt * (e.ef / (D * D)), dA, dB, terms);
        }
    }
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
void orc_rast_db_bwd(int B, int H, int W, int64_t pos_bs, const real *pos, int T, const int32_t *tris, const real *rast, const real *d_db, real *d_pos,
                     int terms)
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
            o[0] += term_of(dax + ey[k1] * d.w[k2] - ey[k2] * d.w[k1], terms);
            o[1] += term_of(day + ex[k2] * d.w[k1] - ex[k1] * d.w[k2], terms);
            o[3] += term_of(-d.px * dax - d.py * day + ex[k1] * d.y[k2] - ex[k2] * d.y[k1] + ey[k2] * d.x[k1] - ey[k1] * d.x[k2], terms);
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

/* d attr (accumulated in the `terms` mode) and d rast_db (overwritten) of out_da.  The third vertex's term is -(a0 + a1); its statistics
 * are those of a0 and a1 (|a0| + |a1|, and 1 when either is non-zero), because the kernel forms it from the group sums of a0 and a1. */
void orc_interpolate_da_bwd(int B, int H, int W, int C, int64_t attr_bs, const real *attr, int T, const int32_t *tris, const real *rast, const real *db,
                            int n, const int32_t *idx, const real *d_out_da, real *d_attr, real *d_db, int terms)
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
                D[(size_t)tri[0] * C + c] += term_of(a0, terms); D[(size_t)tri[1] * C + c] += term_of(a1, terms);
                if (terms == 0) D[(size_t)tri[2] * C + c] -= a0 + a1;
                else if (terms == 1) D[(size_t)tri[2] * C + c] += R_FABS(a0) + R_FABS(a1);
                else D[(size_t)tri[2] * C + c] += (real)(a0 != RC(0) || a1 != RC(0));
                e[0] = e[0] + gX * d0; e[1] = e[1] + gY * d0; e[2] = e[2] + gX * d1; e[3] = e[3] + gY * d1;
            }
        }
        for (int k = 0; k < 4; ++k) d_db[4 * i + k] = e[k];
    }
}
