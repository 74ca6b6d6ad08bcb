// raster.cu -- SURVEY section 8 row f2: primary visibility + attribute interpolation on the LBVH that the shadow rays already use, so the
// G-buffer of render/render.py:208-234 (dr.rasterize + dr.interpolate, nvdiffrast -- absent here) can be produced without a rasteriser.
//
//   k_rasterize   : one thread per pixel.  The pixel centre is un-projected with the inverse clip matrix to a near and a far point
//                   (NDC z = -1 / +1), the closest hit along that segment's line is found with bvh_closest (same fixed-order
//                   Moeller-Trumbore predicate as the shadow rays, ties broken by triangle id), and the result is written in
//                   nvdiffrast's `rast` convention: (u, v, z/w, triangle_id + 1), u / v = barycentric weights of vertex 0 / 1,
//                   0 in all channels for background.  Image row iy maps to NDC y = (iy + 0.5) / H * 2 - 1 (no flip, like dr.rasterize).
//                   Depth peeling (render/render.py:308-311 takes every layer from dr.DepthPeeler) is the same launch given a per-pixel
//                   state t_state [B,H,W], zero before layer 0, where t is measured along d = far - near:
//                     - layer k+1 is the closest hit with t > sep(t_prev), sep(t) = fl32(t * (1 + 2^-16)) (peel_sep, bvh_traverse.cuh),
//                       ties in t to the smaller triangle id, written as (u, v, z/w, id + 1) like any rast;
//                     - the state becomes that hit's t, or +inf when there is none; a +inf pixel writes zeros and skips traversal;
//                     - t_prev = 0 gives sep = 0 and mt_hit already requires t > 0, so layer 0 equals rasterize bit for bit.
//                   The separation is a deliberate choice: Moeller-Trumbore's closed bounds make a ray through a shared edge hit both
//                   triangles a few ulp apart, and a plain t > t_prev would return that surface again as a spurious layer.  Surfaces
//                   closer than 2^-16 t (about 128 ulp) along the ray merge into one layer.  Each layer is an ordinary rast: the
//                   backward below and antialias take it unchanged.
//                   There is no far-plane clipping: the search runs along the whole line beyond the near point (t < 1e16), so a surface
//                   beyond the far plane is returned with z/w > 1.
//                   Rounding (each step one IEEE round-to-nearest operation; oracle/mcoracle.c orc_invert4 / orc_rasterize restate it and
//                   the GPU equals that fp32 restatement bit for bit):
//                     - k_invert4: Gauss-Jordan in fp64, pivot = first row with the largest |a| (strict >), d = 1 / pivot (DIV), pivot
//                       row *= d (DMUL), other rows a = fma(-f, pivot row, a) (DFMA), each entry rounded to fp32 at the end;
//                     - pixel centre ((ix + 0.5) / W) * 2 - 1: the * 2 is exact, so FMUL + FADD and FFMA give the same value;
//                     - mul4: fma(m0, x, fma(m1, y, fma(m2, z, m3 * w))) per row; o = near.xyz / near.w and far.xyz / far.w by IEEE
//                       division, d = far - o;
//                     - hit point h = fma(d, t, o) per component, then q = mul4(mtx, h, 1), z/w = q.z / q.w (IEEE division);
//                     - rast = ((1 - u) - v, u, z/w, id + 1).
//   k_interpolate : out[b,y,x,:] = u * A[i0] + v * A[i1] + (1 - u - v) * A[i2]; backward scatters into dA with float atomics and, when
//                   the caller asks for it, writes d rast[...,0:2] = (sum_c g_c (A0_c - A2_c), sum_c g_c (A1_c - A2_c)) (one writer per pixel).
//                   Rounding: out = fma(u, A0, fma(v, A1, ((1 - u) - v) A2)); d rast accumulates du = fma(g_c, A0_c - A2_c, du) (likewise dv)
//                   in channel order from 0.  Both are bit-reproducible and equal the fp32 oracle (orc_interpolate_fwd,
//                   orc_interpolate_bwd_rast) bit for bit; d attr is an order-dependent float-atomic sum.
//
// Geometry gradients (render/render.py:284-291 antialiases every G-buffer layer; geometry/dlmesh.py:75 puts its alpha in the loss):
//
//   k_rasterize_bwd : d rast[...,0:2] -> d pos (clip space).  The forward stays the ray-traced launch; its barycentrics equal the
//                     perspective-correct ones of the clip-space triangle, written in terms of pos so they can be differentiated:
//                       pixel centre (px, py) in NDC, a_i = (x_i - px w_i, y_i - py w_i)       (the clip-space point P = sum_i b_i pos_i
//                       projects onto the pixel centre iff sum_i b_i a_i = 0, so b is proportional to the 2-D cross products)
//                       s0 = a1 x a2, s1 = a2 x a0, s2 = a0 x a1, S = s0 + s1 + s2,  u = s0 / S, v = s1 / S.
//                     With G = du u + dv v: dL/ds0 = (du - G)/S, dL/ds1 = (dv - G)/S, dL/ds2 = -G/S, and for s_i = a_{i+1} x a_{i+2}
//                       dL/da_k = dL/ds_{k+2} (a_{k+1}.y, -a_{k+1}.x) + dL/ds_{k+1} (-a_{k+2}.y, a_{k+2}.x),
//                       d x_k = dL/da_k.x,  d y_k = dL/da_k.y,  d w_k = -px dL/da_k.x - py dL/da_k.y.
//                     z/w and the id carry no gradient (the reference computes depth under no_grad, render.py:228-234).
//                     One thread per pixel; warp-aggregated float atomics (see the kernel).
//
// Screen-space derivatives (render/render.py:225-234 builds the denoiser's depth guide from them; nvdiffrast's layout):
//
//   k_rast_db       : rast_db[b,y,x] = (du/dX, du/dY, dv/dX, dv/dY), X the column and Y the row index in pixels, for the triangle id
//                     stored in rast, from the clip-space pos alone.  With the terms above the px py products cancel, so every s_i is
//                     affine in (px, py):
//                       ds_i/dpx = y_{i+1} w_{i+2} - w_{i+1} y_{i+2},   ds_i/dpy = w_{i+1} x_{i+2} - x_{i+1} w_{i+2},
//                       du/dpx = (ds0/dpx - u dS/dpx) / S  (likewise py, and v with s1),   d/dX = (2/W) d/dpx,  d/dY = (2/H) d/dpy.
//                     All four channels are 0 for background, ids >= T and S == 0.  Every operation is explicitly rounded in one fixed
//                     order (the fp32 build of oracle/geometry.c evaluates the same order), so rast_db is bit-reproducible.  A vertex
//                     with w <= 0 needs no special case: the projective formula holds wherever the pixel has a hit.  One launch after
//                     rasterize or any peel layer; k_rasterize is unchanged.
//   k_interpolate_da: out_da[b,y,x,2k:2k+2] = (dA/dX, dA/dY) of the k-th selected attribute A (attribute-major, nvdiffrast's layout):
//                       dA/dX = db.x (A0 - A2) + db.z (A1 - A2),   dA/dY = db.y (A0 - A2) + db.w (A1 - A2),   0 without a hit.
//                     The selection ('all' or up to 32 indices, repeats allowed) is passed by value.  out_da does not depend on u, v.
//                     Backward: d attr by float atomics (dA0 += gX db.x + gY db.y, dA1 += gX db.z + gY db.w, dA2 -= both), and
//                     d rast_db = (sum gX (A0 - A2), sum gY (A0 - A2), sum gX (A1 - A2), sum gY (A1 - A2)) over the selection, one writer
//                     per pixel in the selection's order (bit-reproducible).
//   k_rasterize_bwd<true>: d rast[...,0:2] (optional) and d rast_db -> d pos.  The rast_db term differentiates the formula above with
//                     respect to s_i, S and the ds_i/dp terms, then maps dL/ds_i to d pos like the barycentric term and adds the direct
//                     terms of ds_i/dp in (x_k, y_k, w_k).  k_rasterize_bwd<false> is the d rast-only kernel.
//   k_aa_topo_*     : edge adjacency of a triangle list: the 3T undirected edge keys go into an open-addressing hash table (64-bit
//                     atomicCAS, linear probing) that counts the triangles on each key and keeps the first two; a second pass resolves
//                     adj[t,k] = the other triangle on edge (tri[t,k], tri[t,(k+1)%3]), -1 on a boundary edge, -2 with three or more.
//                     Only the set of triangles on an edge decides the answer, so it does not depend on insertion order.
//   k_antialias     : pixel-pair analytic antialiasing (Laine et al. 2020, "Modular Primitives for High-Performance Differentiable
//                     Rendering"), with these semantics:
//                       1. pairs: horizontally / vertically adjacent pixels whose triangle ids differ;
//                       2. front side: covered beats background; between triangles the smaller z/w, ties to the smaller id.  f / F = the
//                          front pixel / its triangle, o = the other pixel;
//                       3. candidate edges of F: boundary (-1), shared by >= 3 triangles (-2), or F and its neighbour face opposite ways
//                          (sign of det[[x0,y0,w0],[x1,y1,w1],[x2,y2,w2]]); edges with an endpoint at w <= 0 are skipped;
//                       4. axis rule: horizontal pairs take edges with |dY| >= |dX| in pixels, vertical pairs the others;
//                       5. crossing: e(p) = a_A x a_B (w_A w_B times the affine screen-space edge function), t = e_f / (e_f - e_o) when
//                          e_f and e_o have strictly opposite signs; the smallest t of the candidate edges wins;
//                       6. blend: o gains max(0, t - 1/2) (c_f - c_o), f gains max(0, 1/2 - t) (c_o - c_f); a pixel's <= 4 pairs add
//                          in the fixed order left, right, up, down.
//                     The pair logic (rules 1-5 and the d pos scatter) is csrc/antialias.cuh, shared with csrc/composite.cu.
//                     The forward is a per-pixel gather (each thread evaluates its own <= 4 pairs), so it is bit-deterministic without
//                     colour atomics.  The backward gathers d color the same way; d pos (dt/d(x, y, w) of the crossing edge's endpoints,
//                     dt/de_f = -e_o / D^2, dt/de_o = e_f / D^2 with D = e_f - e_o) is scattered with float atomics by the pixel that owns
//                     the pair (the left / upper one).  Nothing flows through ids, the facing test or the front test.
//                     The pair arithmetic uses explicitly rounded operations (no FMA contraction) so that the CPU restatement in
//                     oracle/geometry.c, compiled with -ffp-contract=off, makes the same discrete decisions.
//                     Rounding of the outputs with one writer per pixel (both bit-reproducible and equal to the fp32 oracle bit for bit):
//                       - forward: v = c_p, then per pair p gains, in pair order, v = v + w (c_q - c_p), each operation rounded
//                         (orc_antialias_fwd);
//                       - d color: v = g_p, then per pair in pair order v = fma(-w, g_p, v) when p gains and v = fma(w, g_q, v) when q
//                         gains (orc_antialias_bwd_color); it does not depend on whether d pos is computed.
//                     d pos is an order-dependent float-atomic sum, within float rounding of the oracle's scatter.
#include "ctx.h"
#include "bvh_traverse.cuh"
#include "antialias.cuh"

namespace {

struct RasterParams {
    BvhView bvh;
    const float *mtx, *inv;      // [B,4,4] row-major, clip = mtx * (p, 1)
    int B, H, W;
    float *rast;
    float *t_state;              // [B,H,W] depth-peeling state (t of the last layer's hit, +inf when exhausted), or null for plain rasterize
};

__device__ __forceinline__ void mul4(const float *__restrict__ m, float x, float y, float z, float w, float (&o)[4])
{
#pragma unroll
    for (int r = 0; r < 4; ++r) o[r] = fmaf(__ldg(m + 4 * r), x, fmaf(__ldg(m + 4 * r + 1), y, fmaf(__ldg(m + 4 * r + 2), z, __ldg(m + 4 * r + 3) * w)));
}

__global__ void __launch_bounds__(128) k_rasterize(const RasterParams p)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = (int64_t)p.B * p.H * p.W;
    if (i >= n) return;
    int b, iy, ix;
    px_decode(i, p.H, p.W, b, iy, ix);
    const float x = ((float)ix + 0.5f) / (float)p.W * 2.0f - 1.0f, y = ((float)iy + 0.5f) / (float)p.H * 2.0f - 1.0f;
    float a[4], c[4];
    mul4(p.inv + 16 * b, x, y, -1.0f, 1.0f, a);
    mul4(p.inv + 16 * b, x, y, 1.0f, 1.0f, c);
    const f3 o = F3(__fdiv_rn(a[0], a[3]), __fdiv_rn(a[1], a[3]), __fdiv_rn(a[2], a[3]));
    const f3 f = F3(__fdiv_rn(c[0], c[3]), __fdiv_rn(c[1], c[3]), __fdiv_rn(c[2], c[3]));
    const f3 d = F3(__fsub_rn(f.x, o.x), __fsub_rn(f.y, o.y), __fsub_rn(f.z, o.z));
    float t_lo = 0.0f;
    if (p.t_state) {
        const float t_prev = p.t_state[i];
        if (t_prev == INFINITY) { reinterpret_cast<float4 *>(p.rast)[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f); return; }
        t_lo = peel_sep(t_prev);
    }
    float t, u, v;
    const int id = bvh_closest(p.bvh, o, d, t_lo, t, u, v);
    float4 out = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (id >= 0) {
        const f3 h = F3(__fmaf_rn(d.x, t, o.x), __fmaf_rn(d.y, t, o.y), __fmaf_rn(d.z, t, o.z));
        float q[4];
        mul4(p.mtx + 16 * b, h.x, h.y, h.z, 1.0f, q);
        out = make_float4(__fsub_rn(__fsub_rn(1.0f, u), v), u, __fdiv_rn(q[2], q[3]), (float)(id + 1));
    }
    reinterpret_cast<float4 *>(p.rast)[i] = out;
    if (p.t_state) p.t_state[i] = id >= 0 ? t : INFINITY;
}

// inverse of B row-major 4x4 matrices, Gauss-Jordan with partial pivoting in fp64 (one thread per matrix; a singular matrix gives NaNs,
// i.e. an all-background image)
__global__ void k_invert4(const float *__restrict__ m, float *__restrict__ inv, int B)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    double a[4][8];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) { a[r][c] = (double)m[16 * b + 4 * r + c]; a[r][4 + c] = r == c ? 1.0 : 0.0; }
    for (int col = 0; col < 4; ++col) {
        int piv = col;
        for (int r = col + 1; r < 4; ++r) if (fabs(a[r][col]) > fabs(a[piv][col])) piv = r;
        for (int c = 0; c < 8; ++c) { const double t = a[col][c]; a[col][c] = a[piv][c]; a[piv][c] = t; }
        const double d = 1.0 / a[col][col];
        for (int c = 0; c < 8; ++c) a[col][c] *= d;
        for (int r = 0; r < 4; ++r) {
            if (r == col) continue;
            const double f = a[r][col];
            for (int c = 0; c < 8; ++c) a[r][c] = __fma_rn(-f, a[col][c], a[r][c]);
        }
    }
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) inv[16 * b + 4 * r + c] = (float)a[r][4 + c];
}

struct InterpParams {
    const float *attr; int64_t attr_bs; int V, C;
    const int32_t *tris; int T;
    const float4 *rast;
    const float *dout; float *out, *dattr;
    float4 *drast;
    int64_t npx, px_per_batch;
};

// MODE 0: forward; 1: backward to the attributes; 2: backward to rast (d_rast, every pixel written) and, when dattr != null, to the attributes.
template <int MODE>
__global__ void __launch_bounds__(256) k_interpolate(const InterpParams p)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.npx) return;
    const float4 r = __ldg(p.rast + i);
    const int id = (int)r.w - 1;
    if (id < 0 || id >= p.T) {
        if (MODE == 0) for (int c = 0; c < p.C; ++c) p.out[i * p.C + c] = 0.0f;
        if (MODE == 2) p.drast[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        return;
    }
    const int i0 = __ldg(p.tris + 3 * (size_t)id), i1 = __ldg(p.tris + 3 * (size_t)id + 1), i2 = __ldg(p.tris + 3 * (size_t)id + 2);
    const int64_t base = (i / p.px_per_batch) * p.attr_bs;
    const float w0 = r.x, w1 = r.y, w2 = 1.0f - r.x - r.y;
    float du = 0.0f, dv = 0.0f;
    for (int c = 0; c < p.C; ++c) {
        if (MODE == 0) {
            const float *A = p.attr + base;
            p.out[i * p.C + c] = fmaf(w0, __ldg(A + (size_t)i0 * p.C + c), fmaf(w1, __ldg(A + (size_t)i1 * p.C + c), w2 * __ldg(A + (size_t)i2 * p.C + c)));
        } else {
            const float g = __ldg(p.dout + i * p.C + c);
            if (MODE == 1 || p.dattr) {
                float *D = p.dattr + base;
                atomicAdd(D + (size_t)i0 * p.C + c, w0 * g); atomicAdd(D + (size_t)i1 * p.C + c, w1 * g); atomicAdd(D + (size_t)i2 * p.C + c, w2 * g);
            }
            if (MODE == 2) {
                const float *A = p.attr + base;
                const float a2 = __ldg(A + (size_t)i2 * p.C + c);
                du = __fmaf_rn(g, __fsub_rn(__ldg(A + (size_t)i0 * p.C + c), a2), du);
                dv = __fmaf_rn(g, __fsub_rn(__ldg(A + (size_t)i1 * p.C + c), a2), dv);
            }
        }
    }
    if (MODE == 2) p.drast[i] = make_float4(du, dv, 0.0f, 0.0f);
}

#define MCS_DIFF_ATTRS_MAX 32

struct InterpDaParams {
    const float *attr; int64_t attr_bs; int V, C;
    const int32_t *tris; int T;
    const float4 *rast, *db;
    float *out_da;                              // forward: [B,H,W,2n]
    const float *dout_da; float *dattr;         // backward: d out_da [B,H,W,2n]; d attr (caller-zeroed, atomics) or null
    float4 *ddb;                                // backward: d rast_db (every pixel written) or null
    int64_t npx, px_per_batch;
    int n, all;                                 // n selected attributes; all != 0: the k-th is attribute k, else idx[k]
    int32_t idx[MCS_DIFF_ATTRS_MAX];
};

// out_da and its backward (semantics in the file header).  Differences and products are explicitly rounded so the forward and
// d rast_db equal the fp32 oracle bit for bit.
// d attr: lanes of a warp that hit the same triangle of the same image are grouped once per pixel (as k_rasterize_bwd) and sum their
// per-vertex terms once per selected attribute (warp_group_sum).
template <bool BWD>
__global__ void __launch_bounds__(256) k_interpolate_da(const InterpDaParams p)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool agg = BWD && p.dattr;      // then every lane of the warp reaches __match_any_sync (no early exit before it)
    if (i >= p.npx && !agg) return;
    int id = -1;
    if (i < p.npx) {
        id = (int)__ldg(p.rast + i).w - 1;
        if (id >= p.T) id = -1;
    }
    const int n = p.n;
    if (id < 0 && i < p.npx) {
        if (!BWD) for (int k = 0; k < 2 * n; ++k) p.out_da[i * 2 * n + k] = 0.0f;
        if (BWD && p.ddb) p.ddb[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    const unsigned lane = threadIdx.x & 31u;
    unsigned peers = 1u << lane;
    if (agg) {
        const long long key = id >= 0 ? (long long)(i / p.px_per_batch) * p.T + id : -1ll - (long long)lane;
        peers = __match_any_sync(0xFFFFFFFFu, key);
    }
    if (id < 0) return;
    const int i0 = __ldg(p.tris + 3 * (size_t)id), i1 = __ldg(p.tris + 3 * (size_t)id + 1), i2 = __ldg(p.tris + 3 * (size_t)id + 2);
    const int64_t base = (i / p.px_per_batch) * p.attr_bs;
    const float4 db = __ldg(p.db + i);
    const bool need_a = !BWD || p.ddb;
    float e0 = 0.0f, e1 = 0.0f, e2 = 0.0f, e3 = 0.0f;
    for (int k = 0; k < n; ++k) {
        const int c = p.all ? k : p.idx[k];
        float d0 = 0.0f, d1 = 0.0f;
        if (need_a) {
            const float *A = p.attr + base;
            const float a2 = __ldg(A + (size_t)i2 * p.C + c);
            d0 = __fsub_rn(__ldg(A + (size_t)i0 * p.C + c), a2);
            d1 = __fsub_rn(__ldg(A + (size_t)i1 * p.C + c), a2);
        }
        if (!BWD) {
            p.out_da[(i * n + k) * 2] = __fadd_rn(__fmul_rn(db.x, d0), __fmul_rn(db.z, d1));
            p.out_da[(i * n + k) * 2 + 1] = __fadd_rn(__fmul_rn(db.y, d0), __fmul_rn(db.w, d1));
        } else {
            const float gX = __ldg(p.dout_da + (i * n + k) * 2), gY = __ldg(p.dout_da + (i * n + k) * 2 + 1);
            if (p.dattr) {
                float a[2] = {gX * db.x + gY * db.y, gX * db.z + gY * db.w};
                const bool issue = peers == (1u << lane) ? gX != 0.0f || gY != 0.0f : warp_group_sum(peers, a) && (a[0] != 0.0f || a[1] != 0.0f);
                if (issue) {
                    float *D = p.dattr + base;
                    atomicAdd(D + (size_t)i0 * p.C + c, a[0]); atomicAdd(D + (size_t)i1 * p.C + c, a[1]); atomicAdd(D + (size_t)i2 * p.C + c, -(a[0] + a[1]));
                }
            }
            if (p.ddb) {
                e0 = __fadd_rn(e0, __fmul_rn(gX, d0)); e1 = __fadd_rn(e1, __fmul_rn(gY, d0));
                e2 = __fadd_rn(e2, __fmul_rn(gX, d1)); e3 = __fadd_rn(e3, __fmul_rn(gY, d1));
            }
        }
    }
    if (BWD && p.ddb) p.ddb[i] = make_float4(e0, e1, e2, e3);
}

// ------------------------------------------------------------------------------------------------------------------------------------
// rasterize backward: d rast[...,0:2] -> d pos through u = s0 / S, v = s1 / S (derivation in the file header)
// ------------------------------------------------------------------------------------------------------------------------------------
struct RastBwdParams {
    const float *pos; int64_t pos_bs; int V;
    const int32_t *tris; int T;
    const float4 *rast, *drast;
    int B, H, W;
    float *dpos;
    const float4 *drast_db;      // k_rasterize_bwd<true>: d rast_db (drast may then be null)
    float4 *rast_db;             // k_rast_db: output
};

// triangle id of the clip-space mesh seen from pixel centre (px, py) (file header): vertex ids, (x, y, w), a_k, s_k = a_{k+1} x a_{k+2}
// and S = (s0 + s1) + s2
struct ClipTri { int vi[3]; float x[3], y[3], w[3]; float2 a[3]; float s[3], S; };

__device__ __forceinline__ ClipTri clip_tri(const float *P, const int32_t *tris, int id, float px, float py)
{
    ClipTri c;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        c.vi[k] = __ldg(tris + 3 * (size_t)id + k);
        const float *q = P + 4 * (size_t)c.vi[k];
        c.x[k] = __ldg(q); c.y[k] = __ldg(q + 1); c.w[k] = __ldg(q + 3);
        c.a[k] = clip_a(c.x[k], c.y[k], c.w[k], px, py);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) c.s[k] = clip_edge(c.a[k == 2 ? 0 : k + 1], c.a[k == 0 ? 2 : k - 1]);
    c.S = __fadd_rn(__fadd_rn(c.s[0], c.s[1]), c.s[2]);
    return c;
}

// rast_db (file header): one thread per pixel, explicitly rounded in the order of oracle/geometry.c's orc_rast_db
__global__ void __launch_bounds__(256) k_rast_db(const RastBwdParams p)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = (int64_t)p.B * p.H * p.W;
    if (i >= n) return;
    const float4 r = __ldg(p.rast + i);
    const int id = (int)r.w - 1;
    float4 out = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    if (id >= 0 && id < p.T) {
        int b, iy, ix;
        px_decode(i, p.H, p.W, b, iy, ix);
        const ClipTri c = clip_tri(p.pos + (int64_t)b * p.pos_bs, p.tris, id, px_ndc(ix, p.W), px_ndc(iy, p.H));
        const float S = c.S;
        if (S != 0.0f) {
            float dx[3], dy[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int k1 = k == 2 ? 0 : k + 1, k2 = k == 0 ? 2 : k - 1;
                dx[k] = __fsub_rn(__fmul_rn(c.y[k1], c.w[k2]), __fmul_rn(c.w[k1], c.y[k2]));
                dy[k] = __fsub_rn(__fmul_rn(c.w[k1], c.x[k2]), __fmul_rn(c.x[k1], c.w[k2]));
            }
            const float dSx = __fadd_rn(__fadd_rn(dx[0], dx[1]), dx[2]), dSy = __fadd_rn(__fadd_rn(dy[0], dy[1]), dy[2]);
            const float u = __fdiv_rn(c.s[0], S), v = __fdiv_rn(c.s[1], S);
            const float sx = __fdiv_rn(2.0f, (float)p.W), sy = __fdiv_rn(2.0f, (float)p.H);
            out.x = __fmul_rn(__fdiv_rn(__fsub_rn(dx[0], __fmul_rn(u, dSx)), S), sx);
            out.y = __fmul_rn(__fdiv_rn(__fsub_rn(dy[0], __fmul_rn(u, dSy)), S), sy);
            out.z = __fmul_rn(__fdiv_rn(__fsub_rn(dx[1], __fmul_rn(v, dSx)), S), sx);
            out.w = __fmul_rn(__fdiv_rn(__fsub_rn(dy[1], __fmul_rn(v, dSy)), S), sy);
        }
    }
    p.rast_db[i] = out;
}

// Lanes of a warp that hit the same triangle of the same image sum their 9 vertex gradients with shuffles (warp_group_sum) and one
// lane issues the atomics: 0.093 ms against 0.354 ms with 9 atomics per pixel at 8 x 512^2 on the bench mesh (H100 80GB HBM3, 400 W),
// where consecutive pixels of a row mostly share a triangle.
// DB: d rast (may be null) and d rast_db; without DB this is the d rast-only kernel.
template <bool DB>
__global__ void __launch_bounds__(256) k_rasterize_bwd(const RastBwdParams p)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = (int64_t)p.B * p.H * p.W;
    int id = -1, b = 0;
    float gv[3][3] = {};         // (d x, d y, d w) of vertex k
    int vi[3] = {0, 0, 0};
    if (i < n) {
        const float4 r = __ldg(p.rast + i);
        id = (int)r.w - 1;
        const float4 g = DB && !p.drast ? make_float4(0.0f, 0.0f, 0.0f, 0.0f) : __ldg(p.drast + i);
        float4 h = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        bool zero = g.x == 0.0f && g.y == 0.0f;
        if (DB) {
            h = __ldg(p.drast_db + i);
            zero = zero && h.x == 0.0f && h.y == 0.0f && h.z == 0.0f && h.w == 0.0f;
        }
        if (id >= p.T || zero) id = -1;
        if (id >= 0) {
            int iy, ix;
            px_decode(i, p.H, p.W, b, iy, ix);
            const float px = px_ndc(ix, p.W), py = px_ndc(iy, p.H);
            const ClipTri c = clip_tri(p.pos + (int64_t)b * p.pos_bs, p.tris, id, px, py);
#pragma unroll
            for (int k = 0; k < 3; ++k) vi[k] = c.vi[k];
            const float S = c.S;
            if (S == 0.0f) {
                id = -1;
            } else {
                const float u = c.s[0] / S, v = c.s[1] / S, G = g.x * u + g.y * v;
                float gs[3] = {(g.x - G) / S, (g.y - G) / S, -G / S};
                float ex[3], ey[3];
                if (DB) {
                    // L = sum_{c = u, v; p = px, py} h_cp (ds_c/dp - c dS/dp) / S with h the pixel-scaled d rast_db; the ds_i/dp terms
                    // are contractible here, unlike k_rast_db's
                    float dx[3], dy[3];
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        const int k1 = k == 2 ? 0 : k + 1, k2 = k == 0 ? 2 : k - 1;
                        dx[k] = c.y[k1] * c.w[k2] - c.w[k1] * c.y[k2];
                        dy[k] = c.w[k1] * c.x[k2] - c.x[k1] * c.w[k2];
                    }
                    const float dSx = dx[0] + dx[1] + dx[2], dSy = dy[0] + dy[1] + dy[2];
                    const float sx = 2.0f / (float)p.W, sy = 2.0f / (float)p.H;
                    const float hxu = h.x * sx, hyu = h.y * sy, hxv = h.z * sx, hyv = h.w * sy;
                    const float Kx = hxu * u + hxv * v, Ky = hyu * u + hyv * v;
                    ex[0] = (hxu - Kx) / S; ex[1] = (hxv - Kx) / S; ex[2] = -Kx / S;          // dL / d(ds_i/dpx)
                    ey[0] = (hyu - Ky) / S; ey[1] = (hyv - Ky) / S; ey[2] = -Ky / S;          // dL / d(ds_i/dpy)
                    const float mu = -(hxu * dSx + hyu * dSy) / S, mv = -(hxv * dSx + hyv * dSy) / S;      // dL/du, dL/dv
                    const float Ldb = (hxu * (dx[0] - u * dSx) + hyu * (dy[0] - u * dSy) + hxv * (dx[1] - v * dSx) + hyv * (dy[1] - v * dSy)) / S;
                    const float GS = -(Ldb + mu * u + mv * v) / S;                                  // dL/dS
                    gs[0] += mu / S + GS; gs[1] += mv / S + GS; gs[2] += GS;
                }
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const int k1 = k == 2 ? 0 : k + 1, k2 = k == 0 ? 2 : k - 1;
                    float gx = gs[k2] * c.a[k1].y - gs[k1] * c.a[k2].y;
                    float gy = gs[k1] * c.a[k2].x - gs[k2] * c.a[k1].x;
                    float gw = -px * gx - py * gy;
                    if (DB) {
                        gx += ey[k1] * c.w[k2] - ey[k2] * c.w[k1];
                        gy += ex[k2] * c.w[k1] - ex[k1] * c.w[k2];
                        gw += ex[k1] * c.y[k2] - ex[k2] * c.y[k1] + ey[k2] * c.x[k1] - ey[k1] * c.x[k2];
                    }
                    gv[k][0] = gx; gv[k][1] = gy; gv[k][2] = gw;
                }
            }
        }
    }
    const unsigned lane = threadIdx.x & 31u;
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, id >= 0 ? (long long)b * p.T + id : -1ll - (long long)lane);
    if (id < 0) return;
    bool lead = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) lead = warp_group_sum(peers, gv[k]);
    if (!lead) return;
    float *D = p.dpos + (int64_t)b * p.pos_bs;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float *d = D + 4 * (size_t)vi[k];
        atomicAdd(d, gv[k][0]); atomicAdd(d + 1, gv[k][1]); atomicAdd(d + 3, gv[k][2]);
    }
}

// ------------------------------------------------------------------------------------------------------------------------------------
// edge adjacency: open-addressing hash of the undirected edge keys (workspace: keys[cap] u64, count[cap] i32, first two triangles[cap][2])
// ------------------------------------------------------------------------------------------------------------------------------------
#define AA_EMPTY 0xFFFFFFFFFFFFFFFFull

__device__ __forceinline__ unsigned long long aa_hash(unsigned long long k)
{
    k ^= k >> 33; k *= 0xFF51AFD7ED558CCDull; k ^= k >> 33; k *= 0xC4CEB9FE1A85EC53ull; k ^= k >> 33;
    return k;
}

__global__ void __launch_bounds__(256) k_aa_topo_insert(const int32_t *__restrict__ tris, int T, unsigned long long *keys, int *cnt, int *first2,
                                                        unsigned long long mask, int32_t *__restrict__ slot)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * (int64_t)T) return;
    const int t = (int)(i / 3), k = (int)(i % 3);
    const uint32_t a = (uint32_t)__ldg(tris + 3 * (size_t)t + k), c = (uint32_t)__ldg(tris + 3 * (size_t)t + (k == 2 ? 0 : k + 1));
    const unsigned long long key = ((unsigned long long)min(a, c) << 32) | max(a, c);
    unsigned long long h = aa_hash(key) & mask;
    for (;;) {
        const unsigned long long prev = atomicCAS(keys + h, AA_EMPTY, key);
        if (prev == AA_EMPTY || prev == key) break;
        h = (h + 1) & mask;
    }
    const int n = atomicAdd(cnt + h, 1);
    if (n < 2) first2[2 * h + n] = t;
    slot[i] = (int32_t)h;
}

__global__ void __launch_bounds__(256) k_aa_topo_resolve(int T, const int *__restrict__ cnt, const int *__restrict__ first2, int32_t *adj)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 3 * (int64_t)T) return;
    const int t = (int)(i / 3);
    const int h = adj[i];
    const int c = __ldg(cnt + h);
    int r;
    if (c == 1) r = -1;
    else if (c >= 3) r = -2;
    else { const int f0 = __ldg(first2 + 2 * (size_t)h); r = f0 == t ? __ldg(first2 + 2 * (size_t)h + 1) : f0; }
    adj[i] = r;
}

static uint64_t aa_topo_capacity(int32_t T)
{
    uint64_t cap = 64;
    while (cap < 4 * (uint64_t)T) cap <<= 1;     // >= 4/3 slots per key even for a triangle soup (3T distinct edges), ~2.7 for a closed mesh
    return cap;
}

// ------------------------------------------------------------------------------------------------------------------------------------
// antialias
// ------------------------------------------------------------------------------------------------------------------------------------
struct AAParams {
    AAGeom g;
    const float *color; int C;
    float *out;
    const float *dout; float *dcolor, *dpos;
    int64_t npx;
};

// One thread per pixel: its pairs (antialias.cuh), then the blend of every channel as a per-pixel gather.
template <bool BWD>
__global__ void __launch_bounds__(256) k_antialias(const AAParams p)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.npx) return;
    int b, iy, ix;
    px_decode(i, p.g.H, p.g.W, b, iy, ix);
    const float4 r = __ldg(p.g.rast + i);
    const int C = p.C;
    const AAPairs pr = aa_pixel_pairs<BWD>(p.g, i, b, iy, ix, r, p.dpos, [&](bool gain_self, int, int64_t j) {
        const int64_t gi = gain_self ? i : j, oi = gain_self ? j : i;
        float dLdt = 0.0f;
        for (int c = 0; c < C; ++c) dLdt = fmaf(__ldg(p.dout + gi * C + c), __ldg(p.color + oi * C + c) - __ldg(p.color + gi * C + c), dLdt);
        return dLdt;
    });
    if (!BWD) {
        const float *cp = p.color + i * C;
        float *o = p.out + i * C;
        for (int c = 0; c < C; ++c) {
            const float cs = __ldg(cp + c);
            float v = cs;
#pragma unroll
            for (int d = 0; d < 4; ++d)
                if (pr.on[d] && pr.self[d]) v = __fadd_rn(v, __fmul_rn(pr.w[d], __fsub_rn(__ldg(p.color + pr.j[d] * C + c), cs)));
            o[c] = v;
        }
    } else if (p.dcolor) {
        // out_p = c_p + sum_{pairs p gains} w (c_q - c_p);  out_q = c_q + w (c_p - c_q) for the pairs q gains
        const float *gp = p.dout + i * C;
        float *dc = p.dcolor + i * C;
        for (int c = 0; c < C; ++c) {
            const float g = __ldg(gp + c);
            float v = g;
#pragma unroll
            for (int d = 0; d < 4; ++d)
                if (pr.on[d]) v = pr.self[d] ? __fmaf_rn(-pr.w[d], g, v) : __fmaf_rn(pr.w[d], __ldg(p.dout + pr.j[d] * C + c), v);
            dc[c] = v;
        }
    }
}

// Nearest-texel material fetch (stand-in for dr.texture with filter_mode='nearest', render/texture.py:66-75): out[i,:] = tex[idx[i],:];
// the backward pass scatters with float atomics (torch's index backward sorts the 2 M indices first and is ~8x slower).
template <bool BWD>
__global__ void __launch_bounds__(256) k_texel_fetch(const float *__restrict__ tex, const int64_t *__restrict__ idx, int64_t n, int C, int64_t T,
                                                     float *__restrict__ out, const float *__restrict__ dout, float *__restrict__ dtex)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t t = __ldg(idx + i);
    const bool ok = t >= 0 && t < T;
    for (int c = 0; c < C; ++c) {
        if (!BWD) out[i * C + c] = ok ? __ldg(tex + t * C + c) : 0.0f;
        else if (ok) atomicAdd(dtex + t * C + c, __ldg(dout + i * C + c));
    }
}

}  // namespace

extern "C" {

static int rasterize_launch(mcs_ctx *c, const float *mtx, int32_t B, int32_t H, int32_t W, float *t_state, float *rast, mcs_stream stream)
{
    if (int e = mcs_buf_reserve(c->mtx_inv, sizeof(float) * 16 * (size_t)B, (cudaStream_t)stream)) return e;
    float *inv_mtx = (float *)c->mtx_inv.p;
    k_invert4<<<(B + 63) / 64, 64, 0, (cudaStream_t)stream>>>(mtx, inv_mtx, B);
    MCS_LAUNCH_CHECK();
    RasterParams p{};
    p.bvh = BvhView{(const float4 *)c->nodes.p, (const float4 *)c->tris.p, nullptr, nullptr};
    p.mtx = mtx; p.inv = inv_mtx; p.B = B; p.H = H; p.W = W; p.rast = rast; p.t_state = t_state;
    const int64_t n = (int64_t)B * H * W;
    k_rasterize<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_rasterize(mcs_ctx *c, const float *mtx, int32_t B, int32_t H, int32_t W, float *rast, mcs_stream stream)
{
    MCS_REQUIRE(c && c->T > 0, "mcs_rasterize: no acceleration structure built (call mcs_bvh_build first)");
    MCS_REQUIRE(mtx && rast && B > 0 && H > 0 && W > 0, "mcs_rasterize: bad arguments");
    return rasterize_launch(c, mtx, B, H, W, nullptr, rast, stream);
}

int mcs_rasterize_peel(mcs_ctx *c, const float *mtx, int32_t B, int32_t H, int32_t W, float *t_state, float *rast, mcs_stream stream)
{
    MCS_REQUIRE(c && c->T > 0, "mcs_rasterize_peel: no acceleration structure built (call mcs_bvh_build first)");
    MCS_REQUIRE(mtx && t_state && rast && B > 0 && H > 0 && W > 0, "mcs_rasterize_peel: bad arguments");
    return rasterize_launch(c, mtx, B, H, W, t_state, rast, stream);
}

static int interp_common(InterpParams &p, const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T,
                         const float *rast, int32_t B, int32_t H, int32_t W)
{
    MCS_REQUIRE(attr && tris && rast && V > 0 && C > 0 && T > 0 && B > 0 && H > 0 && W > 0, "mcs_interpolate: bad arguments");
    p.attr = attr; p.attr_bs = attr_batch_stride; p.V = V; p.C = C; p.tris = tris; p.T = T; p.rast = (const float4 *)rast;
    p.px_per_batch = (int64_t)H * W; p.npx = p.px_per_batch * B;
    return 0;
}

int mcs_interpolate_fwd(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                        int32_t B, int32_t H, int32_t W, float *out, mcs_stream stream)
{
    InterpParams p{};
    if (int e = interp_common(p, attr, attr_batch_stride, V, C, tris, T, rast, B, H, W)) return e;
    MCS_REQUIRE(out != nullptr, "mcs_interpolate_fwd: null output");
    p.out = out;
    k_interpolate<0><<<(unsigned)((p.npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_interpolate_bwd(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                        int32_t B, int32_t H, int32_t W, const float *d_out, float *d_attr, mcs_stream stream)
{
    InterpParams p{};
    if (int e = interp_common(p, attr, attr_batch_stride, V, C, tris, T, rast, B, H, W)) return e;
    MCS_REQUIRE(d_out && d_attr, "mcs_interpolate_bwd: null gradient pointer");
    p.dout = d_out; p.dattr = d_attr;
    k_interpolate<1><<<(unsigned)((p.npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_interpolate_bwd_rast(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                             int32_t B, int32_t H, int32_t W, const float *d_out, float *d_attr, float *d_rast, mcs_stream stream)
{
    InterpParams p{};
    if (int e = interp_common(p, attr, attr_batch_stride, V, C, tris, T, rast, B, H, W)) return e;
    MCS_REQUIRE(d_out && d_rast, "mcs_interpolate_bwd_rast: null gradient pointer");
    p.dout = d_out; p.dattr = d_attr; p.drast = (float4 *)d_rast;
    k_interpolate<2><<<(unsigned)((p.npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

// outs: the entry point's own pointers are present
static int rast_bwd_common(RastBwdParams &p, const char *name, bool outs, const float *pos, int64_t pos_batch_stride, int32_t V,
                           const int32_t *tris, int32_t T, const float *rast, int32_t B, int32_t H, int32_t W)
{
    MCS_REQUIRE(pos && tris && rast && outs && V > 0 && T > 0 && B > 0 && H > 0 && W > 0 && pos_batch_stride >= 0, "%s: bad arguments", name);
    p.pos = pos; p.pos_bs = pos_batch_stride; p.V = V; p.tris = tris; p.T = T; p.rast = (const float4 *)rast;
    p.B = B; p.H = H; p.W = W;
    return 0;
}

int mcs_rasterize_bwd(const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const float *rast, int32_t B, int32_t H,
                      int32_t W, const float *d_rast, float *d_pos, mcs_stream stream)
{
    RastBwdParams p{};
    if (int e = rast_bwd_common(p, "mcs_rasterize_bwd", d_rast && d_pos, pos, pos_batch_stride, V, tris, T, rast, B, H, W)) return e;
    p.drast = (const float4 *)d_rast; p.dpos = d_pos;
    const int64_t n = (int64_t)B * H * W;
    k_rasterize_bwd<false><<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_rast_db(const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const float *rast, int32_t B, int32_t H,
                int32_t W, float *rast_db, mcs_stream stream)
{
    RastBwdParams p{};
    if (int e = rast_bwd_common(p, "mcs_rast_db", rast_db != nullptr, pos, pos_batch_stride, V, tris, T, rast, B, H, W)) return e;
    p.rast_db = (float4 *)rast_db;
    const int64_t n = (int64_t)B * H * W;
    k_rast_db<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_rasterize_bwd_db(const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const float *rast, int32_t B,
                         int32_t H, int32_t W, const float *d_rast, const float *d_rast_db, float *d_pos, mcs_stream stream)
{
    RastBwdParams p{};
    if (int e = rast_bwd_common(p, "mcs_rasterize_bwd_db", d_rast_db && d_pos, pos, pos_batch_stride, V, tris, T, rast, B, H, W)) return e;
    p.drast = (const float4 *)d_rast; p.drast_db = (const float4 *)d_rast_db; p.dpos = d_pos;
    const int64_t n = (int64_t)B * H * W;
    k_rasterize_bwd<true><<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

static int interp_da_common(InterpDaParams &p, const char *name, const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C,
                            const int32_t *tris, int32_t T, const float *rast, const float *rast_db, int32_t B, int32_t H, int32_t W,
                            int32_t n_diff, const int32_t *diff_idx)
{
    MCS_REQUIRE(attr && tris && rast && rast_db && V > 0 && C > 0 && T > 0 && B > 0 && H > 0 && W > 0 && attr_batch_stride >= 0,
                "%s: bad arguments", name);
    if (diff_idx == nullptr) {
        MCS_REQUIRE(n_diff == C, "%s: without an index list n_diff (%d) must equal C (%d)", name, n_diff, C);
    } else {
        MCS_REQUIRE(n_diff >= 1 && n_diff <= MCS_DIFF_ATTRS_MAX, "%s: %d attribute indices (1 to %d allowed)", name, n_diff, MCS_DIFF_ATTRS_MAX);
        for (int k = 0; k < n_diff; ++k) {
            MCS_REQUIRE(diff_idx[k] >= 0 && diff_idx[k] < C, "%s: attribute index %d out of range [0, %d)", name, diff_idx[k], C);
            p.idx[k] = diff_idx[k];
        }
    }
    p.attr = attr; p.attr_bs = attr_batch_stride; p.V = V; p.C = C; p.tris = tris; p.T = T;
    p.rast = (const float4 *)rast; p.db = (const float4 *)rast_db;
    p.px_per_batch = (int64_t)H * W; p.npx = p.px_per_batch * B;
    p.n = n_diff; p.all = diff_idx == nullptr;
    return 0;
}

int mcs_interpolate_da_fwd(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                           const float *rast_db, int32_t B, int32_t H, int32_t W, int32_t n_diff, const int32_t *diff_idx, float *out_da,
                           mcs_stream stream)
{
    InterpDaParams p{};
    if (int e = interp_da_common(p, "mcs_interpolate_da_fwd", attr, attr_batch_stride, V, C, tris, T, rast, rast_db, B, H, W, n_diff, diff_idx))
        return e;
    MCS_REQUIRE(out_da != nullptr, "mcs_interpolate_da_fwd: null output");
    p.out_da = out_da;
    k_interpolate_da<false><<<(unsigned)((p.npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_interpolate_da_bwd(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                           const float *rast_db, int32_t B, int32_t H, int32_t W, int32_t n_diff, const int32_t *diff_idx, const float *d_out_da,
                           float *d_attr, float *d_rast_db, mcs_stream stream)
{
    InterpDaParams p{};
    if (int e = interp_da_common(p, "mcs_interpolate_da_bwd", attr, attr_batch_stride, V, C, tris, T, rast, rast_db, B, H, W, n_diff, diff_idx))
        return e;
    MCS_REQUIRE(d_out_da && (d_attr || d_rast_db), "mcs_interpolate_da_bwd: null gradient pointer");
    p.dout_da = d_out_da; p.dattr = d_attr; p.ddb = (float4 *)d_rast_db;
    k_interpolate_da<true><<<(unsigned)((p.npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int64_t mcs_aa_topology_workspace_bytes(int32_t T)
{
    if (T <= 0) return 0;
    return (int64_t)aa_topo_capacity(T) * (sizeof(unsigned long long) + sizeof(int) + 2 * sizeof(int));
}

int mcs_aa_topology(const int32_t *tris, int32_t T, void *workspace, int32_t *adj, mcs_stream stream)
{
    MCS_REQUIRE(tris && workspace && adj && T > 0, "mcs_aa_topology: bad arguments");
    MCS_REQUIRE(((uintptr_t)workspace & 7) == 0, "mcs_aa_topology: workspace must be 8-byte aligned");
    const uint64_t cap = aa_topo_capacity(T);
    unsigned long long *keys = (unsigned long long *)workspace;
    int *cnt = (int *)(keys + cap), *first2 = cnt + cap;
    cudaStream_t s = (cudaStream_t)stream;
    MCS_CUDA(cudaMemsetAsync(keys, 0xFF, cap * sizeof(unsigned long long), s));
    MCS_CUDA(cudaMemsetAsync(cnt, 0, cap * sizeof(int), s));
    const int64_t n = 3 * (int64_t)T;
    k_aa_topo_insert<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(tris, T, keys, cnt, first2, cap - 1, adj);
    MCS_LAUNCH_CHECK();
    k_aa_topo_resolve<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(T, cnt, first2, adj);
    MCS_LAUNCH_CHECK();
    return 0;
}

static int aa_common(AAParams &p, const float *color, int32_t C, const float *rast, int32_t B, int32_t H, int32_t W, const float *pos,
                     int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const int32_t *adj)
{
    MCS_REQUIRE(color && rast && pos && tris && adj && C > 0 && B > 0 && H > 0 && W > 0 && V > 0 && T > 0 && pos_batch_stride >= 0,
                "mcs_antialias: bad arguments");
    p.color = color; p.C = C;
    p.g = AAGeom{(const float4 *)rast, B, H, W, pos, pos_batch_stride, V, tris, T, adj};
    p.npx = (int64_t)B * H * W;
    return 0;
}

int mcs_antialias_fwd(const float *color, int32_t C, const float *rast, int32_t B, int32_t H, int32_t W, const float *pos, int64_t pos_batch_stride,
                      int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, float *out, mcs_stream stream)
{
    AAParams p{};
    if (int e = aa_common(p, color, C, rast, B, H, W, pos, pos_batch_stride, V, tris, T, adj)) return e;
    MCS_REQUIRE(out != nullptr, "mcs_antialias_fwd: null output");
    p.out = out;
    k_antialias<false><<<(unsigned)((p.npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_antialias_bwd(const float *color, int32_t C, const float *rast, int32_t B, int32_t H, int32_t W, const float *pos, int64_t pos_batch_stride,
                      int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, const float *d_out, float *d_color, float *d_pos, mcs_stream stream)
{
    AAParams p{};
    if (int e = aa_common(p, color, C, rast, B, H, W, pos, pos_batch_stride, V, tris, T, adj)) return e;
    MCS_REQUIRE(d_out && (d_color || d_pos), "mcs_antialias_bwd: null gradient pointer");
    p.dout = d_out; p.dcolor = d_color; p.dpos = d_pos;
    k_antialias<true><<<(unsigned)((p.npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_texel_fetch_fwd(const float *tex, int64_t T, int32_t C, const int64_t *idx, int64_t n, float *out, mcs_stream stream)
{
    MCS_REQUIRE(tex && idx && out && T > 0 && C > 0 && n >= 0, "mcs_texel_fetch_fwd: bad arguments");
    if (n == 0) return 0;
    k_texel_fetch<false><<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(tex, idx, n, C, T, out, nullptr, nullptr);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_texel_fetch_bwd(int64_t T, int32_t C, const int64_t *idx, int64_t n, const float *d_out, float *d_tex, mcs_stream stream)
{
    MCS_REQUIRE(idx && d_out && d_tex && T > 0 && C > 0 && n >= 0, "mcs_texel_fetch_bwd: bad arguments");
    if (n == 0) return 0;
    k_texel_fetch<true><<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(nullptr, idx, n, C, T, nullptr, d_out, d_tex);
    MCS_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
