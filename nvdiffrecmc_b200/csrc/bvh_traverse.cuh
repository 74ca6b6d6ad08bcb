// bvh_traverse.cuh -- device-side ray traversal of the libmcshade acceleration structure.
//
// Replaces optixTrace() (render/optixutils/c_src/envsampling/kernel.cu:101-118): the H100 has no RT
// cores, so visibility is a hand-written stack traversal of a binary BVH whose 64-byte nodes hold
// BOTH children's boxes (one node visit = four 128-bit loads through the read-only path, then two
// slab tests); a leaf is a run of up to MCS_LEAF_MAX consecutive triangles in Morton order (an LBVH
// subtree collapsed at build time), each stored as three float4 (v0, e1, e2).  Child codes: >= 0 internal
// node index, < 0 leaf with ~code = (first_triangle << 3) | (count - 1).
//
// Parity contract (DESIGN.md "visibility"): the boolean result equals the oracle's brute-force loop
// bit for bit because (a) the triangle predicate mt_hit() is evaluated with the exact operation
// order of oracle/mcoracle.c:mt_hit (explicit FMAs, IEEE reciprocal), and (b) box culling is
// conservative: leaf boxes are padded by 1e-5 x scene extent and the slab comparison is relaxed by
// 4 ulp, so the set of triangles tested may differ from brute force but never drops a hit.
#pragma once
#include "common.cuh"

struct BvhView {
    const float4 *nodes;
    const float4 *tris;
    const float *qgrid;      // origin xyz, cell xyz, 1 / cell xyz of the quantisation grid
    const uint4 *nodesq4;    // 64-byte 4-wide quantised nodes (bvh.cu:k_emit_nodesq, wide part); may be null
};

// Moeller-Trumbore with a fixed evaluation order (mirrors oracle mt_hit()).  Returns true on a hit
// with t in (tmin, tmax), tmin >= 0; u, v, t are written on a hit.
__device__ __forceinline__ bool mt_hit(f3 o, f3 d, f3 v0, f3 e1, f3 e2, float tmax, float &t_out, float &u_out, float &v_out, float tmin = 0.0f)
{
    float px = __fmaf_rn(d.y, e2.z, -__fmul_rn(d.z, e2.y));
    float py = __fmaf_rn(d.z, e2.x, -__fmul_rn(d.x, e2.z));
    float pz = __fmaf_rn(d.x, e2.y, -__fmul_rn(d.y, e2.x));
    float det = __fmaf_rn(e1.x, px, __fmaf_rn(e1.y, py, __fmul_rn(e1.z, pz)));
    if (det == 0.0f) return false;
    float inv = __frcp_rn(det);
    float tx = __fsub_rn(o.x, v0.x), ty = __fsub_rn(o.y, v0.y), tz = __fsub_rn(o.z, v0.z);
    float u = __fmul_rn(__fmaf_rn(tx, px, __fmaf_rn(ty, py, __fmul_rn(tz, pz))), inv);
    if (u < 0.0f || u > 1.0f) return false;
    float qx = __fmaf_rn(ty, e1.z, -__fmul_rn(tz, e1.y));
    float qy = __fmaf_rn(tz, e1.x, -__fmul_rn(tx, e1.z));
    float qz = __fmaf_rn(tx, e1.y, -__fmul_rn(ty, e1.x));
    float v = __fmul_rn(__fmaf_rn(d.x, qx, __fmaf_rn(d.y, qy, __fmul_rn(d.z, qz))), inv);
    if (v < 0.0f || __fadd_rn(u, v) > 1.0f) return false;
    float t = __fmul_rn(__fmaf_rn(e2.x, qx, __fmaf_rn(e2.y, qy, __fmul_rn(e2.z, qz))), inv);
    if (!(t > tmin && t < tmax)) return false;
    t_out = t; u_out = u; v_out = v;
    return true;
}

struct RayPre {
    float ix, iy, iz;      // 1/d (zero components nudged to +-1e-30 so 0*inf cannot produce NaN)
    float ox, oy, oz;      // o * (1/d)
};
__device__ __forceinline__ RayPre ray_pre(f3 o, f3 d)
{
    RayPre r;
    float dx = fabsf(d.x) < 1e-30f ? copysignf(1e-30f, d.x) : d.x;
    float dy = fabsf(d.y) < 1e-30f ? copysignf(1e-30f, d.y) : d.y;
    float dz = fabsf(d.z) < 1e-30f ? copysignf(1e-30f, d.z) : d.z;
    r.ix = 1.0f / dx; r.iy = 1.0f / dy; r.iz = 1.0f / dz;
    r.ox = o.x * r.ix; r.oy = o.y * r.iy; r.oz = o.z * r.iz;
    return r;
}

// Depth-peeling separation: the next layer along a ray is the closest hit with t > peel_sep(t_prev), one exactly rounded fp32
// multiply by 1 + 2^-16 (exact in fp32, about 128 ulp of t).  A plain t > t_prev would return the same surface again where a ray
// crosses a shared edge: Moeller-Trumbore's closed bounds accept it on both triangles at t values a few ulp apart.  Surfaces closer
// than this along the ray merge into one layer, as nvdiffrast's peeler drops fragments at equal depth.  tests/peel_oracle.c restates it.
__device__ __forceinline__ float peel_sep(float t) { return __fmul_rn(t, 1.0000152587890625f); }

#define MCS_STACK 64
#define MCS_LEAF_MAX 4
#define MCS_TMAX 1e16f

// Any-hit query: true if some triangle is hit with t in (0, 1e16).
__device__ __forceinline__ bool bvh_occluded(const BvhView &b, f3 o, f3 d)
{
    const RayPre r = ray_pre(o, d);
    int stack[MCS_STACK];
    int sp = 0;
    int node = 0;
    while (true) {
        if (node >= 0) {
            const float4 *n = b.nodes + 4 * (size_t)node;
            const float4 q0 = __ldg(n), q1 = __ldg(n + 1), q2 = __ldg(n + 2), q3 = __ldg(n + 3);
            float a0 = fmaf(q0.x, r.ix, -r.ox), a1 = fmaf(q0.y, r.ix, -r.ox);
            float b0 = fmaf(q0.z, r.iy, -r.oy), b1 = fmaf(q0.w, r.iy, -r.oy);
            float c0 = fmaf(q2.x, r.iz, -r.oz), c1 = fmaf(q2.y, r.iz, -r.oz);
            float tn0 = fmaxf(fmaxf(fminf(a0, a1), fminf(b0, b1)), fmaxf(fminf(c0, c1), 0.0f));
            float tf0 = fminf(fminf(fmaxf(a0, a1), fmaxf(b0, b1)), fminf(fmaxf(c0, c1), MCS_TMAX));
            a0 = fmaf(q1.x, r.ix, -r.ox); a1 = fmaf(q1.y, r.ix, -r.ox);
            b0 = fmaf(q1.z, r.iy, -r.oy); b1 = fmaf(q1.w, r.iy, -r.oy);
            c0 = fmaf(q2.z, r.iz, -r.oz); c1 = fmaf(q2.w, r.iz, -r.oz);
            float tn1 = fmaxf(fmaxf(fminf(a0, a1), fminf(b0, b1)), fmaxf(fminf(c0, c1), 0.0f));
            float tf1 = fminf(fminf(fmaxf(a0, a1), fmaxf(b0, b1)), fminf(fmaxf(c0, c1), MCS_TMAX));
            const bool h0 = tn0 <= tf0 * 1.0000004f, h1 = tn1 <= tf1 * 1.0000004f;
            const int ch0 = __float_as_int(q3.x), ch1 = __float_as_int(q3.y);
            if (h0 && h1) {
                const bool first0 = tn0 <= tn1;         // nearer child first: occluders close to the origin end the ray early
                stack[sp++] = first0 ? ch1 : ch0;
                node = first0 ? ch0 : ch1;
                continue;
            }
            if (h0) { node = ch0; continue; }
            if (h1) { node = ch1; continue; }
        } else {
            const int code = ~node;
            const int start = code >> 3, cnt = (code & 7) + 1;
            for (int k = 0; k < cnt; ++k) {
                const float4 *t = b.tris + 3 * (size_t)(start + k);
                const float4 t0 = __ldg(t), t1 = __ldg(t + 1), t2 = __ldg(t + 2);
                float tt, uu, vv;
                if (mt_hit(o, d, F3(t0.x, t0.y, t0.z), F3(t1.x, t1.y, t1.z), F3(t2.x, t2.y, t2.z), MCS_TMAX, tt, uu, vv)) return true;
            }
        }
        if (sp == 0) return false;
        node = stack[--sp];
    }
}

// Closest-hit query (primary rays of the synthetic G-buffer producer).  Ties in t are resolved
// towards the smaller original triangle id, matching the oracle's brute-force scan.  Only hits with
// t > t_lo count (t_lo = 0: every hit mt_hit accepts; depth peeling passes the previous layer's
// separated t).  t_lo enters as the lower clamp of each box's entry distance, so a box is skipped
// for it only when its relaxed exit distance lies strictly before t_lo: the culling stays as
// conservative as the t_best bound, and with t_lo = 0 the code is the plain closest-hit walk.
__device__ __forceinline__ int bvh_closest(const BvhView &b, f3 o, f3 d, float t_lo, float &t_best, float &u_best, float &v_best)
{
    const RayPre r = ray_pre(o, d);
    int stack[MCS_STACK];
    int sp = 0;
    int node = 0;
    int best = -1;
    t_best = MCS_TMAX; u_best = 0.0f; v_best = 0.0f;
    while (true) {
        if (node >= 0) {
            const float4 *n = b.nodes + 4 * (size_t)node;
            const float4 q0 = __ldg(n), q1 = __ldg(n + 1), q2 = __ldg(n + 2), q3 = __ldg(n + 3);
            float a0 = fmaf(q0.x, r.ix, -r.ox), a1 = fmaf(q0.y, r.ix, -r.ox);
            float b0 = fmaf(q0.z, r.iy, -r.oy), b1 = fmaf(q0.w, r.iy, -r.oy);
            float c0 = fmaf(q2.x, r.iz, -r.oz), c1 = fmaf(q2.y, r.iz, -r.oz);
            float tn0 = fmaxf(fmaxf(fminf(a0, a1), fminf(b0, b1)), fmaxf(fminf(c0, c1), t_lo));
            float tf0 = fminf(fminf(fmaxf(a0, a1), fmaxf(b0, b1)), fminf(fmaxf(c0, c1), t_best));
            a0 = fmaf(q1.x, r.ix, -r.ox); a1 = fmaf(q1.y, r.ix, -r.ox);
            b0 = fmaf(q1.z, r.iy, -r.oy); b1 = fmaf(q1.w, r.iy, -r.oy);
            c0 = fmaf(q2.z, r.iz, -r.oz); c1 = fmaf(q2.w, r.iz, -r.oz);
            float tn1 = fmaxf(fmaxf(fminf(a0, a1), fminf(b0, b1)), fmaxf(fminf(c0, c1), t_lo));
            float tf1 = fminf(fminf(fmaxf(a0, a1), fmaxf(b0, b1)), fminf(fmaxf(c0, c1), t_best));
            const bool h0 = tn0 <= tf0 * 1.0000004f + 1e-30f, h1 = tn1 <= tf1 * 1.0000004f + 1e-30f;
            const int ch0 = __float_as_int(q3.x), ch1 = __float_as_int(q3.y);
            if (h0 && h1) {
                const bool first0 = tn0 <= tn1;
                stack[sp++] = first0 ? ch1 : ch0;
                node = first0 ? ch0 : ch1;
                continue;
            }
            if (h0) { node = ch0; continue; }
            if (h1) { node = ch1; continue; }
        } else {
            const int code = ~node;
            const int start = code >> 3, cnt = (code & 7) + 1;
            for (int k = 0; k < cnt; ++k) {
                const float4 *t = b.tris + 3 * (size_t)(start + k);
                const float4 t0 = __ldg(t), t1 = __ldg(t + 1), t2 = __ldg(t + 2);
                float tt, uu, vv;
                // exact ties in t are resolved by the original triangle id (brute-force order)
                if (mt_hit(o, d, F3(t0.x, t0.y, t0.z), F3(t1.x, t1.y, t1.z), F3(t2.x, t2.y, t2.z), MCS_TMAX, tt, uu, vv, t_lo)) {
                    const int id = __float_as_int(t0.w);
                    if (tt < t_best || (tt == t_best && id < best)) { t_best = tt; u_best = uu; v_best = vv; best = id; }
                }
            }
        }
        if (sp == 0) return best;
        node = stack[--sp];
    }
}
