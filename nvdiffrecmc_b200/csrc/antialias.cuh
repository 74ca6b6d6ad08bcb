// antialias.cuh -- the silhouette-edge pair logic of analytic antialiasing (rules 1-6 of csrc/raster.cu's header), shared by
// raster.cu's k_antialias and composite.cu's layer compositing so that both make the same decisions from one copy of the rules.
// Pixel-centre helpers of the clip-space triangle (px_ndc, clip_a, clip_edge) live here too: the rasterize backward and rast_db use them.
#pragma once
#include "common.cuh"

namespace {

// image b, row iy and column ix of flat pixel index i of a [B,H,W] image
__device__ __forceinline__ void px_decode(int64_t i, int H, int W, int &b, int &iy, int &ix)
{
    ix = (int)(i % W); const int64_t t = i / W; iy = (int)(t % H); b = (int)(t / H);
}

// NDC coordinate of pixel centre i of n (image row iy -> NDC y = (iy + 0.5) / H * 2 - 1, as k_rasterize), explicitly rounded
__device__ __forceinline__ float px_ndc(int i, int n) { return __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn((float)i, 0.5f), (float)n), 2.0f), 1.0f); }

// a = (x - px w, y - py w) of clip-space vertex (x, y, w) seen from NDC point (px, py), explicitly rounded
__device__ __forceinline__ float2 clip_a(float x, float y, float w, float px, float py)
{
    return make_float2(__fsub_rn(x, __fmul_rn(px, w)), __fsub_rn(y, __fmul_rn(py, w)));
}

// edge function a_A x a_B, explicitly rounded
__device__ __forceinline__ float clip_edge(float2 a, float2 b) { return __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)); }

// The geometry one antialias pass reads: rast [B,H,W,4], clip-space pos [V,4] (pos_bs 0) or [B,V,4] (pos_bs V*4), tris [T,3] and their
// edge adjacency adj [T,3] (k_aa_topo_*).
struct AAGeom {
    const float4 *rast; int B, H, W;
    const float *pos; int64_t pos_bs; int V;
    const int32_t *tris; int T;
    const int32_t *adj;
};

struct AAEdge {
    float t, ef, eo;
    int va, vb;
    float3 A, B;          // (x, y, w) of the edge's endpoints
};

__device__ __forceinline__ float3 aa_vert(const float *P, int v)
{
    const float *q = P + 4 * (size_t)v;
    return make_float3(__ldg(q), __ldg(q + 1), __ldg(q + 3));
}

// homogeneous edge function a_A x a_B at NDC point (px, py)
__device__ __forceinline__ float aa_edge(float3 A, float3 B, float px, float py)
{
    return clip_edge(clip_a(A.x, A.y, A.z, px, py), clip_a(B.x, B.y, B.z, px, py));
}

// facing: det[[x0,y0,w0],[x1,y1,w1],[x2,y2,w2]] > 0
__device__ __forceinline__ bool aa_facing(float3 a, float3 b, float3 c)
{
    const float m0 = __fsub_rn(__fmul_rn(b.y, c.z), __fmul_rn(b.z, c.y));
    const float m1 = __fsub_rn(__fmul_rn(b.x, c.z), __fmul_rn(b.z, c.x));
    const float m2 = __fsub_rn(__fmul_rn(b.x, c.y), __fmul_rn(b.y, c.x));
    return __fadd_rn(__fsub_rn(__fmul_rn(a.x, m0), __fmul_rn(a.y, m1)), __fmul_rn(a.z, m2)) > 0.0f;
}

// Closest crossing silhouette edge of front triangle F between pixel centres f and o (rules 3-5).
__device__ bool aa_search(const AAGeom &p, const float *P, int F, bool horiz, float fx, float fy, float ox, float oy, AAEdge &e)
{
    int vi[3];
    float3 q[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { vi[k] = __ldg(p.tris + 3 * (size_t)F + k); q[k] = aa_vert(P, vi[k]); }
    int facing = -1;
    bool found = false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int k1 = k == 2 ? 0 : k + 1;
        const float3 A = q[k], B = q[k1];
        if (!(A.z > 0.0f && B.z > 0.0f)) continue;
        const int nb = __ldg(p.adj + 3 * (size_t)F + k);
        if (nb >= 0 && nb < p.T) {
            if (facing < 0) facing = aa_facing(q[0], q[1], q[2]) ? 1 : 0;
            const int n0 = __ldg(p.tris + 3 * (size_t)nb), n1 = __ldg(p.tris + 3 * (size_t)nb + 1), n2 = __ldg(p.tris + 3 * (size_t)nb + 2);
            if ((aa_facing(aa_vert(P, n0), aa_vert(P, n1), aa_vert(P, n2)) ? 1 : 0) == facing) continue;
        }
        const float dX = __fmul_rn(__fsub_rn(__fdiv_rn(B.x, B.z), __fdiv_rn(A.x, A.z)), (float)p.W);
        const float dY = __fmul_rn(__fsub_rn(__fdiv_rn(B.y, B.z), __fdiv_rn(A.y, A.z)), (float)p.H);
        if ((fabsf(dY) >= fabsf(dX)) != horiz) continue;
        const float ef = aa_edge(A, B, fx, fy), eo = aa_edge(A, B, ox, oy);
        if (!((ef > 0.0f && eo < 0.0f) || (ef < 0.0f && eo > 0.0f))) continue;
        const float t = __fdiv_rn(ef, __fsub_rn(ef, eo));
        if (!found || t < e.t) { found = true; e.t = t; e.ef = ef; e.eo = eo; e.va = vi[k]; e.vb = vi[k1]; e.A = A; e.B = B; }
    }
    return found;
}

__device__ __forceinline__ int aa_tid(float4 r, int T)
{
    const int id = (int)r.w - 1;
    return id < T ? id : -1;
}

// Pair (this pixel p, neighbour q): true when the pair has a crossing edge with a nonzero blend weight w; gain_self tells whether p
// (else q) gains w * (c_other - c_self); p_front whether p is the front pixel.
__device__ __forceinline__ bool aa_pair(const AAGeom &p, const float *P, float px, float py, int tp, float zp, float qx, float qy, int tq, float zq,
                                        bool horiz, float &w, bool &gain_self, bool &p_front, AAEdge &e)
{
    if (tp == tq) return false;
    bool pf;
    if (tq < 0) pf = true;
    else if (tp < 0) pf = false;
    else if (zp < zq) pf = true;
    else if (zq < zp) pf = false;
    else pf = tp < tq;
    const bool found = pf ? aa_search(p, P, tp, horiz, px, py, qx, qy, e) : aa_search(p, P, tq, horiz, qx, qy, px, py, e);
    if (!found) return false;
    bool gain_front;
    if (e.t < 0.5f) { w = __fsub_rn(0.5f, e.t); gain_front = true; }
    else if (e.t > 0.5f) { w = __fsub_rn(e.t, 0.5f); gain_front = false; }
    else return false;
    gain_self = gain_front == pf;
    p_front = pf;
    return true;
}

__device__ __forceinline__ void aa_edge_grad(const AAEdge &e, float px, float py, float s, float (&gA)[3], float (&gB)[3])
{
    const float ax = e.A.x - px * e.A.z, ay = e.A.y - py * e.A.z, bx = e.B.x - px * e.B.z, by = e.B.y - py * e.B.z;
    gA[0] += s * by; gA[1] -= s * bx; gA[2] += s * (py * bx - px * by);
    gB[0] -= s * ay; gB[1] += s * ax; gB[2] += s * (px * ay - py * ax);
}

// The blend pairs of one pixel, indexed by direction d in the fixed order left, right, up, down (rule 6): on[d] = a pair with a
// nonzero weight w[d]; self[d] = this pixel gains (else the neighbour j[d] does).
struct AAPairs {
    float w[4];
    int64_t j[4];
    bool on[4], self[4];
};

// neighbour in direction d of pixel (ix, iy)
__device__ __forceinline__ int aa_nbx(int d, int ix) { return d == 0 ? ix - 1 : (d == 1 ? ix + 1 : ix); }
__device__ __forceinline__ int aa_nby(int d, int iy) { return d == 2 ? iy - 1 : (d == 3 ? iy + 1 : iy); }

// The pairs of pixel i = (b, iy, ix) with rast r.  With DPOS and dpos != null, every pair this pixel owns (right, down) takes
// dldt(gain_self, d, j) = sum over its channels of g_gain (c_other - c_gain), g the gradient of the antialiased output, and scatters
// dL/dt dt/d(x, y, w) of the crossing edge's endpoints into dpos (caller-zeroed, float atomics): dt/de_f = -e_o / D^2,
// dt/de_o = e_f / D^2, D = e_f - e_o; o gains (t - 1/2)(c_f - c_o), f gains (1/2 - t)(c_o - c_f).
template <bool DPOS, class DLdt>
__device__ __forceinline__ AAPairs aa_pixel_pairs(const AAGeom &g, int64_t i, int b, int iy, int ix, float4 r, float *dpos, DLdt dldt)
{
    AAPairs pr;
    const int tp = aa_tid(r, g.T);
    const float px = px_ndc(ix, g.W), py = px_ndc(iy, g.H);
    const float *P = g.pos + (int64_t)b * g.pos_bs;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
        pr.on[d] = false;
        pr.self[d] = false;
        pr.w[d] = 0.0f;
        const int nx = aa_nbx(d, ix), ny = aa_nby(d, iy);
        pr.j[d] = i + (nx - ix) + (int64_t)(ny - iy) * g.W;
        if (nx < 0 || nx >= g.W || ny < 0 || ny >= g.H) continue;
        const int64_t j = pr.j[d];
        const float4 rq = __ldg(g.rast + j);
        const int tq = aa_tid(rq, g.T);
        if (tq == tp) continue;
        const float qx = px_ndc(nx, g.W), qy = px_ndc(ny, g.H);
        float w; bool gain_self, p_front; AAEdge e;
        if (!aa_pair(g, P, px, py, tp, r.z, qx, qy, tq, rq.z, d < 2, w, gain_self, p_front, e)) continue;
        pr.on[d] = true; pr.w[d] = w; pr.self[d] = gain_self;
        if (DPOS && dpos && (d == 1 || d == 3)) {
            float dLdt = dldt(gain_self, d, j);
            const bool gain_front = gain_self == p_front;
            if (gain_front) dLdt = -dLdt;
            if (dLdt != 0.0f) {
                const float D = e.ef - e.eo, iD2 = 1.0f / (D * D);
                const float sf = dLdt * (-e.eo * iD2), so = dLdt * (e.ef * iD2);
                float gA[3] = {0.0f, 0.0f, 0.0f}, gB[3] = {0.0f, 0.0f, 0.0f};
                aa_edge_grad(e, p_front ? px : qx, p_front ? py : qy, sf, gA, gB);
                aa_edge_grad(e, p_front ? qx : px, p_front ? qy : py, so, gA, gB);
                float *DA = dpos + (int64_t)b * g.pos_bs + 4 * (size_t)e.va, *DB = dpos + (int64_t)b * g.pos_bs + 4 * (size_t)e.vb;
                atomicAdd(DA, gA[0]); atomicAdd(DA + 1, gA[1]); atomicAdd(DA + 3, gA[2]);
                atomicAdd(DB, gB[0]); atomicAdd(DB + 1, gB[1]); atomicAdd(DB + 3, gB[2]);
            }
        }
    }
    return pr;
}

}  // namespace
