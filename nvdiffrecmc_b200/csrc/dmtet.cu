// dmtet.cu -- DMTet's per-iteration geometry on sm_90a: marching tetrahedra (geometry/dmtet.py:91-141 of the reference) and the
// SDF regulariser sdf_reg_loss (dmtet.py:147-153), forward and backward, with no sort and no host synchronisation.
//
// Static per-grid tables (built once per tet grid by the caller, nvdiffrecmc_b200/dmtet.py; layout in include/mcshade.h):
//   edges [E,2] int32      the grid's unique edges (a < b), sorted lexicographically -- the reference's DMTetGeometry.all_edges;
//   tet_edges [T,6] int32  index into `edges` of each tet's base edges (0,1) (0,2) (0,3) (1,2) (1,3) (2,3);
//   v2e offsets [V+1] / v2e edges [2E] int32: for each grid vertex, its incident edges in ascending edge index (a CSR).
//
// Contract (what the reference computes, restated without its torch.unique):
//   occ(v) = sdf[v] > 0 (NaN is unoccupied).  Edge e = (a, b) crosses iff occ(a) != occ(b).  The reference's vertex list is exactly the
//   crossing edges in edge order: vertex id = exclusive scan of the crossing flags.  Vertex position, rounded in this order:
//       D = sa + (-sb);  w0 = (-sb) / D;  w1 = sa / D;  v = pa * w0 + pb * w1           (each operation IEEE fp32, no contraction)
//   Tet t has occupancy code c = occ(t0) + 2 occ(t1) + 4 occ(t2) + 8 occ(t3) and NT[c] triangles.  Faces: every 1-triangle tet in tet
//   order, then every 2-triangle tet in tet order with its two faces adjacent; face k of tet t is (vid of tet_edges[t][TT[c][3k+j]]),
//   j = 0..2, and its uv_idx is (4t, 4t+k+1, 4t+k+2).
//
// Count phase (one launch): per edge the crossing flag, per tet the pair (1 if NT = 1, 1 if NT = 2), both scanned exclusively by a
//   single-pass decoupled look-back (Merrill & Garland 2016) over tiles of MCS_DMTET_TILE items taken in ticket order, so a tile's
//   predecessors are resident or done.  Writes vid [E] (-1 where the edge does not cross), the tet prefix pair [T,2] and counts[3] =
//   (vertices, 1-triangle tets, 2-triangle tets), on the device; the caller reads the counts back once and sizes the outputs.
// Emit phase: verts from the crossing edges, faces and uv_idx from the tets.
// Backward: one thread per grid vertex walks its incident edges in ascending edge index and adds each crossing edge's contribution,
//   in the order of the reference's autograd graph:
//       dw0 = <g, pa>, dw1 = <g, pb>   (x, then y, then z);   dD = (-dw0) * (w0 / D) + (-dw1) * (w1 / D)
//       d pa += g * w0,  d sa += dw1 / D + dD;      d pb += g * w1,  d sb += -(dw0 / D + dD)
//   A vertex on no crossing edge gets exactly 0.  Dense outputs, no atomics, bit-reproducible.
// sdf_reg_loss: per edge mask = sign(s0) != sign(s1) with torch.sign's values (1, -1, and 0 for +-0 and for NaN); terms
//   bce(s0, s1 > 0) and bce(s1, s0 > 0), with bce(x, y) = log1p(exp(-|x|)) + max(x, 0) - x y in double; per-CTA partials (sum0, sum1, count) over fixed chunks, finished in double
//   by one CTA: loss = sum0 / M + sum1 / M (NaN when M = 0).  Backward: per vertex over the CSR of the same edges, in ascending edge
//   order, d sdf += ((sigmoid(x) - y) * d loss) / M for each masked edge the vertex is an end of; 0 when M = 0.  Neither pass syncs.
#include "common.cuh"

namespace {

constexpr int DT_THREADS = 256;
constexpr int DT_ITEMS = MCS_DMTET_TILE / DT_THREADS;
static_assert(DT_ITEMS * DT_THREADS == MCS_DMTET_TILE, "tile = threads x items");
constexpr unsigned long long FLAG_AGG = 1ull << 62, FLAG_PREFIX = 1ull << 63, VALUE_MASK = FLAG_AGG - 1ull;
constexpr int PAIR_SHIFT = 31;                // tet value: (#1-triangle) in bits 0..30, (#2-triangle) in bits 31..61
constexpr unsigned long long LOW_MASK = (1ull << PAIR_SHIFT) - 1ull;
constexpr int REG_CHUNK = 4096;               // sdf_reg_loss: edges per partial

__constant__ int8_t c_tri[16][6] = {
    {-1, -1, -1, -1, -1, -1}, {1, 0, 2, -1, -1, -1}, {4, 0, 3, -1, -1, -1}, {1, 4, 2, 1, 3, 4},
    {3, 1, 5, -1, -1, -1},    {2, 3, 0, 2, 5, 3},    {1, 4, 0, 1, 5, 4},    {4, 2, 5, -1, -1, -1},
    {4, 5, 2, -1, -1, -1},    {4, 1, 0, 4, 5, 1},    {3, 2, 0, 3, 5, 2},    {1, 3, 5, -1, -1, -1},
    {4, 1, 2, 4, 3, 1},       {3, 0, 4, -1, -1, -1}, {2, 0, 1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1}};
__constant__ int8_t c_ntri[16] = {0, 1, 1, 2, 1, 2, 2, 1, 1, 2, 2, 1, 2, 1, 1, 0};

struct Grid {
    const float *sdf; int64_t ss;               // sdf and its element stride
    const float *pos; int64_t ps0, ps1;         // pos [V,3] and its element strides
    const int2 *edges; int E;
    const int4 *tets; const int32_t *tet_edges; int T;
    int nEt, nTt;                               // tiles of edges, of tets
};

__device__ __forceinline__ bool occ(const Grid &g, int v) { return __ldg(g.sdf + (int64_t)v * g.ss) > 0.0f; }
__device__ __forceinline__ int tet_code(const Grid &g, int t)
{
    const int4 q = __ldg(g.tets + t);
    return (int)occ(g, q.x) | ((int)occ(g, q.y) << 1) | ((int)occ(g, q.z) << 2) | ((int)occ(g, q.w) << 3);
}
__device__ __forceinline__ f3 ld_pos(const Grid &g, int v)
{
    const float *p = g.pos + (int64_t)v * g.ps0;
    return F3(__ldg(p), __ldg(p + g.ps1), __ldg(p + 2 * g.ps1));
}

struct Weights { float D, w0, w1; };
__device__ __forceinline__ Weights edge_weights(float sa, float sb)
{
    Weights w;
    w.D = __fadd_rn(sa, -sb);
    w.w0 = __fdiv_rn(-sb, w.D);
    w.w1 = __fdiv_rn(sa, w.D);
    return w;
}

__device__ __forceinline__ unsigned long long shfl_up_u64(unsigned long long v, int d)
{
    return __shfl_up_sync(0xFFFFFFFFu, v, d);
}

// ---- count phase: crossing flags and tet pairs, both scanned in one launch ----
__global__ void __launch_bounds__(DT_THREADS) k_dmt_count(const Grid g, int32_t *__restrict__ vid, int2 *__restrict__ tpre, int32_t *__restrict__ counts,
                                                          unsigned long long *ws)
{
    __shared__ unsigned int s_tile;
    __shared__ unsigned long long s_warp[DT_THREADS / 32];
    __shared__ unsigned long long s_prefix;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_tile = atomicAdd((unsigned int *)ws, 1u);
    __syncthreads();
    const int ticket = (int)s_tile;
    const bool is_tet = ticket >= g.nEt;
    const int tile = is_tet ? ticket - g.nEt : ticket;
    const int n = is_tet ? g.T : g.E;
    const int ntiles = is_tet ? g.nTt : g.nEt;
    volatile unsigned long long *flags = ws + 1 + (is_tet ? g.nEt : 0);
    const int base = tile * MCS_DMTET_TILE + tid * DT_ITEMS;

    unsigned long long val[DT_ITEMS], local = 0;
#pragma unroll
    for (int k = 0; k < DT_ITEMS; ++k) {
        const int i = base + k;
        unsigned long long v = 0;
        if (i < n) {
            if (is_tet) {
                const int nt = c_ntri[tet_code(g, i)];
                v = nt == 1 ? 1ull : (nt == 2 ? (1ull << PAIR_SHIFT) : 0ull);
            } else {
                const int2 e = __ldg(g.edges + i);
                v = occ(g, e.x) != occ(g, e.y) ? 1ull : 0ull;
            }
        }
        val[k] = v;
        local += v;
    }
    // CTA exclusive scan of the per-thread sums (warp shuffles, then the warp totals in warp order)
    unsigned long long inc = local;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long o = shfl_up_u64(inc, d);
        if (lane >= d) inc += o;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    unsigned long long woff = 0, total = 0;
#pragma unroll
    for (int w = 0; w < DT_THREADS / 32; ++w) {
        const unsigned long long t = s_warp[w];
        if (w < warp) woff += t;
        total += t;
    }
    // decoupled look-back over the tiles of this domain
    if (tid == 0) {
        unsigned long long run = 0;
        if (tile == 0) {
            flags[0] = total | FLAG_PREFIX;
        } else {
            flags[tile] = total | FLAG_AGG;
            for (int j = tile - 1; j >= 0; --j) {
                unsigned long long f;
                do { f = flags[j]; } while (f == 0ull);
                run += f & VALUE_MASK;
                if (f & FLAG_PREFIX) break;
            }
            __threadfence();
            flags[tile] = (run + total) | FLAG_PREFIX;
        }
        s_prefix = run;
        if (tile == ntiles - 1) {
            const unsigned long long all = run + total;
            if (is_tet) { counts[1] = (int32_t)(all & LOW_MASK); counts[2] = (int32_t)(all >> PAIR_SHIFT); }
            else counts[0] = (int32_t)all;
        }
    }
    __syncthreads();
    unsigned long long ex = s_prefix + woff + inc - local;
#pragma unroll
    for (int k = 0; k < DT_ITEMS; ++k) {
        const int i = base + k;
        if (i < n) {
            if (is_tet) tpre[i] = make_int2((int)(ex & LOW_MASK), (int)(ex >> PAIR_SHIFT));
            else vid[i] = val[k] ? (int32_t)ex : -1;
        }
        ex += val[k];
    }
}

// ---- emit phase: vertices per crossing edge, then faces and uv_idx per tet (one launch, edge blocks first) ----
__global__ void __launch_bounds__(256) k_dmt_emit(const Grid g, const int32_t *__restrict__ vid, const int2 *__restrict__ tpre,
                                                  const int32_t *__restrict__ counts, float *__restrict__ verts, int64_t *__restrict__ faces,
                                                  int64_t *__restrict__ uv_idx, int edge_blocks)
{
    if ((int)blockIdx.x < edge_blocks) {
        const int e = blockIdx.x * blockDim.x + threadIdx.x;
        if (e >= g.E) return;
        const int id = __ldg(vid + e);
        if (id < 0) return;
        const int2 ab = __ldg(g.edges + e);
        const Weights w = edge_weights(__ldg(g.sdf + (int64_t)ab.x * g.ss), __ldg(g.sdf + (int64_t)ab.y * g.ss));
        const f3 pa = ld_pos(g, ab.x), pb = ld_pos(g, ab.y);
        float *o = verts + 3 * (int64_t)id;
        o[0] = __fadd_rn(__fmul_rn(pa.x, w.w0), __fmul_rn(pb.x, w.w1));
        o[1] = __fadd_rn(__fmul_rn(pa.y, w.w0), __fmul_rn(pb.y, w.w1));
        o[2] = __fadd_rn(__fmul_rn(pa.z, w.w0), __fmul_rn(pb.z, w.w1));
        return;
    }
    const int t = (blockIdx.x - edge_blocks) * blockDim.x + threadIdx.x;
    if (t >= g.T) return;
    const int c = tet_code(g, t);
    const int nt = c_ntri[c];
    if (nt == 0) return;
    const int2 pre = __ldg(tpre + t);
    const int64_t f0 = nt == 1 ? (int64_t)pre.x : (int64_t)__ldg(counts + 1) + 2 * (int64_t)pre.y;
    const int32_t *te = g.tet_edges + 6 * (int64_t)t;
    for (int k = 0; k < nt; ++k) {
        int64_t *fo = faces + 3 * (f0 + k), *uo = uv_idx + 3 * (f0 + k);
#pragma unroll
        for (int j = 0; j < 3; ++j) fo[j] = (int64_t)__ldg(vid + __ldg(te + c_tri[c][3 * k + j]));
        uo[0] = 4 * (int64_t)t; uo[1] = 4 * (int64_t)t + k + 1; uo[2] = 4 * (int64_t)t + k + 2;
    }
}

// ---- backward: per grid vertex, gather over its incident edges in ascending edge index ----
__global__ void __launch_bounds__(256) k_dmt_bwd(const Grid g, int V, const int32_t *__restrict__ vid, const int32_t *__restrict__ off,
                                                 const int32_t *__restrict__ adj, const float *__restrict__ d_verts, float *__restrict__ d_pos,
                                                 float *__restrict__ d_sdf)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    float gx = 0.0f, gy = 0.0f, gz = 0.0f, gs = 0.0f;
    const int j1 = __ldg(off + v + 1);
    for (int j = __ldg(off + v); j < j1; ++j) {
        const int e = __ldg(adj + j);
        const int id = __ldg(vid + e);
        if (id < 0) continue;
        const int2 ab = __ldg(g.edges + e);
        const Weights w = edge_weights(__ldg(g.sdf + (int64_t)ab.x * g.ss), __ldg(g.sdf + (int64_t)ab.y * g.ss));
        const f3 pa = ld_pos(g, ab.x), pb = ld_pos(g, ab.y);
        const float *gp = d_verts + 3 * (int64_t)id;
        const float g0 = __ldg(gp), g1 = __ldg(gp + 1), g2 = __ldg(gp + 2);
        const float dw0 = __fadd_rn(__fadd_rn(__fmul_rn(g0, pa.x), __fmul_rn(g1, pa.y)), __fmul_rn(g2, pa.z));
        const float dw1 = __fadd_rn(__fadd_rn(__fmul_rn(g0, pb.x), __fmul_rn(g1, pb.y)), __fmul_rn(g2, pb.z));
        const float dD = __fadd_rn(__fmul_rn(-dw0, __fdiv_rn(w.w0, w.D)), __fmul_rn(-dw1, __fdiv_rn(w.w1, w.D)));
        float wv, ds;
        if (v == ab.x) { wv = w.w0; ds = __fadd_rn(__fdiv_rn(dw1, w.D), dD); }
        else { wv = w.w1; ds = -__fadd_rn(__fdiv_rn(dw0, w.D), dD); }
        gx = __fadd_rn(gx, __fmul_rn(g0, wv));
        gy = __fadd_rn(gy, __fmul_rn(g1, wv));
        gz = __fadd_rn(gz, __fmul_rn(g2, wv));
        gs = __fadd_rn(gs, ds);
    }
    d_pos[3 * (int64_t)v] = gx; d_pos[3 * (int64_t)v + 1] = gy; d_pos[3 * (int64_t)v + 2] = gz;
    d_sdf[v] = gs;
}

// ---- sdf_reg_loss ----
__device__ __forceinline__ int sgn(float x) { return (int)(0.0f < x) - (int)(x < 0.0f); }      // torch.sign: 0 for +-0 and NaN
__device__ __forceinline__ bool reg_mask(float s0, float s1) { return sgn(s0) != sgn(s1); }
__device__ __forceinline__ double bce(double x, double y) { return log1p(exp(-fabs(x))) + fmax(x, 0.0) - x * y; }

__device__ __forceinline__ double warp_sum_d(double v)
{
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
    return v;
}

// fixed-order sum of (a, b, c) over the CTA; the result is valid in thread 0
__device__ __forceinline__ void block_sum3(double &a, double &b, double &c)
{
    __shared__ double s[3][256 / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    a = warp_sum_d(a); b = warp_sum_d(b); c = warp_sum_d(c);
    if (lane == 0) { s[0][warp] = a; s[1][warp] = b; s[2][warp] = c; }
    __syncthreads();
    if (threadIdx.x == 0) {
        a = b = c = 0.0;
        for (int w = 0; w < 256 / 32; ++w) { a += s[0][w]; b += s[1][w]; c += s[2][w]; }
    }
}

__global__ void __launch_bounds__(256) k_reg_partial(const float *__restrict__ sdf, int64_t ss, const int2 *__restrict__ edges, int E,
                                                     double *__restrict__ part)
{
    double s0 = 0.0, s1 = 0.0, cnt = 0.0;
    const int i1 = min(E, (int)(blockIdx.x + 1) * REG_CHUNK);
    for (int i = blockIdx.x * REG_CHUNK + threadIdx.x; i < i1; i += 256) {
        const int2 e = __ldg(edges + i);
        const float a = __ldg(sdf + (int64_t)e.x * ss), b = __ldg(sdf + (int64_t)e.y * ss);
        if (!reg_mask(a, b)) continue;
        s0 += bce((double)a, b > 0.0f ? 1.0 : 0.0);
        s1 += bce((double)b, a > 0.0f ? 1.0 : 0.0);
        cnt += 1.0;
    }
    block_sum3(s0, s1, cnt);
    if (threadIdx.x == 0) { part[3 * blockIdx.x] = s0; part[3 * blockIdx.x + 1] = s1; part[3 * blockIdx.x + 2] = cnt; }
}

__global__ void __launch_bounds__(256) k_reg_finish(const double *__restrict__ part, int nparts, float *__restrict__ loss, float *__restrict__ m)
{
    double s0 = 0.0, s1 = 0.0, cnt = 0.0;
    for (int i = threadIdx.x; i < nparts; i += 256) { s0 += part[3 * i]; s1 += part[3 * i + 1]; cnt += part[3 * i + 2]; }
    block_sum3(s0, s1, cnt);
    if (threadIdx.x == 0) {
        *loss = (float)(s0 / cnt + s1 / cnt);
        *m = (float)cnt;
    }
}

__global__ void __launch_bounds__(256) k_reg_bwd(const float *__restrict__ sdf, int64_t ss, int V, const int2 *__restrict__ edges,
                                                 const int32_t *__restrict__ off, const int32_t *__restrict__ adj, const float *__restrict__ m,
                                                 const float *__restrict__ d_loss, float *__restrict__ d_sdf)
{
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= V) return;
    const float M = __ldg(m), dl = __ldg(d_loss);
    float acc = 0.0f;
    const int j1 = __ldg(off + v + 1);
    for (int j = __ldg(off + v); j < j1; ++j) {
        const int2 e = __ldg(edges + __ldg(adj + j));
        const float a = __ldg(sdf + (int64_t)e.x * ss), b = __ldg(sdf + (int64_t)e.y * ss);
        if (!reg_mask(a, b)) continue;
        const float x = v == e.x ? a : b, y = (v == e.x ? b : a) > 0.0f ? 1.0f : 0.0f;
        const float sig = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x)));
        acc = __fadd_rn(acc, __fdiv_rn(__fmul_rn(__fsub_rn(sig, y), dl), M));
    }
    d_sdf[v] = acc;
}

int tiles(int n) { return (n + MCS_DMTET_TILE - 1) / MCS_DMTET_TILE; }

}  // namespace

int64_t mcs_dmtet_workspace_bytes(int32_t E, int32_t T)
{
    if (E < 1 || T < 1) return -1;
    return (int64_t)sizeof(unsigned long long) * (1 + tiles(E) + tiles(T));
}

int mcs_dmtet_count(const float *sdf, int64_t sdf_stride, const int32_t *edges, int32_t E, const int32_t *tets, int32_t T, int32_t *vid,
                    int32_t *tet_prefix, int32_t *counts, void *workspace, mcs_stream stream)
{
    MCS_REQUIRE(sdf && edges && tets && vid && tet_prefix && counts && workspace, "dmtet_count: null argument");
    MCS_REQUIRE(E >= 1 && T >= 1 && sdf_stride >= 0, "dmtet_count: bad sizes (E %d, T %d, sdf stride %lld)", E, T, (long long)sdf_stride);
    MCS_REQUIRE(((uintptr_t)edges & 7) == 0 && ((uintptr_t)tets & 15) == 0 && ((uintptr_t)tet_prefix & 7) == 0 && ((uintptr_t)workspace & 7) == 0,
                "dmtet_count: misaligned table or workspace");
    Grid g{};
    g.sdf = sdf; g.ss = sdf_stride;
    g.edges = (const int2 *)edges; g.E = E; g.tets = (const int4 *)tets; g.T = T;
    g.nEt = tiles(E); g.nTt = tiles(T);
    const cudaStream_t s = (cudaStream_t)stream;
    MCS_CUDA(cudaMemsetAsync(workspace, 0, (size_t)mcs_dmtet_workspace_bytes(E, T), s));
    k_dmt_count<<<g.nEt + g.nTt, DT_THREADS, 0, s>>>(g, vid, (int2 *)tet_prefix, counts, (unsigned long long *)workspace);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_dmtet_emit(const float *pos, int64_t pos_stride0, int64_t pos_stride1, const float *sdf, int64_t sdf_stride, const int32_t *edges, int32_t E,
                   const int32_t *tets, const int32_t *tet_edges, int32_t T, const int32_t *vid, const int32_t *tet_prefix, const int32_t *counts,
                   float *verts, int64_t *faces, int64_t *uv_idx, mcs_stream stream)
{
    MCS_REQUIRE(pos && sdf && edges && tets && tet_edges && vid && tet_prefix && counts && verts && faces && uv_idx, "dmtet_emit: null argument");
    MCS_REQUIRE(E >= 1 && T >= 1 && pos_stride0 >= 0 && pos_stride1 >= 0 && sdf_stride >= 0, "dmtet_emit: bad sizes or strides");
    MCS_REQUIRE(((uintptr_t)edges & 7) == 0 && ((uintptr_t)tets & 15) == 0 && ((uintptr_t)tet_prefix & 7) == 0, "dmtet_emit: misaligned table");
    Grid g{};
    g.sdf = sdf; g.ss = sdf_stride; g.pos = pos; g.ps0 = pos_stride0; g.ps1 = pos_stride1;
    g.edges = (const int2 *)edges; g.E = E; g.tets = (const int4 *)tets; g.tet_edges = tet_edges; g.T = T;
    const int eb = (E + 255) / 256, tb = (T + 255) / 256;
    k_dmt_emit<<<eb + tb, 256, 0, (cudaStream_t)stream>>>(g, vid, (const int2 *)tet_prefix, counts, verts, faces, uv_idx, eb);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_dmtet_bwd(const float *pos, int64_t pos_stride0, int64_t pos_stride1, const float *sdf, int64_t sdf_stride, int32_t V, const int32_t *edges,
                  int32_t E, const int32_t *vid, const int32_t *v2e_offsets, const int32_t *v2e_edges, const float *d_verts, float *d_pos, float *d_sdf,
                  mcs_stream stream)
{
    MCS_REQUIRE(pos && sdf && edges && vid && v2e_offsets && v2e_edges && d_verts && d_pos && d_sdf, "dmtet_bwd: null argument");
    MCS_REQUIRE(V >= 1 && E >= 1 && pos_stride0 >= 0 && pos_stride1 >= 0 && sdf_stride >= 0, "dmtet_bwd: bad sizes or strides");
    MCS_REQUIRE(((uintptr_t)edges & 7) == 0, "dmtet_bwd: misaligned edge table");
    Grid g{};
    g.sdf = sdf; g.ss = sdf_stride; g.pos = pos; g.ps0 = pos_stride0; g.ps1 = pos_stride1;
    g.edges = (const int2 *)edges; g.E = E;
    k_dmt_bwd<<<(V + 255) / 256, 256, 0, (cudaStream_t)stream>>>(g, V, vid, v2e_offsets, v2e_edges, d_verts, d_pos, d_sdf);
    MCS_LAUNCH_CHECK();
    return 0;
}

int32_t mcs_sdf_reg_num_partials(int32_t E) { return E < 1 ? 1 : (E + REG_CHUNK - 1) / REG_CHUNK; }

int mcs_sdf_reg_fwd(const float *sdf, int64_t sdf_stride, const int32_t *edges, int32_t E, double *partials, float *loss, float *m, mcs_stream stream)
{
    MCS_REQUIRE(sdf && partials && loss && m && (edges || E == 0), "sdf_reg_fwd: null argument");
    MCS_REQUIRE(E >= 0 && sdf_stride >= 0, "sdf_reg_fwd: bad sizes or strides");
    MCS_REQUIRE(((uintptr_t)edges & 7) == 0, "sdf_reg_fwd: misaligned edge table");
    const cudaStream_t s = (cudaStream_t)stream;
    const int np = mcs_sdf_reg_num_partials(E);
    k_reg_partial<<<np, 256, 0, s>>>(sdf, sdf_stride, (const int2 *)edges, E, partials);
    MCS_LAUNCH_CHECK();
    k_reg_finish<<<1, 256, 0, s>>>(partials, np, loss, m);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_sdf_reg_bwd(const float *sdf, int64_t sdf_stride, int32_t V, const int32_t *edges, const int32_t *v2e_offsets, const int32_t *v2e_edges,
                    const float *m, const float *d_loss, float *d_sdf, mcs_stream stream)
{
    MCS_REQUIRE(sdf && v2e_offsets && m && d_loss && d_sdf, "sdf_reg_bwd: null argument");
    MCS_REQUIRE(V >= 1 && sdf_stride >= 0, "sdf_reg_bwd: bad sizes or strides");
    MCS_REQUIRE(((uintptr_t)edges & 7) == 0, "sdf_reg_bwd: misaligned edge table");
    k_reg_bwd<<<(V + 255) / 256, 256, 0, (cudaStream_t)stream>>>(sdf, sdf_stride, V, (const int2 *)edges, v2e_offsets, v2e_edges, m, d_loss, d_sdf);
    MCS_LAUNCH_CHECK();
    return 0;
}
