// bvh.cu -- acceleration-structure build (LBVH) + stand-alone ray queries for sm_90a.
//
// Replaces optix_build_bvh -> optixAccelBuild (render/optixutils/c_src/torch_bindings.cpp:37-116),
// which the training loop calls EVERY iteration (geometry/dlmesh.py:50, dmtet.py:202).  The
// reference cudaFree/cudaMalloc's its buffers per call and builds on legacy stream 0; here the
// whole build is 11 hand-written launches (13 with the shadow view's own topology) on the caller's stream (incl. the onesweep radix sort), no host sync, no
// allocation in steady state (ctx.h), no library code.
//
// Pipeline (canonical, bit-identical to oracle/mcoracle.c:orc_lbvh_build so the integer structure
// can be compared exactly):
//   1. tri_bounds  : per-triangle AABB + reduction of centroid / scene bounds (order-preserving
//                    uint encoding + atomicMin/Max, warp-aggregated)
//   2. morton      : 30-bit Morton code of the AABB centre normalised to the centroid bounds
//   3. sort        : stable LSD radix sort of (code, triangle id), hand-written onesweep (k_rs_hist_all + 4 x k_rs_pass), 30 bits
//   4. karras      : Karras-2012 topology, one thread per internal node
//   5. leaves+refit: padded leaf boxes, sorted triangle records (v0,e1,e2 as 3 x float4), bottom-up
//                    box union with arrival counters (second thread to arrive continues)
//   6. emit        : 64-byte fp32 binary traversal nodes holding both children's boxes (stand-alone visibility / closest-hit queries)
//   7. emit_nodesq : 16-bit quantised child records on a scene-wide power-of-two grid, as a 4-wide (4 x 16 B: the grandchildren
//                    of binary node i) view of the same tree -- what the fused kernel's shadow rays walk above MCS_SAH_MAX_TRIS
//   8. ploc + emit_shadow (5 <= T <= MCS_SAH_MAX_TRIS, two more launches): the shadow rays' 4-wide view gets its own SAH
//                    topology and its own triangle order instead (see k_ploc)
#include "bvh_traverse.cuh"
#include "ctx.h"

int mcs_buf_reserve(DevBuf &b, size_t bytes, cudaStream_t s)
{
    if (bytes <= b.cap) return 0;
    size_t ncap = b.cap ? b.cap : 256;
    while (ncap < bytes) ncap *= 2;
    if (b.p) MCS_CUDA(cudaFreeAsync(b.p, s));
    b.p = nullptr; b.cap = 0;
    MCS_CUDA(cudaMallocAsync(&b.p, ncap, s));
    b.cap = ncap;
    return 0;
}

namespace {

// order-preserving float <-> uint mapping for atomicMin/atomicMax
__device__ __forceinline__ uint32_t f2ord(float f) { uint32_t b = __float_as_uint(f); return (b & 0x80000000u) ? ~b : (b | 0x80000000u); }
__device__ __forceinline__ float ord2f(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u); }

__global__ void k_bounds_init(uint32_t *bounds)
{
    int i = threadIdx.x;
    if (i < 12) bounds[i] = ((i / 3) & 1) ? 0u : 0xFFFFFFFFu;   // [0..2] cmin, [3..5] cmax, [6..8] smin, [9..11] smax
}

__global__ void __launch_bounds__(256) k_tri_bounds(const float *__restrict__ verts, const int32_t *__restrict__ tris, int T,
                                                    float *__restrict__ tlo, float *__restrict__ thi, uint32_t *bounds)
{
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    float c[3] = {0, 0, 0};
    bool valid = t < T;
    if (valid) {
        int i0 = tris[3 * t], i1 = tris[3 * t + 1], i2 = tris[3 * t + 2];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            float x = verts[3 * (size_t)i0 + a], y = verts[3 * (size_t)i1 + a], z = verts[3 * (size_t)i2 + a];
            lo[a] = fminf(x, fminf(y, z));
            hi[a] = fmaxf(x, fmaxf(y, z));
            c[a] = __fmul_rn(__fadd_rn(lo[a], hi[a]), 0.5f);
            tlo[3 * (size_t)t + a] = lo[a];
            thi[3 * (size_t)t + a] = hi[a];
        }
    }
    // warp shuffle reduction -> shared-memory atomics -> ONE set of 12 global atomics per CTA.  (One set per WARP, as in round 1, is
    // 400 k atomics on 12 addresses at 1 M triangles: 260 us, the largest item of the 715 us rebuild -- profiles/r02_bvh_build.json.)
    __shared__ uint32_t sb[12];
    if (threadIdx.x < 12) sb[threadIdx.x] = ((threadIdx.x / 3) & 1) ? 0u : 0xFFFFFFFFu;
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        float cmn = valid ? c[a] : INFINITY, cmx = valid ? c[a] : -INFINITY, smn = lo[a], smx = hi[a];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            cmn = fminf(cmn, __shfl_xor_sync(0xFFFFFFFFu, cmn, o));
            cmx = fmaxf(cmx, __shfl_xor_sync(0xFFFFFFFFu, cmx, o));
            smn = fminf(smn, __shfl_xor_sync(0xFFFFFFFFu, smn, o));
            smx = fmaxf(smx, __shfl_xor_sync(0xFFFFFFFFu, smx, o));
        }
        if ((threadIdx.x & 31) == 0 && cmn <= cmx) {
            atomicMin(sb + a, f2ord(cmn));
            atomicMax(sb + 3 + a, f2ord(cmx));
            atomicMin(sb + 6 + a, f2ord(smn));
            atomicMax(sb + 9 + a, f2ord(smx));
        }
    }
    __syncthreads();
    if (threadIdx.x < 12) {
        if ((threadIdx.x / 3) & 1) atomicMax(bounds + threadIdx.x, sb[threadIdx.x]);
        else atomicMin(bounds + threadIdx.x, sb[threadIdx.x]);
    }
}

__device__ __forceinline__ uint32_t expand_bits10(uint32_t v)
{
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}

__global__ void __launch_bounds__(256) k_morton(const float *__restrict__ tlo, const float *__restrict__ thi, int T, const uint32_t *__restrict__ bounds,
                                                uint32_t *__restrict__ keys, int32_t *__restrict__ vals)
{
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    uint32_t q[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        float cmin = ord2f(bounds[a]), cmax = ord2f(bounds[3 + a]);
        float ext = __fsub_rn(cmax, cmin);
        float c = __fmul_rn(__fadd_rn(tlo[3 * (size_t)t + a], thi[3 * (size_t)t + a]), 0.5f);
        float n = ext > 0.0f ? __fdiv_rn(__fsub_rn(c, cmin), ext) : 0.0f;
        int qi = (int)__fmul_rn(n, 1024.0f);
        q[a] = (uint32_t)min(max(qi, 0), 1023);
    }
    keys[t] = (expand_bits10(q[0]) << 2) | (expand_bits10(q[1]) << 1) | expand_bits10(q[2]);
    vals[t] = t;
}

// ---------------------------------------------------------------------------------------------
// Hand-written stable LSD radix sort of (Morton key, triangle id) pairs: 30-bit keys, four passes of 8 / 8 / 8 / 6 bits, one launch
// per pass ("onesweep": Adinets & Merrill 2022).  A launch of the upfront histogram kernel counts all four digits of every key once
// (global digit totals do not depend on the order); each pass kernel then
//   * takes tiles of RS_TILE = 4096 consecutive keys in TICKET order (an atomic counter: a tile's predecessors are always resident or
//     done, so the look-back below cannot deadlock);
//   * counts the tile's digits per warp (warp w owns 512 consecutive keys, walked in 16 rounds of 32 in index order);
//   * publishes the tile's digit counts and obtains its global offsets by DECOUPLED LOOK-BACK over the predecessors' flags (thread d
//     handles digit d: walk back until an inclusive prefix is found, adding aggregates on the way);
//   * scatters: rank within a round by __match_any_sync (lanes with the same digit, ordered by lane), rounds and warps in order, so
//     equal keys keep their input order -- the order of the oracle's qsort by (key, id) because ids start in increasing order.
// Replaces cub::DeviceRadixSort::SortPairs (round 1) with the same launch count; no library code is left in the rebuild.
// ---------------------------------------------------------------------------------------------
#define RS_THREADS 256
#define RS_ITEMS 16
#define RS_TILE (RS_THREADS * RS_ITEMS)
#define RS_FLAG_AGG 0x40000000u
#define RS_FLAG_PREFIX 0x80000000u
#define RS_VALUE_MASK 0x3FFFFFFFu

__host__ __device__ __forceinline__ int rs_shift(int pass) { return 8 * pass; }
__host__ __device__ __forceinline__ uint32_t rs_mask(int pass) { return pass == 3 ? 0x3Fu : 0xFFu; }

__global__ void __launch_bounds__(RS_THREADS) k_rs_hist_all(const uint32_t *__restrict__ keys, int T, uint32_t *__restrict__ G)
{
    __shared__ uint32_t h[4][256];
    for (int i = threadIdx.x; i < 1024; i += RS_THREADS) (&h[0][0])[i] = 0u;
    __syncthreads();
    const int base = blockIdx.x * RS_TILE;
#pragma unroll 4
    for (int k = 0; k < RS_ITEMS; ++k) {
        const int i = base + k * RS_THREADS + threadIdx.x;
        if (i < T) {
            const uint32_t key = keys[i];
            atomicAdd(&h[0][key & 0xFFu], 1u); atomicAdd(&h[1][(key >> 8) & 0xFFu], 1u);
            atomicAdd(&h[2][(key >> 16) & 0xFFu], 1u); atomicAdd(&h[3][(key >> 24) & 0x3Fu], 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 1024; i += RS_THREADS) {
        const uint32_t v = (&h[0][0])[i];
        if (v) atomicAdd(G + i, v);
    }
}

__global__ void __launch_bounds__(RS_THREADS) k_rs_pass(const uint32_t *__restrict__ keys_in, const int32_t *__restrict__ vals_in, uint32_t *__restrict__ keys_out,
                                                        int32_t *__restrict__ vals_out, int T, int pass, const uint32_t *__restrict__ G, unsigned int *ticket,
                                                        volatile uint32_t *flags)
{
    __shared__ uint32_t wc[RS_THREADS / 32][256];     // per-warp digit counts -> per-warp running output offsets
    __shared__ uint32_t dbase[256];                   // exclusive scan of the global digit totals
    __shared__ unsigned int s_tile;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int shift = rs_shift(pass);
    const uint32_t mask = rs_mask(pass);
    if (tid == 0) s_tile = atomicAdd(ticket, 1u);
    for (int i = tid; i < (RS_THREADS / 32) * 256; i += RS_THREADS) (&wc[0][0])[i] = 0u;
    {   // exclusive scan of G[pass][0..255] (one value per thread: warp scan + warp totals)
        const uint32_t g = __ldg(G + pass * 256 + tid);
        uint32_t x = g;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o); if (lane >= o) x += y; }
        __shared__ uint32_t wtot[RS_THREADS / 32];
        if (lane == 31) wtot[warp] = x;
        __syncthreads();
        uint32_t off = 0;
        for (int w = 0; w < warp; ++w) off += wtot[w];
        dbase[tid] = off + x - g;
    }
    __syncthreads();
    const int tile = (int)s_tile;
    const int wbase = tile * RS_TILE + warp * (RS_TILE / (RS_THREADS / 32));
    // ---- digits of this warp's 512 keys, in index order; per-warp counts ----
    uint32_t key[RS_ITEMS]; int32_t val[RS_ITEMS];
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const int i = wbase + r * 32 + lane;
        const bool ok = i < T;
        key[r] = ok ? keys_in[i] : 0xFFFFFFFFu;
        val[r] = ok ? vals_in[i] : 0;
        if (ok) atomicAdd(&wc[warp][(key[r] >> shift) & mask], 1u);
    }
    __syncthreads();
    // ---- digit d = tid: tile count, look-back, per-warp exclusive offsets ----
    {
        uint32_t cnt = 0;
#pragma unroll
        for (int w = 0; w < RS_THREADS / 32; ++w) cnt += wc[w][tid];
        volatile uint32_t *my_flag = flags + (size_t)tile * 256 + tid;
        *my_flag = cnt | RS_FLAG_AGG;
        uint32_t run = 0;
        for (int j = tile - 1; j >= 0; --j) {
            uint32_t f;
            do { f = flags[(size_t)j * 256 + tid]; } while (f == 0u);
            run += f & RS_VALUE_MASK;
            if (f & RS_FLAG_PREFIX) break;
        }
        __threadfence();
        *my_flag = ((run + cnt) & RS_VALUE_MASK) | RS_FLAG_PREFIX;
        uint32_t off = dbase[tid] + run;
#pragma unroll
        for (int w = 0; w < RS_THREADS / 32; ++w) { const uint32_t c = wc[w][tid]; wc[w][tid] = off; off += c; }
    }
    __syncthreads();
    // ---- stable scatter: rounds in order, lanes in order within a digit ----
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const bool ok = (wbase + r * 32 + lane) < T;
        const uint32_t d = ok ? ((key[r] >> shift) & mask) : 0x1FFu;
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, d);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        uint32_t pos = 0;
        if (ok) pos = wc[warp][d];
        __syncwarp();
        if (ok && rank == 0) wc[warp][d] = pos + (uint32_t)__popc(peers);
        __syncwarp();
        if (ok) { keys_out[pos + rank] = key[r]; vals_out[pos + rank] = val[r]; }
    }
}

static int rs_sort_pairs(uint32_t *keys_a, int32_t *vals_a, uint32_t *keys_b, int32_t *vals_b, int T, DevBuf &work, cudaStream_t s)
{
    // input in (keys_a, vals_a); four passes a -> b -> a -> b -> a: the sorted pairs end in (keys_a, vals_a)
    const int ntiles = (T + RS_TILE - 1) / RS_TILE;
    const size_t words = 4 * 256 + 4 + (size_t)4 * ntiles * 256;
    if (int e = mcs_buf_reserve(work, words * sizeof(uint32_t), s)) return e;
    uint32_t *G = (uint32_t *)work.p;
    unsigned int *tickets = (unsigned int *)(G + 4 * 256);
    uint32_t *flags = G + 4 * 256 + 4;
    MCS_CUDA(cudaMemsetAsync(work.p, 0, words * sizeof(uint32_t), s));
    k_rs_hist_all<<<ntiles, RS_THREADS, 0, s>>>(keys_a, T, G);
    MCS_LAUNCH_CHECK();
    for (int pass = 0; pass < 4; ++pass) {
        const bool fwd = (pass & 1) == 0;
        k_rs_pass<<<ntiles, RS_THREADS, 0, s>>>(fwd ? keys_a : keys_b, fwd ? vals_a : vals_b, fwd ? keys_b : keys_a, fwd ? vals_b : vals_a, T, pass, G, tickets + pass,
                                               flags + (size_t)pass * ntiles * 256);
        MCS_LAUNCH_CHECK();
    }
    return 0;
}

__device__ __forceinline__ int lbvh_delta(const uint32_t *__restrict__ k, int n, int i, int j)
{
    if (j < 0 || j >= n) return -1;
    uint32_t a = k[i], b = k[j];
    if (a == b) return 32 + __clz((uint32_t)i ^ (uint32_t)j);
    return __clz(a ^ b);
}

// Karras 2012, "Maximizing Parallelism in the Construction of BVHs, Octrees, and k-d Trees"
__global__ void __launch_bounds__(256) k_karras(const uint32_t *__restrict__ k, int T, int32_t *__restrict__ left, int32_t *__restrict__ right,
                                                int32_t *__restrict__ parent, int2 *__restrict__ range)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T - 1) return;
    int d = (lbvh_delta(k, T, i, i + 1) - lbvh_delta(k, T, i, i - 1)) >= 0 ? 1 : -1;
    int dmin = lbvh_delta(k, T, i, i - d);
    int lmax = 2;
    while (lbvh_delta(k, T, i, i + lmax * d) > dmin) lmax *= 2;
    int l = 0;
    for (int t = lmax / 2; t >= 1; t /= 2)
        if (lbvh_delta(k, T, i, i + (l + t) * d) > dmin) l += t;
    int j = i + l * d;
    int dnode = lbvh_delta(k, T, i, j);
    int sp = 0, t = l;
    do {
        t = (t + 1) >> 1;
        if (lbvh_delta(k, T, i, i + (sp + t) * d) > dnode) sp += t;
    } while (t > 1);
    int gamma = i + sp * d + (d < 0 ? -1 : 0);
    int lo_ = min(i, j), hi_ = max(i, j);
    int lc = (lo_ == gamma) ? (T - 1) + gamma : gamma;
    int rc = (hi_ == gamma + 1) ? (T - 1) + gamma + 1 : gamma + 1;
    left[i] = lc; right[i] = rc;
    parent[lc] = i; parent[rc] = i;
    range[i] = make_int2(lo_, hi_);           // sorted-triangle range covered by this node
    if (i == 0) parent[0] = -1;
}

// Bottom-up refit with arrival counters.  The triangles under an LBVH node are consecutive in Morton order, so a CTA that owns
// REFIT_THREADS consecutive leaves also owns every internal node whose range lies inside that span -- for those the publish / observe
// fences only have to order memory for threads of the SAME CTA (fence.cta); a device-wide fence is paid only at the few nodes whose
// range crosses a CTA boundary (the top ~log2(T / 1024) levels).  Round 1 fenced device-wide twice per level for every thread:
// 237 us of the 465 us rebuild at 1 M triangles, 50 of 136 us at 7 k (profiles/r02_bvh_build.json).
#define REFIT_THREADS 1024
__global__ void __launch_bounds__(REFIT_THREADS) k_leaves_refit(const float *__restrict__ verts, const int32_t *__restrict__ tris, int T,
                                                                const float *__restrict__ tlo, const float *__restrict__ thi,
                                                                const int32_t *__restrict__ prim, const uint32_t *__restrict__ bounds,
                                                                const int32_t *__restrict__ left, const int32_t *__restrict__ right, const int32_t *__restrict__ parent,
                                                                const int2 *__restrict__ range, float *lo, float *hi, int *flags, float4 *__restrict__ trirec)
{
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= T) return;
    const int span_lo = blockIdx.x * blockDim.x, span_hi = span_lo + blockDim.x - 1;
    float ex = __fsub_rn(ord2f(bounds[9]), ord2f(bounds[6]));
    float ey = __fsub_rn(ord2f(bounds[10]), ord2f(bounds[7]));
    float ez = __fsub_rn(ord2f(bounds[11]), ord2f(bounds[8]));
    float pad = __fmul_rn(1e-5f, fmaxf(ex, fmaxf(ey, ez)));
    int t = prim[j];
    int node = (T - 1) + j;
    float l[3], h[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        l[a] = __fsub_rn(tlo[3 * (size_t)t + a], pad);
        h[a] = __fadd_rn(thi[3 * (size_t)t + a], pad);
        lo[3 * (size_t)node + a] = l[a];
        hi[3 * (size_t)node + a] = h[a];
    }
    // sorted triangle record
    {
        int i0 = tris[3 * t], i1 = tris[3 * t + 1], i2 = tris[3 * t + 2];
        float ax = verts[3 * (size_t)i0], ay = verts[3 * (size_t)i0 + 1], az = verts[3 * (size_t)i0 + 2];
        float bx = verts[3 * (size_t)i1], by = verts[3 * (size_t)i1 + 1], bz = verts[3 * (size_t)i1 + 2];
        float cx = verts[3 * (size_t)i2], cy = verts[3 * (size_t)i2 + 1], cz = verts[3 * (size_t)i2 + 2];
        trirec[3 * (size_t)j + 0] = make_float4(ax, ay, az, __int_as_float(t));
        trirec[3 * (size_t)j + 1] = make_float4(__fsub_rn(bx, ax), __fsub_rn(by, ay), __fsub_rn(bz, az), 0.0f);
        trirec[3 * (size_t)j + 2] = make_float4(__fsub_rn(cx, ax), __fsub_rn(cy, ay), __fsub_rn(cz, az), 0.0f);
    }
    if (T == 1) return;
    // bottom-up: the second thread to reach a node computes its box
    int p = parent[node];
    while (p >= 0) {
        const int2 rg = range[p];
        const bool inside = rg.x >= span_lo && rg.y <= span_hi;      // every leaf under p belongs to this CTA
        if (inside) __threadfence_block(); else __threadfence();     // publish the child box this thread wrote
        if (atomicAdd(flags + p, 1) == 0) return;
        if (inside) __threadfence_block(); else __threadfence();     // observe the sibling's box
        int lc = left[p], rc = right[p];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            float v0 = __ldcg(lo + 3 * (size_t)lc + a), v1 = __ldcg(lo + 3 * (size_t)rc + a);
            float w0 = __ldcg(hi + 3 * (size_t)lc + a), w1 = __ldcg(hi + 3 * (size_t)rc + a);
            lo[3 * (size_t)p + a] = fminf(v0, v1);
            hi[3 * (size_t)p + a] = fmaxf(w0, w1);
        }
        p = parent[p];
    }
}

// Traversal nodes: node i holds the boxes of its two children.  A child whose subtree covers at most
// MCS_LEAF_MAX triangles is emitted as a leaf run (the triangles of an LBVH subtree are consecutive in
// Morton order); the internal nodes below it are simply never referenced.
__device__ __forceinline__ int child_code(int c, int T, const int2 *range)
{
    if (c >= T - 1) return ~(((c - (T - 1)) << 3) | 0);
    const int2 r = range[c];
    const int cnt = r.y - r.x + 1;
    return cnt <= MCS_LEAF_MAX ? ~((r.x << 3) | (cnt - 1)) : c;
}

__device__ __forceinline__ void emit_node(int i, int T, const int32_t *left, const int32_t *right, const int2 *range, const float *lo, const float *hi,
                                          float4 *nodes)
{
    if (T <= MCS_LEAF_MAX) {
        if (i == 0) {   // tiny mesh: the root is one leaf run; child 1 is an empty box (node 0 of lo/hi is the root box, or the only leaf)
            nodes[0] = make_float4(lo[0], hi[0], lo[1], hi[1]);
            nodes[1] = make_float4(INFINITY, -INFINITY, INFINITY, -INFINITY);
            nodes[2] = make_float4(lo[2], hi[2], INFINITY, -INFINITY);
            nodes[3] = make_float4(__int_as_float(~((0 << 3) | (T - 1))), __int_as_float(~0), 0.0f, 0.0f);
        }
        return;
    }
    if (i >= T - 1) return;
    int c0 = left[i], c1 = right[i];
    const float *l0 = lo + 3 * (size_t)c0, *h0 = hi + 3 * (size_t)c0, *l1 = lo + 3 * (size_t)c1, *h1 = hi + 3 * (size_t)c1;
    nodes[4 * (size_t)i + 0] = make_float4(l0[0], h0[0], l0[1], h0[1]);
    nodes[4 * (size_t)i + 1] = make_float4(l1[0], h1[0], l1[1], h1[1]);
    nodes[4 * (size_t)i + 2] = make_float4(l0[2], h0[2], l1[2], h1[2]);
    nodes[4 * (size_t)i + 3] = make_float4(__int_as_float(child_code(c0, T, range)), __int_as_float(child_code(c1, T, range)), 0.0f, 0.0f);
}

// Scene-wide quantisation grid of the shadow-ray view (see emit_nodeq): origin = root box min, cell = smallest power of two with
// 65532 cells covering the root extent.  lo / hi of node 0 are the root box (for T == 1: the only leaf).
__device__ __forceinline__ void quant_grid(const float *lo, const float *hi, float org[3], float inv_cell[3], float cell[3])
{
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        org[a] = lo[a];
        const float ext = __fsub_rn(hi[a], lo[a]);
        // smallest power of two >= ext / 65532 (exponent arithmetic: no rounding in the grid itself)
        int e;
        const float m = frexpf(fmaxf(ext, 1e-30f) * (1.0f / 65532.0f), &e);  // value = m * 2^e, m in [0.5, 1)
        const int k = (m == 0.5f) ? e - 1 : e;
        inv_cell[a] = ldexpf(1.0f, -k);
        cell[a] = ldexpf(1.0f, k);
    }
}

// One 16-byte child record: the box rounded outward on the grid and inflated by two cells per side; l == nullptr is an unused slot
// (inverted box, never entered).
__device__ __forceinline__ uint4 quant_child(const float *l, const float *h, const float org[3], const float inv_cell[3], uint32_t word)
{
    uint32_t ql[3] = {65535u, 65535u, 65535u}, qh[3] = {0u, 0u, 0u};
    if (l) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float fl = floorf(__fmul_rn(__fsub_rn(l[a], org[a]), inv_cell[a])) - 2.0f;
            const float fh = ceilf(__fmul_rn(__fsub_rn(h[a], org[a]), inv_cell[a])) + 2.0f;
            ql[a] = (uint32_t)fminf(fmaxf(fl, 0.0f), 65535.0f);
            qh[a] = (uint32_t)fminf(fmaxf(fh, 0.0f), 65535.0f);
        }
    }
    return make_uint4(ql[0] | (qh[0] << 16), ql[1] | (qh[1] << 16), ql[2] | (qh[2] << 16), word);
}

// Quantised 4-wide view of the tree for the shadow rays.  The fused kernel's trace loop is instruction-issue bound; with fp32
// 64-byte binary nodes (four loads per visit) the L1 data pipe was a co-limiter as well (75 % busy, profiles/r01_v5_*).  A child
// record with its box as 16-bit integers on ONE scene-wide grid is 16 bytes -- one 128-bit load per child:
//   uint4 child = { lo.x | hi.x << 16,  lo.y | hi.y << 16,  lo.z | hi.z << 16,  child code }
// and node i of the 4-wide view holds the records of the (up to four) GRANDCHILDREN of binary node i: half the visits per ray.
// Grid: origin = root box min, cell = smallest power of two with 65532 cells covering the root extent (per axis), so
// cell * (1/d) is exact and the decode is one byte-permute + one FMA per plane (envshade.cu:trace_queue); the permute also picks
// the entry / exit plane by the sign of the ray direction.  Boxes are rounded outward and inflated by two more cells per side,
// which covers the quantisation rounding and the < 0.51-cell error of the biased decode: culling stays conservative, the
// visibility result is unchanged (tests/test_gpu_envshade.py records tests, incl. a 330 k-triangle mesh).
__device__ __forceinline__ void emit_nodeq(const int i, int T, const int32_t *left, const int32_t *right, const int2 *range, const float *lo, const float *hi,
                                           uint4 *nodesq4, float *qgrid)
{
    float org[3], inv_cell[3], cell[3];
    quant_grid(lo, hi, org, inv_cell, cell);
    if (i == 0)
        for (int a = 0; a < 3; ++a) { qgrid[a] = org[a]; qgrid[3 + a] = cell[a]; qgrid[6 + a] = inv_cell[a]; }
    const bool tiny = T <= MCS_LEAF_MAX;
    if (!nodesq4 || (tiny ? i != 0 : i >= T - 1)) return;
    int cn[2], code[2];
    if (tiny) { cn[0] = 0; cn[1] = -1; code[0] = ~((0 << 3) | (T - 1)); code[1] = ~0; }
    else { cn[0] = left[i]; cn[1] = right[i]; code[0] = child_code(cn[0], T, range); code[1] = child_code(cn[1], T, range); }
    // 4-wide view: node i holds the (up to four) GRANDCHILDREN of binary node i -- a child that is a leaf run stays one slot, an
    // internal child is replaced by its two children.  Same index space as the binary nodes (no allocation; nodes on odd levels
    // are never referenced).  A ray visits ~half as many nodes (13.8 vs 28.8 on the benchmark mesh) and tests fewer boxes (52 vs 58).
    // Unused slots are inverted boxes (lo = 65535, hi = 0): with sign-selected planes entry > exit for every ray.
    int gn[4] = {-1, -1, -1, -1}, gcode[4] = {~0, ~0, ~0, ~0}, ng = 0;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
        if (cn[c] < 0) continue;
        if (code[c] < 0) { gn[ng] = cn[c]; gcode[ng] = code[c]; ++ng; }
        else {
            const int g0 = left[cn[c]], g1 = right[cn[c]];
            gn[ng] = g0; gcode[ng] = child_code(g0, T, range); ++ng;
            gn[ng] = g1; gcode[ng] = child_code(g1, T, range); ++ng;
        }
    }
    // child words: the payload (internal: node index; leaf run: (first triangle << 3) | (count - 1)) in the low 28 bits; the top
    // nibble of slot 0 flags which of the four slots are leaf runs, so the walker classifies all four with one shift and two ANDs.
    // Unused slots are flagged as leaves with an inverted box (never entered).
    uint32_t leaf_bits = 0u;
#pragma unroll
    for (int c = 0; c < 4; ++c) leaf_bits |= (gcode[c] < 0 ? 1u : 0u) << c;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const uint32_t payload = (uint32_t)(gcode[c] < 0 ? ~gcode[c] : gcode[c]) & 0x0FFFFFFFu;
        const bool used = gn[c] >= 0;
        nodesq4[4 * (size_t)i + c] = quant_child(used ? lo + 3 * (size_t)gn[c] : nullptr, used ? hi + 3 * (size_t)gn[c] : nullptr, org, inv_cell,
                                                 payload | (c == 0 ? leaf_bits << 28 : 0u));
    }
}

// One launch for both node views.  nodesq4 == nullptr: only the grid is written (the shadow-ray view comes from k_emit_shadow).
__global__ void __launch_bounds__(256) k_emit_both(int T, const int32_t *left, const int32_t *right, const int2 *range, const float *lo, const float *hi,
                                                   float4 *nodes, uint4 *nodesq4, float *qgrid)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    emit_node(i, T, left, right, range, lo, hi, nodes);
    emit_nodeq(i, T, left, right, range, lo, hi, nodesq4, qgrid);
}

// ---------------------------------------------------------------------------------------------
// SAH topology for the shadow-ray view.  The any-hit shadow rays (two env_shade launches per training step) are most of the
// step; the Morton LBVH they used to walk is the lowest-quality tree in common use.  So the shadow view gets its own tree, rebuilt
// with the LBVH every iteration (the geometry is trainable):
//   * k_ploc: PLOC clustering (Meister & Bittner, "Parallel Locally-Ordered Clustering for BVH construction", TVCG 2018) over the
//     leaves in Morton order, in ONE CTA: every cluster finds its nearest neighbour (smallest merged surface area) among the
//     PLOC_RADIUS clusters on either side, mutual pairs merge, the array is compacted in order; repeat until one cluster is left.
//     Ties go to the lower index, so the minimum-area pair of every round is mutual and each round merges at least one pair.  A
//     merged node is collapsed to a leaf run when it has <= SAH_LEAF_MAX triangles and the leaf's SAH cost does not exceed the
//     subtree's.  Then, top-down in reverse creation order, every node gets the first slot of its triangles in depth-first
//     leaf order, so the triangles of every subtree (and of every leaf run) are consecutive.
//   * k_emit_shadow: the triangle records in that order, and the 4-wide quantised nodes by an SAH-greedy collapse (open the
//     internal child of largest surface area until there are four).  Record format, leaf nibble, grid and inflation as emit_nodeq.
// The canonical LBVH, its fp32 nodes and its Morton-ordered triangle records (closest-hit queries, trace_visibility, export) are
// not touched.  Above MCS_SAH_MAX_TRIS triangles one CTA takes too long and the shadow view stays the LBVH grandchild collapse.
// A refit (rebuild = 0) reruns the clustering on the refitted leaf boxes in the Morton order of the last rebuild.
// ---------------------------------------------------------------------------------------------
#ifndef MCS_SAH_MAX_TRIS
#define MCS_SAH_MAX_TRIS 16384
#endif
#define PLOC_THREADS 1024
#define PLOC_RADIUS 8           // radius 16: same kernel time on the bench mesh, 130 us more per rebuild
#define SAH_LEAF_MAX 8          // 3-bit count field of a leaf run
#define SAH_CI 1.2f             // cost of a binary node relative to one triangle test (2.0: equal, 3.0: slower kernel)
#define SAH_CT 1.0f

__device__ __forceinline__ float half_area(float4 l, float4 h)
{
    const float dx = h.x - l.x, dy = h.y - l.y, dz = h.z - l.z;
    return dx * dy + dy * dz + dz * dx;
}

// exclusive block scan of two counters (PLOC_THREADS threads); *total = the sums
__device__ __forceinline__ int2 block_exscan2(int2 v, int2 *total, int2 *sw)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int2 x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int yx = __shfl_up_sync(0xFFFFFFFFu, x.x, o), yy = __shfl_up_sync(0xFFFFFFFFu, x.y, o);
        if (lane >= o) { x.x += yx; x.y += yy; }
    }
    if (lane == 31) sw[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int2 w = sw[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int yx = __shfl_up_sync(0xFFFFFFFFu, w.x, o), yy = __shfl_up_sync(0xFFFFFFFFu, w.y, o);
            if (lane >= o) { w.x += yx; w.y += yy; }
        }
        sw[lane] = w;
    }
    __syncthreads();
    const int2 base = warp ? sw[warp - 1] : make_int2(0, 0);
    *total = sw[31];
    return make_int2(base.x + x.x - v.x, base.y + x.y - v.y);
}

struct ShadowTree {
    int32_t *left, *right;  // [T-1] children (internal 0..T-2, root 0; leaf of sorted triangle j: T-1+j)
    float4 *box;            // [T-1][2] lo (w: unused), hi
    int32_t *cnt;           // [T-1] triangles under the node; negative: the node is a leaf run of -cnt triangles
    int32_t *first;         // [2T-1] first slot of the node's triangles in depth-first leaf order
};

// Scratch: cluster ids [2][T], cluster boxes [2][T][2] (lo.w = SAH cost, hi.w = triangle count), nearest neighbour [T], next free
// node id before each round [T].
__global__ void __launch_bounds__(PLOC_THREADS) k_ploc(int T, const float *lo, const float *hi, ShadowTree st, int32_t *cid, float4 *cbox, int32_t *nn,
                                                       int32_t *round_id)
{
    __shared__ int2 sw[32];
    const int tid = threadIdx.x;
    for (int j = tid; j < T; j += PLOC_THREADS) {
        const size_t n = (size_t)(T - 1 + j);
        const float4 l = make_float4(lo[3 * n], lo[3 * n + 1], lo[3 * n + 2], 0.0f), h = make_float4(hi[3 * n], hi[3 * n + 1], hi[3 * n + 2], 0.0f);
        cid[j] = T - 1 + j;
        cbox[2 * j] = make_float4(l.x, l.y, l.z, SAH_CT * half_area(l, h));
        cbox[2 * j + 1] = make_float4(h.x, h.y, h.z, __int_as_float(1));
    }
    __syncthreads();
    int n = T, next_id = T - 2, rounds = 0, buf = 0;
    while (n > 1) {
        int32_t *ci = cid + (size_t)buf * T, *co = cid + (size_t)(buf ^ 1) * T;
        float4 *bi = cbox + (size_t)buf * 2 * T, *bo = cbox + (size_t)(buf ^ 1) * 2 * T;
        if (tid == 0) round_id[rounds] = next_id;
        // ---- nearest neighbour within the radius (ties: lower index) ----
        for (int i = tid; i < n; i += PLOC_THREADS) {
            const float4 li = bi[2 * i], hi_ = bi[2 * i + 1];
            float best = INFINITY;
            int bj = -1;
            const int j0 = max(0, i - PLOC_RADIUS), j1 = min(n - 1, i + PLOC_RADIUS);
            for (int j = j0; j <= j1; ++j) {
                if (j == i) continue;
                const float4 lj = bi[2 * j], hj = bi[2 * j + 1];
                // (NaN -> +inf keeps the order total, so a mutual pair exists even for non-finite geometry)
                const float a = fminf(half_area(make_float4(fminf(li.x, lj.x), fminf(li.y, lj.y), fminf(li.z, lj.z), 0.0f),
                                                make_float4(fmaxf(hi_.x, hj.x), fmaxf(hi_.y, hj.y), fmaxf(hi_.z, hj.z), 0.0f)), INFINITY);
                if (a < best || bj < 0) { best = a; bj = j; }
            }
            nn[i] = bj;
        }
        __syncthreads();
        // ---- merge mutual pairs (the lower index keeps the merged cluster), compact in order ----
        const int per = (n + PLOC_THREADS - 1) / PLOC_THREADS, beg = min(n, tid * per), end = min(n, beg + per);
        int2 mine = make_int2(0, 0);            // (clusters kept, merges)
        for (int i = beg; i < end; ++i) {
            const int j = nn[i];
            const bool mutual = nn[j] == i;
            mine.x += (!mutual || i < j) ? 1 : 0;
            mine.y += (mutual && i < j) ? 1 : 0;
        }
        int2 tot;
        int2 pos = block_exscan2(mine, &tot, sw);
        for (int i = beg; i < end; ++i) {
            const int j = nn[i];
            const bool mutual = nn[j] == i;
            if (mutual && i > j) continue;
            if (!mutual) { co[pos.x] = ci[i]; bo[2 * pos.x] = bi[2 * i]; bo[2 * pos.x + 1] = bi[2 * i + 1]; ++pos.x; continue; }
            const float4 la = bi[2 * i], ha = bi[2 * i + 1], lb = bi[2 * j], hb = bi[2 * j + 1];
            const float4 l = make_float4(fminf(la.x, lb.x), fminf(la.y, lb.y), fminf(la.z, lb.z), 0.0f);
            const float4 h = make_float4(fmaxf(ha.x, hb.x), fmaxf(ha.y, hb.y), fmaxf(ha.z, hb.z), 0.0f);
            const float A = half_area(l, h);
            const int cnt = __float_as_int(ha.w) + __float_as_int(hb.w);
            const float c_int = SAH_CI * A + la.w + lb.w, c_leaf = SAH_CT * A * (float)cnt;
            const bool leaf = cnt <= SAH_LEAF_MAX && c_leaf <= c_int;
            const int id = next_id - pos.y;
            st.left[id] = ci[i]; st.right[id] = ci[j];
            st.box[2 * id] = l; st.box[2 * id + 1] = h;
            st.cnt[id] = leaf ? -cnt : cnt;
            co[pos.x] = id;
            bo[2 * pos.x] = make_float4(l.x, l.y, l.z, leaf ? c_leaf : c_int);
            bo[2 * pos.x + 1] = make_float4(h.x, h.y, h.z, __int_as_float(cnt));
            ++pos.x; ++pos.y;
        }
        n = tot.x; next_id -= tot.y; buf ^= 1; ++rounds;
        __syncthreads();
    }
    // ---- depth-first leaf order, top-down: a node is created in a later round than its children ----
    if (tid == 0) { round_id[rounds] = next_id; st.first[0] = 0; }      // next_id == -1: the last merge created the root, node 0
    __syncthreads();
    for (int r = rounds - 1; r >= 0; --r) {
        for (int id = round_id[r + 1] + 1 + tid; id <= round_id[r]; id += PLOC_THREADS) {
            const int f = st.first[id], l = st.left[id];
            st.first[l] = f;
            st.first[st.right[id]] = f + (l >= T - 1 ? 1 : abs(st.cnt[l]));
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_emit_shadow(int T, ShadowTree st, const float *lo, const float *hi, const float4 *__restrict__ tris,
                                                     float4 *__restrict__ stris, uint4 *__restrict__ nodesq4)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= T) return;
    {   // triangle records in depth-first leaf order
        const int d = st.first[T - 1 + i];
        stris[3 * (size_t)d] = tris[3 * (size_t)i];
        stris[3 * (size_t)d + 1] = tris[3 * (size_t)i + 1];
        stris[3 * (size_t)d + 2] = tris[3 * (size_t)i + 2];
    }
    if (i >= T - 1 || (i != 0 && st.cnt[i] < 0)) return;       // leaf runs have no node (the root is always a node)
    auto is_node = [&](int x) { return x < T - 1 && st.cnt[x] > 0; };
    int s[4] = {st.left[i], st.right[i], -1, -1}, ns = 2;
    while (ns < 4) {     // open the internal child of largest surface area
        int b = -1;
        float ba = -1.0f;
        for (int c = 0; c < ns; ++c)
            if (is_node(s[c])) {
                const float a = half_area(st.box[2 * s[c]], st.box[2 * s[c] + 1]);
                if (a > ba) { ba = a; b = c; }
            }
        if (b < 0) break;
        const int x = s[b];
        s[b] = st.left[x]; s[ns++] = st.right[x];
    }
    float org[3], inv_cell[3], cell[3];
    quant_grid(lo, hi, org, inv_cell, cell);
    uint32_t leaf_bits = 0u;
    for (int c = 0; c < 4; ++c) leaf_bits |= (c >= ns || !is_node(s[c]) ? 1u : 0u) << c;
    for (int c = 0; c < 4; ++c) {
        uint32_t payload = 0u;
        const float *l = nullptr, *h = nullptr;
        float bl[3], bh[3];
        if (c < ns) {
            const int x = s[c];
            if (x >= T - 1) { l = lo + 3 * (size_t)x; h = hi + 3 * (size_t)x; payload = (uint32_t)st.first[x] << 3; }
            else {
                const float4 a = st.box[2 * x], b = st.box[2 * x + 1];
                bl[0] = a.x; bl[1] = a.y; bl[2] = a.z; bh[0] = b.x; bh[1] = b.y; bh[2] = b.z;
                l = bl; h = bh;
                payload = st.cnt[x] > 0 ? (uint32_t)x : ((uint32_t)st.first[x] << 3) | (uint32_t)(-st.cnt[x] - 1);
            }
        }
        nodesq4[4 * (size_t)i + c] = quant_child(l, h, org, inv_cell, (payload & 0x0FFFFFFFu) | (c == 0 ? leaf_bits << 28 : 0u));
    }
}

typedef BvhView VisView;
__global__ void __launch_bounds__(128) k_visibility(VisView b, const float *__restrict__ ro, const float *__restrict__ rd, int64_t n, uint8_t *__restrict__ vis)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    f3 o = F3(ro[3 * i], ro[3 * i + 1], ro[3 * i + 2]), d = F3(rd[3 * i], rd[3 * i + 1], rd[3 * i + 2]);
    vis[i] = bvh_occluded(b, o, d) ? 0 : 1;        // fp32 nodes, same triangles and predicate as the fused env_shade kernel
}

// AFTER: only hits with t > peel_sep(t_after[i]) count.  +inf gives a miss: every box's clamped entry is +inf, so the walk ends after
// the root.  A template parameter rather than a null test, so that the plain query keeps its constant bound (46 registers, not 47).
template <bool AFTER>
__global__ void __launch_bounds__(128) k_closest(BvhView b, const float *__restrict__ ro, const float *__restrict__ rd, const float *__restrict__ t_after,
                                                 int64_t n, int32_t *__restrict__ tri_id, float *__restrict__ tuv)
{
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    f3 o = F3(ro[3 * i], ro[3 * i + 1], ro[3 * i + 2]), d = F3(rd[3 * i], rd[3 * i + 1], rd[3 * i + 2]);
    float t, u, v;
    int id = bvh_closest(b, o, d, AFTER ? peel_sep(t_after[i]) : 0.0f, t, u, v);
    tri_id[i] = id; tuv[3 * i] = t; tuv[3 * i + 1] = u; tuv[3 * i + 2] = v;
}

inline unsigned nblk(int64_t n, int b) { return (unsigned)((n + b - 1) / b); }

}  // namespace

extern "C" {

int mcs_ctx_create(mcs_ctx **out)
{
    MCS_REQUIRE(out != nullptr, "mcs_ctx_create: null output pointer");
    int dev = 0;
    MCS_CUDA(cudaGetDevice(&dev));
    mcs_ctx *c = new mcs_ctx();
    c->device = dev;
    *out = c;
    return 0;
}

int mcs_ctx_destroy(mcs_ctx *c)
{
    delete c;
    return 0;
}

int mcs_bvh_build(mcs_ctx *c, const float *verts, int32_t V, const int32_t *tris, int32_t T, uint32_t rebuild, mcs_stream stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    MCS_REQUIRE(c != nullptr, "mcs_bvh_build: null context");
    MCS_REQUIRE(verts && tris, "mcs_bvh_build: null geometry pointer");
    // ops.py:131-132: "Got empty training triangle mesh (unrecoverable discontinuity)"
    MCS_REQUIRE(T > 0 && V > 0, "Got empty training triangle mesh (unrecoverable discontinuity)");
    MCS_REQUIRE(T <= (1 << 25), "mcs_bvh_build: at most 2^25 triangles (28-bit child words of the quantised nodes), got %d", T);
    MCS_REQUIRE(rebuild != 0 || c->T == T, "mcs_bvh_build: refit (rebuild=0) needs an existing structure with the same triangle count (have %d, got %d)", c->T, T);
    const bool sah = T > MCS_LEAF_MAX && T <= MCS_SAH_MAX_TRIS;       // does the shadow view get its own SAH topology?
    const size_t nT = (size_t)T, nN = 2 * nT - 1;
    const size_t sT = sah ? nT : 0, sN = sah ? nN : 0;                 // 0: the SAH topology's buffers are left as they are
    const struct { DevBuf &b; size_t bytes; } need[] = {
        {c->bounds, 12 * sizeof(uint32_t)}, {c->tlo, nT * 3 * sizeof(float)}, {c->thi, nT * 3 * sizeof(float)},
        {c->keys, nT * sizeof(uint32_t)}, {c->keys_alt, nT * sizeof(uint32_t)}, {c->vals, nT * sizeof(int32_t)}, {c->vals_alt, nT * sizeof(int32_t)},
        {c->left, nT * sizeof(int32_t)}, {c->right, nT * sizeof(int32_t)}, {c->parent, nN * sizeof(int32_t)},
        {c->lo, nN * 3 * sizeof(float)}, {c->hi, nN * 3 * sizeof(float)}, {c->flags, nT * sizeof(int)}, {c->range, nT * sizeof(int2)},
        {c->nodes, nT * 4 * sizeof(float4)}, {c->tris, nT * 3 * sizeof(float4)}, {c->nodesq4, nT * 4 * sizeof(uint4)}, {c->qgrid, 16 * sizeof(float)},
        {c->sleft, sT * sizeof(int32_t)}, {c->sright, sT * sizeof(int32_t)}, {c->scnt, sT * sizeof(int32_t)}, {c->sbox, sT * 2 * sizeof(float4)},
        {c->sfirst, sN * sizeof(int32_t)}, {c->cbox, sT * 4 * sizeof(float4)}, {c->cid, sT * 2 * sizeof(int32_t)}, {c->nn, sT * sizeof(int32_t)},
        {c->round_id, sT * sizeof(int32_t)}, {c->stris, sT * 3 * sizeof(float4)},
    };
    for (const auto &r : need)
        if (int e = mcs_buf_reserve(r.b, r.bytes, s)) return e;
    c->shadow = BvhView{nullptr, (const float4 *)(sah ? c->stris.p : c->tris.p), (const float *)c->qgrid.p, (const uint4 *)c->nodesq4.p};

    uint32_t *bounds = (uint32_t *)c->bounds.p;
    float *tlo = (float *)c->tlo.p, *thi = (float *)c->thi.p;
    k_bounds_init<<<1, 32, 0, s>>>(bounds);
    k_tri_bounds<<<nblk(T, 256), 256, 0, s>>>(verts, tris, T, tlo, thi, bounds);
    MCS_LAUNCH_CHECK();
    if (rebuild) {
        // Measured and dropped for the small meshes (7-11 k triangles, where any multi-pass sort is latency-bound launches): a single-CTA
        // shared-memory bitonic sort of 64-bit (key, id) composites -- bit-identical structure but 60-140 us on one SM; and the whole
        // rebuild as ONE single-CTA launch -- 522 us (seven dependent gather / refit chains per thread).  profiles/r02_bvh_build.json.
        k_morton<<<nblk(T, 256), 256, 0, s>>>(tlo, thi, T, bounds, (uint32_t *)c->keys_alt.p, (int32_t *)c->vals_alt.p);
        MCS_LAUNCH_CHECK();
        if (int e = rs_sort_pairs((uint32_t *)c->keys_alt.p, (int32_t *)c->vals_alt.p, (uint32_t *)c->keys.p, (int32_t *)c->vals.p, T, c->sort_tmp, s)) return e;
        if (T > 1) {
            k_karras<<<nblk(T - 1, 256), 256, 0, s>>>((const uint32_t *)c->keys_alt.p, T, (int32_t *)c->left.p, (int32_t *)c->right.p, (int32_t *)c->parent.p,
                                                      (int2 *)c->range.p);
            MCS_LAUNCH_CHECK();
        }
    }
    MCS_CUDA(cudaMemsetAsync(c->flags.p, 0, nT * sizeof(int), s));
    k_leaves_refit<<<nblk(T, REFIT_THREADS), REFIT_THREADS, 0, s>>>(verts, tris, T, tlo, thi, (const int32_t *)c->vals_alt.p, bounds, (const int32_t *)c->left.p,
                                                                   (const int32_t *)c->right.p, (const int32_t *)c->parent.p, (const int2 *)c->range.p,
                                                                   (float *)c->lo.p, (float *)c->hi.p, (int *)c->flags.p, (float4 *)c->tris.p);
    MCS_LAUNCH_CHECK();
    k_emit_both<<<nblk(T > 1 ? T - 1 : 1, 256), 256, 0, s>>>(T, (const int32_t *)c->left.p, (const int32_t *)c->right.p, (const int2 *)c->range.p,
                                                              (const float *)c->lo.p, (const float *)c->hi.p, (float4 *)c->nodes.p,
                                                              sah ? nullptr : (uint4 *)c->nodesq4.p, (float *)c->qgrid.p);
    MCS_LAUNCH_CHECK();
    if (sah) {
        const ShadowTree st{(int32_t *)c->sleft.p, (int32_t *)c->sright.p, (float4 *)c->sbox.p, (int32_t *)c->scnt.p, (int32_t *)c->sfirst.p};
        k_ploc<<<1, PLOC_THREADS, 0, s>>>(T, (const float *)c->lo.p, (const float *)c->hi.p, st, (int32_t *)c->cid.p, (float4 *)c->cbox.p,
                                          (int32_t *)c->nn.p, (int32_t *)c->round_id.p);
        MCS_LAUNCH_CHECK();
        k_emit_shadow<<<nblk(T, 256), 256, 0, s>>>(T, st, (const float *)c->lo.p, (const float *)c->hi.p, (const float4 *)c->tris.p, (float4 *)c->stris.p,
                                                   (uint4 *)c->nodesq4.p);
        MCS_LAUNCH_CHECK();
    }
    c->T = T; c->V = V;
    return 0;
}

int mcs_bvh_export(mcs_ctx *c, uint32_t *morton, int32_t *prim, int32_t *left, int32_t *right, float *lo, float *hi, mcs_stream stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    MCS_REQUIRE(c && c->T > 0, "mcs_bvh_export: no acceleration structure built");
    size_t T = (size_t)c->T;
    MCS_CUDA(cudaMemcpyAsync(morton, c->keys_alt.p, T * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
    MCS_CUDA(cudaMemcpyAsync(prim, c->vals_alt.p, T * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    if (T > 1) {
        MCS_CUDA(cudaMemcpyAsync(left, c->left.p, (T - 1) * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
        MCS_CUDA(cudaMemcpyAsync(right, c->right.p, (T - 1) * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
    }
    MCS_CUDA(cudaMemcpyAsync(lo, c->lo.p, (2 * T - 1) * 3 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    MCS_CUDA(cudaMemcpyAsync(hi, c->hi.p, (2 * T - 1) * 3 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return 0;
}

int mcs_bvh_export_shadow(mcs_ctx *c, uint32_t *nodesq4, float *tris, float *qgrid, mcs_stream stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    MCS_REQUIRE(c && c->T > 0, "mcs_bvh_export_shadow: no acceleration structure built");
    const size_t T = (size_t)c->T;
    MCS_CUDA(cudaMemcpyAsync(nodesq4, c->shadow.nodesq4, (T > 1 ? T - 1 : 1) * 4 * sizeof(uint4), cudaMemcpyDeviceToDevice, s));
    MCS_CUDA(cudaMemcpyAsync(tris, c->shadow.tris, T * 3 * sizeof(float4), cudaMemcpyDeviceToDevice, s));
    MCS_CUDA(cudaMemcpyAsync(qgrid, c->shadow.qgrid, 9 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return 0;
}

int mcs_trace_visibility(mcs_ctx *c, const float *ro, const float *rd, int64_t n, uint8_t *vis, mcs_stream stream)
{
    MCS_REQUIRE(c && c->T > 0, "mcs_trace_visibility: no acceleration structure built (call mcs_bvh_build first)");
    MCS_REQUIRE(n >= 0 && (n == 0 || (ro && rd && vis)), "mcs_trace_visibility: bad arguments");
    if (n == 0) return 0;
    VisView b{(const float4 *)c->nodes.p, (const float4 *)c->tris.p, nullptr, nullptr};
    k_visibility<<<nblk(n, 128), 128, 0, (cudaStream_t)stream>>>(b, ro, rd, n, vis);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_trace_closest(mcs_ctx *c, const float *ro, const float *rd, int64_t n, int32_t *tri_id, float *tuv, mcs_stream stream)
{
    MCS_REQUIRE(c && c->T > 0, "mcs_trace_closest: no acceleration structure built (call mcs_bvh_build first)");
    MCS_REQUIRE(n >= 0 && (n == 0 || (ro && rd && tri_id && tuv)), "mcs_trace_closest: bad arguments");
    if (n == 0) return 0;
    BvhView b{(const float4 *)c->nodes.p, (const float4 *)c->tris.p, nullptr, nullptr};
    k_closest<false><<<nblk(n, 128), 128, 0, (cudaStream_t)stream>>>(b, ro, rd, nullptr, n, tri_id, tuv);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_trace_closest_after(mcs_ctx *c, const float *ro, const float *rd, const float *t_after, int64_t n, int32_t *tri_id, float *tuv,
                            mcs_stream stream)
{
    MCS_REQUIRE(c && c->T > 0, "mcs_trace_closest_after: no acceleration structure built (call mcs_bvh_build first)");
    MCS_REQUIRE(n >= 0 && (n == 0 || (ro && rd && t_after && tri_id && tuv)), "mcs_trace_closest_after: bad arguments");
    if (n == 0) return 0;
    BvhView b{(const float4 *)c->nodes.p, (const float4 *)c->tris.p, nullptr, nullptr};
    k_closest<true><<<nblk(n, 128), 128, 0, (cudaStream_t)stream>>>(b, ro, rd, t_after, n, tri_id, tuv);
    MCS_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
