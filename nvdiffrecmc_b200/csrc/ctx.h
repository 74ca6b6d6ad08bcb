// ctx.h -- the opaque per-scene context behind mcs_ctx (replaces OptiXState,
// render/optixutils/c_src/optix_wrapper.h:17-37): owns the acceleration structure and all build
// workspace.  Buffers grow by doubling and are stream-ordered (cudaMallocAsync), so the per-iteration
// rebuild (geometry/dlmesh.py:50, dmtet.py:202) never synchronises the host or touches the allocator
// in steady state.
#pragma once
#include "bvh_traverse.cuh"

#define MCS_SKIP_TABLES 4
#define MCS_COUNTER_RING 64

// Freed with its context.  cudaFree (not cudaFreeAsync: no stream is known at destruction) also releases cudaMallocAsync memory;
// OptiXContext.__del__ synchronises the device before it destroys the context.
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
};

struct mcs_ctx {
    int device = 0;
    int T = 0, V = 0;            // triangles / vertices of the current structure (0 = none built)
    // ---- binary LBVH (canonical, exported for parity tests) ----
    DevBuf bounds;               // 12 x uint32 order-preserving encoded: cmin, cmax, smin, smax
    DevBuf tlo, thi;             // [T][3] raw triangle boxes
    DevBuf keys, keys_alt;       // [T] Morton codes (unsorted / sorted)
    DevBuf vals, vals_alt;       // [T] triangle ids   (unsorted / sorted)
    DevBuf left, right, parent;  // [T-1],[T-1],[2T-1]
    DevBuf lo, hi;               // [2T-1][3] padded node boxes
    DevBuf flags;                // [T-1] refit arrival counters
    DevBuf range;                // [T-1] int2: sorted-triangle range of each internal node
    DevBuf sort_tmp;
    // ---- traversal layout ----
    DevBuf nodes;                // [max(T-1,1)] x 4 float4 (two child boxes + child codes)
    DevBuf tris;                 // [T] x 3 float4 in SORTED order: (v0, orig id), (e1, -), (e2, -)
    DevBuf nodesq4;              // [max(T-1,1)] x 4 uint4: 4-wide quantised view, 16-bit boxes on a scene-wide grid (see `shadow`)
    DevBuf qgrid;                // 9 floats: grid origin xyz, cell size xyz, 1 / cell size xyz
    // ---- the shadow-ray view's own SAH topology (bvh.cu:k_ploc; MCS_LEAF_MAX < T <= MCS_SAH_MAX_TRIS) ----
    DevBuf sleft, sright, scnt;  // [T-1] children, triangle counts (negative: leaf run)
    DevBuf sbox;                 // [T-1] x 2 float4 node boxes
    DevBuf sfirst;               // [2T-1] first slot of each node's triangles in depth-first leaf order
    DevBuf cbox, cid;            // k_ploc scratch: [2][T][2] float4 cluster boxes, [2][T] cluster ids (two buffers, swapped every round)
    DevBuf nn, round_id;         // k_ploc scratch: [T] nearest neighbour, [T] next free node id before each round
    DevBuf stris;                // [T] x 3 float4: the triangle records of `tris` in depth-first leaf order
    // What env_shade's shadow rays walk, set by every mcs_bvh_build: nodesq4, qgrid, and the triangle records its leaf runs index
    // (stris for the SAH topology, tris for the LBVH grandchild collapse).  nodes is null: the fp32 nodes belong to the LBVH view.
    BvhView shadow = {};
    // ---- env_shade support ----
    DevBuf lcg_skip[MCS_SKIP_TABLES];   // [5*N*N+3] x uint2 (mul, add) LCG jump-ahead tables, one per cached n_samples_x
    int skip_N[MCS_SKIP_TABLES] = {0, 0, 0, 0};
    int n_skip = 0;
    unsigned skip_evict = 0;
    DevBuf counters;             // ring of 64-byte slots: per-launch work-claim counters of the persistent env_shade grid
    unsigned counter_next = 0;
    DevBuf mtx_inv;              // [B,4,4] inverse clip matrices of the last mcs_rasterize call
};

int mcs_buf_reserve(DevBuf &b, size_t bytes, cudaStream_t s);
