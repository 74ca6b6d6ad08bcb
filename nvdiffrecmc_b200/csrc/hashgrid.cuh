// hashgrid.cuh -- the per-point encoding math of the multiresolution hash grid (contract in hashgrid.cu), shared by the bare encoding's
// kernels (hashgrid.cu) and the fused MLP texture (mlptexture.cu).
#pragma once
#include "common.cuh"

namespace {

// cell of x at level l: corner base g (uint32), fractions t
struct Cell { uint32_t g[3]; float t[3]; };

__device__ __forceinline__ Cell hg_cell(const float s, const float x[3])
{
    Cell c;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float p = fmaf(s, x[d], 0.5f);
        c.g[d] = (uint32_t)__float2int_rd(p);           // cvt.rmi.s32.f32
        c.t[d] = __fsub_rn(p, floorf(p));
    }
    return c;
}

__device__ __forceinline__ uint32_t hg_index(const Cell &cl, int c, bool dense, uint32_t res, uint32_t size)
{
    const uint32_t cx = cl.g[0] + (c & 1), cy = cl.g[1] + ((c >> 1) & 1), cz = cl.g[2] + ((c >> 2) & 1);
    const uint32_t h = dense ? cx + cy * res + cz * (res * res) : (cx ^ (cy * 2654435761u) ^ (cz * 805459861u));
    return (size & (size - 1)) == 0 ? (h & (size - 1)) : h % size;
}

__device__ __forceinline__ void hg_weights(const Cell &cl, int c, float w1[3])
{
#pragma unroll
    for (int d = 0; d < 3; ++d) w1[d] = ((c >> d) & 1) ? cl.t[d] : __fsub_rn(1.0f, cl.t[d]);
}

// d params of one corner, one vector atomic (red.global.add.v2.f32) for both features.  With `agg`, lanes of the warp that scatter into
// the same entry are grouped (warp_group_sum); every lane of the warp must then call this (live = false for a lane without a gradient).
__device__ __forceinline__ void hg_scatter(float2 *base, uint32_t idx, float2 g, bool live, bool agg)
{
    if (agg) {
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, live ? (uint64_t)idx : (1ull << 32) + (threadIdx.x & 31u));
        if (!live) return;
        float v[2] = {g.x, g.y};
        if (warp_group_sum(peers, v)) atomicAdd(base + idx, make_float2(v[0], v[1]));
    } else if (live) {
        atomicAdd(base + idx, g);
    }
}

}  // namespace
