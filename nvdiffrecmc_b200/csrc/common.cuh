// common.cuh -- shared host/device helpers for libmcshade (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/mcshade.h"

// ---------------------------------------------------------------------------------------------
// Error handling: every failure is recorded and returned (the reference drops CUDA/OptiX errors,
// render/optixutils/c_src/common.h:37-61).
// ---------------------------------------------------------------------------------------------
void mcs_set_error(const char *fmt, ...);

#define MCS_CUDA(call)                                                                         \
    do {                                                                                       \
        cudaError_t e_ = (call);                                                               \
        if (e_ != cudaSuccess) {                                                               \
            mcs_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            return 2;                                                                          \
        }                                                                                      \
    } while (0)

#define MCS_REQUIRE(cond, ...)                                                                 \
    do {                                                                                       \
        if (!(cond)) { mcs_set_error(__VA_ARGS__); return 1; }                                 \
    } while (0)

#define MCS_LAUNCH_CHECK() MCS_CUDA(cudaGetLastError())

// ---------------------------------------------------------------------------------------------
// float3 math (fast path: FMA contraction allowed)
// ---------------------------------------------------------------------------------------------
struct f3 { float x, y, z; };
__host__ __device__ __forceinline__ f3 F3(float x, float y, float z) { f3 r; r.x = x; r.y = y; r.z = z; return r; }
__host__ __device__ __forceinline__ f3 F3(float a) { return F3(a, a, a); }
__host__ __device__ __forceinline__ f3 operator+(f3 a, f3 b) { return F3(a.x + b.x, a.y + b.y, a.z + b.z); }
__host__ __device__ __forceinline__ f3 operator-(f3 a, f3 b) { return F3(a.x - b.x, a.y - b.y, a.z - b.z); }
__host__ __device__ __forceinline__ f3 operator*(f3 a, f3 b) { return F3(a.x * b.x, a.y * b.y, a.z * b.z); }
__host__ __device__ __forceinline__ f3 operator*(f3 a, float s) { return F3(a.x * s, a.y * s, a.z * s); }
__host__ __device__ __forceinline__ f3 operator*(float s, f3 a) { return F3(a.x * s, a.y * s, a.z * s); }
__host__ __device__ __forceinline__ f3 operator-(f3 a) { return F3(-a.x, -a.y, -a.z); }
__host__ __device__ __forceinline__ f3 &operator+=(f3 &a, f3 b) { a.x += b.x; a.y += b.y; a.z += b.z; return a; }
__host__ __device__ __forceinline__ f3 &operator-=(f3 &a, f3 b) { a.x -= b.x; a.y -= b.y; a.z -= b.z; return a; }
__host__ __device__ __forceinline__ float sum(f3 a) { return a.x + a.y + a.z; }
__host__ __device__ __forceinline__ float dot(f3 a, f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__host__ __device__ __forceinline__ f3 cross(f3 a, f3 b) { return F3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(hi, fmaxf(lo, x)); }

// ---------------------------------------------------------------------------------------------
// Warp-grouped atomics: lanes of a warp whose values go to the same addresses sum them first, and
// one lane issues the atomics for the group.  The group is peers = __match_any_sync(0xFFFFFFFF, key):
// every lane of the warp must reach that match (no early exit before it), and a lane with nothing
// to scatter passes a key no live lane can have, so that it groups with no one and then leaves.
// The live lanes of a group call warp_group_sum together: it sums v over the group in lane order
// (shuffles) and returns true in the lane that issues the atomics, the lowest of the group.  A lane
// alone in its group keeps its values and returns true.
// ---------------------------------------------------------------------------------------------
template <int N>
__device__ __forceinline__ bool warp_group_sum(unsigned peers, float (&v)[N])
{
    const unsigned lane = threadIdx.x & 31u;
    if (peers == (1u << lane)) return true;
    float s[N];
#pragma unroll
    for (int k = 0; k < N; ++k) s[k] = 0.0f;
    for (unsigned m = peers; m; m &= m - 1) {
        const int src = __ffs(m) - 1;
#pragma unroll
        for (int k = 0; k < N; ++k) s[k] += __shfl_sync(peers, v[k], src);
    }
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = s[k];
    return (int)lane == __ffs(peers) - 1;
}

// ---------------------------------------------------------------------------------------------
// Strided NHWC accessor built from mcs_tensor (size-1 dims broadcast => stride 0)
// ---------------------------------------------------------------------------------------------
struct TView {
    const float *p;
    int s0, s1, s2, s3;   // element strides, 0 for broadcast dims
    int n0, n1, n2, n3;
    __device__ __forceinline__ int64_t off(int n, int h, int w) const { return (int64_t)n * s0 + (int64_t)h * s1 + (int64_t)w * s2; }
    __device__ __forceinline__ float ld1(int n, int h, int w) const { return __ldg(p + off(n, h, w)); }
    __device__ __forceinline__ f3 ld3(int n, int h, int w) const
    {
        const float *q = p + off(n, h, w);
        if (n3 == 1) { float v = __ldg(q); return F3(v, v, v); }   // channel broadcast (common.h:17-19)
        return F3(__ldg(q), __ldg(q + s3), __ldg(q + 2 * s3));
    }
};

static inline TView make_view(const mcs_tensor *t)
{
    TView v;
    v.p = (const float *)t->ptr;
    v.n0 = t->sizes[0]; v.n1 = t->sizes[1]; v.n2 = t->sizes[2]; v.n3 = t->sizes[3];
    v.s0 = t->sizes[0] == 1 ? 0 : t->strides[0];
    v.s1 = t->sizes[1] == 1 ? 0 : t->strides[1];
    v.s2 = t->sizes[2] == 1 ? 0 : t->strides[2];
    v.s3 = t->sizes[3] == 1 ? 0 : t->strides[3];
    return v;
}

static inline bool view_ok(const mcs_tensor *t) { return t && t->ptr && t->sizes[0] > 0 && t->sizes[1] > 0 && t->sizes[2] > 0 && t->sizes[3] > 0; }
