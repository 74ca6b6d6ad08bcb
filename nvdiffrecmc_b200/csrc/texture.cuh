// texture.cuh -- the clamped / wrapped bilinear tap of the texture contract (stated in texture.cu) and its d tex reduction, shared by the
// texture look-up and the mip chain's fold (texture.cu) and the regulariser taps (taps.cu), so every tap is the look-up's by construction.
#pragma once
#include "common.cuh"

namespace {

template <int VEC> struct Vec { float v[VEC]; };

// one axis of the taps at texel-space coordinate x (texel centres at integer + 0.5 - 0.5 = integers)
__device__ __forceinline__ void tex_axis_at(float x, int n, bool clamp, int &i0, int &i1, float &fr)
{
    fr = __fsub_rn(x, floorf(x));
    const int x0 = __float2int_rd(x);                  // cvt.rmi.s32.f32: saturating, NaN -> 0
    if (clamp) {
        i0 = min(max(x0, 0), n - 1);
        i1 = x0 >= n - 1 ? n - 1 : max(x0 + 1, 0);
    } else {
        i0 = x0 % n;
        if (i0 < 0) i0 += n;
        i1 = i0 + 1 == n ? 0 : i0 + 1;
    }
}

__device__ __forceinline__ void tex_axis(float u, int n, bool clamp, int &i0, int &i1, float &fr)
{
    tex_axis_at(__fsub_rn(__fmul_rn(u, (float)n), 0.5f), n, clamp, i0, i1, fr);
}

__device__ __forceinline__ float bilerp(float t00, float t10, float t01, float t11, float fx, float fy)
{
    const float ox = __fsub_rn(1.0f, fx), oy = __fsub_rn(1.0f, fy);
    const float top = __fadd_rn(__fmul_rn(ox, t00), __fmul_rn(fx, t10));
    const float bot = __fadd_rn(__fmul_rn(ox, t01), __fmul_rn(fx, t11));
    return __fadd_rn(__fmul_rn(oy, top), __fmul_rn(fy, bot));
}

// d tex of one tap and channel group: one vector reduction (red.global.add.v4/.v2.f32)
template <int VEC>
__device__ __forceinline__ void scatter(float *base, int64_t off, Vec<VEC> g, bool live)
{
    if (!live) return;
    float *p = base + off;
    if (VEC == 4) atomicAdd((float4 *)p, make_float4(g.v[0], g.v[1], g.v[2], g.v[3]));
    else if (VEC == 2) atomicAdd((float2 *)p, make_float2(g.v[0], g.v[1]));
    else atomicAdd(p, g.v[0]);
}

// pixel of this thread: an 8 x 4 tile per warp, tiles row-major over each image of the batch
__device__ __forceinline__ bool tex_pixel(int B, int H, int W, int &b, int &y, int &x, int64_t &pix)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t tx = (W + 7) / 8, ty = (H + 3) / 4, per = tx * ty;
    const int64_t w = i >> 5, lane = i & 31;
    b = (int)(w / per);
    const int64_t t = w - (int64_t)b * per;
    y = (int)(t / tx) * 4 + (int)(lane >> 3);
    x = (int)(t % tx) * 8 + (int)(lane & 7);
    const bool in = b < B && y < H && x < W;
    pix = ((int64_t)b * H + y) * W + x;
    return in;
}

// threads of the 8 x 4 tiling of B images of H x W
__host__ __forceinline__ int64_t tex_pixel_threads(int B, int H, int W) { return (int64_t)B * ((W + 7) / 8) * ((H + 3) / 4) * 32; }

}  // namespace
