// texture.cu -- filtered, mip-mapped texture sampling: the stand-in for nvdiffrast's `dr.texture` in the modes the reference calls
// (render/texture.py:27-30,57-68 `Texture2D.sample` and the mip chain's backward, render/render.py:54,75-95 the jittered regulariser taps,
// render/light.py:64,76): filter 'linear' / 'linear-mipmap-linear', boundary 'wrap' / 'clamp', fp32, any C >= 1.
// Semantics (the contract; the CPU oracle oracle/texture.c restates it):
//
// Levels k = 0..L (L <= 15), level k of W_k x H_k texels, [Bt, H_k, W_k, C]; a level with minibatch stride 0 is shared by every pixel
// batch.  'linear' reads level 0 only.  fl() is one IEEE round-to-nearest operation; sums and products are evaluated left to right.
// Bilinear sample S_k(u, v), per channel:
//   x = fl(fl(u * (float)W_k) - 0.5), x0 = cvt.rmi.s32(x) (floor, saturating, NaN -> 0), fx = fl(x - floorf(x)); y0, fy from v, H_k alike;
//   taps (x0, x0+1) x (y0, y0+1): wrap takes each index mod the size into [0, size), clamp clamps it to [0, size - 1] (the +1 never
//   overflows: it is formed after the reduction), so every access is in bounds for every input; values for non-finite uv are unspecified;
//   ox = 1 - fx, oy = 1 - fy, t_ij = texel (x0 + i, y0 + j):  S = oy * (ox * t00 + fx * t10) + fy * (ox * t01 + fx * t11).
// Level of detail ('linear-mipmap-linear'), uv_da = (du/dX, du/dY, dv/dX, dv/dY) per pixel:
//   a = du/dX * W_0, b = du/dY * W_0, c = dv/dX * H_0, d = dv/dY * H_0  (W_0, H_0 as float);
//   A = a*a + c*c, B = b*b + d*d, C = a*b + c*d, h = (A - B) * 0.5, D = h*h + C*C, q = sqrtf(D), M = (A + B) * 0.5 + q
//   (M = the larger eigenvalue of J^T J, the squared major axis of the pixel footprint in texels);
//   lam_raw = 0.5 * det_log2(M); lam = fminf(fmaxf(lam_raw, 0), L) (NaN -> 0; M = 0 gives -inf -> 0);
//   l0 = (int)floorf(lam), f = lam - l0, l1 = min(l0 + 1, L);  out = S_l0 when f == 0 (level l1 is not read), else
//   out = (1 - f) * S_l0 + f * S_l1.
// det_log2(M) (fixed algorithm, as the transcendentals of exact.cuh): 0 -> -inf, +inf -> +inf, NaN or < 0 -> NaN; otherwise M = m 2^e with
//   m in [0.5, 1) (subnormals are first scaled by 2^23, exactly); if m < sqrt(1/2): e -= 1, z = (m + m) - 1, else z = m - 1; zz = z * z;
//   p = P0, p = p * z + P_i for i = 1..8 (Cephes' single-precision logf minimax coefficients); y = (p * z) * zz; y = y - 0.5 * zz;
//   r = y * LOG2EA; r = r + z * LOG2EA; r = r + y; r = r + z; r = r + (float)e   (LOG2EA = log2(e) - 1).
// Adjoints (g = d out):
//   d tex: for each level used, tap t_ij of that level += (w_lvl * w_ij) * g_c, w_lvl = 1 ('linear', or f == 0), 1 - f for l0, f for l1,
//     w_00 = oy*ox, w_10 = oy*fx, w_01 = fy*ox, w_11 = fy*fx.  Float atomics: the only order-dependent result.  A group of channels whose
//     upstream gradients are all exactly zero issues no atomics (background pixels of a masked loss), and neither does level l1 when f == 0.
//   d uv: per level used, su = sum over c ascending, from 0, of g_c * (oy * (t10 - t00) + fy * (t11 - t01)) and
//     sv = sum of g_c * (ox * (t01 - t00) + fx * (t11 - t10)); d u = w_l0 * (W_l0 * su_l0) [+ w_l1 * (W_l1 * su_l1) when f != 0],
//     d v the same with sv and H_k.
//   d uv_da: zero unless 'linear-mipmap-linear', 0 < lam_raw < L and f != 0.  Then gl = sum over c ascending of g_c * (S_l1 - S_l0),
//     gM = gl / (M * 1.38629436f) (d lam / dM = 1 / (2 M ln 2)); if q > 0: r = h / q, e = C / q, gA = gM * (0.5 + 0.5 * r),
//     gB = gM * (0.5 - 0.5 * r), gC = gM * e; if q == 0 the sqrt(D) term contributes no gradient (a non-differentiable point; the
//     project's choice): gA = gB = gM * 0.5, gC = 0.  ga = (a + a) * gA + b * gC, gb = (b + b) * gB + a * gC, gc = (c + c) * gA + d * gC,
//     gd = (d + d) * gB + c * gC;  d uv_da = (ga * W_0, gb * W_0, gc * H_0, gd * H_0).
// Every operation above is explicitly rounded (__fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn / __fsqrt_rn, never contracted), so the
// forward, d uv and d uv_da are bit-reproducible against the fp32 oracle.  No hardware texture filtering: its 8-bit fixed-point weights
// would break the contract.
#include "common.cuh"

// Layout choices, measured with tools/texbench.py on bench.py's shape (8 x 512^2, Texture2D.sample x 3 on 1024^2 chains and the five
// regulariser taps; one H100 80GB HBM3 at a 400 W power limit, DESIGN.md section 4): a warp covers an 8 x 4 pixel tile (backward of the
// three samples 2.77-2.82 ms against 2.88-3.28 ms for a row of 32 pixels); d tex issues plain vector reductions (1.36-1.46 ms) --
// grouping the lanes that hit one texel with __match_any_sync costs more than it saves here (2.77-2.82 ms; taps 1.96-1.99 ms against
// 1.31-1.37 ms).

namespace {

struct TexArgs {
    mcs_texture_levels lv;      // by value: no per-call upload, capturable in a CUDA graph
    float *grad[16];            // d tex per level (null: not wanted)
    const float *uv, *uv_da, *dy;
    float *out, *duv, *duv_da;
    int32_t B, H, W, mip, clamp, want_tex;
};

__device__ __forceinline__ float tex_log2(float x)
{
    if (!(x > 0.0f)) return x == 0.0f ? -INFINITY : NAN;
    if (x == INFINITY) return x;
    int e = 0;
    if (x < 1.17549435e-38f) { x = __fmul_rn(x, 8388608.0f); e = -23; }
    const uint32_t bits = __float_as_uint(x);
    e += (int)((bits >> 23) & 0xffu) - 126;
    const float m = __uint_as_float((bits & 0x7fffffu) | 0x3f000000u);
    float z;
    if (m < 0.707106781186547524f) { e -= 1; z = __fsub_rn(__fadd_rn(m, m), 1.0f); } else { z = __fsub_rn(m, 1.0f); }
    const float zz = __fmul_rn(z, z);
    float p = 7.0376836292e-2f;
    p = __fadd_rn(__fmul_rn(p, z), -1.1514610310e-1f);
    p = __fadd_rn(__fmul_rn(p, z), 1.1676998740e-1f);
    p = __fadd_rn(__fmul_rn(p, z), -1.2420140846e-1f);
    p = __fadd_rn(__fmul_rn(p, z), 1.4249322787e-1f);
    p = __fadd_rn(__fmul_rn(p, z), -1.6668057665e-1f);
    p = __fadd_rn(__fmul_rn(p, z), 2.0000714765e-1f);
    p = __fadd_rn(__fmul_rn(p, z), -2.4999993993e-1f);
    p = __fadd_rn(__fmul_rn(p, z), 3.3333331174e-1f);
    float y = __fmul_rn(__fmul_rn(p, z), zz);
    y = __fsub_rn(y, __fmul_rn(0.5f, zz));
    const float L2EA = 0.44269504088896340736f;
    float r = __fmul_rn(y, L2EA);
    r = __fadd_rn(r, __fmul_rn(z, L2EA));
    r = __fadd_rn(r, y);
    r = __fadd_rn(r, z);
    return __fadd_rn(r, (float)e);
}

// level of detail of one pixel: levels l0 / l1, blend f, and what d uv_da needs
struct Lod { int l0, l1; float f, lam_raw, a, b, c, d, A, B, C, h, q, M; };

__device__ __forceinline__ Lod tex_lod(const float4 da, float W0, float H0, int L)
{
    Lod o;
    o.a = __fmul_rn(da.x, W0); o.b = __fmul_rn(da.y, W0); o.c = __fmul_rn(da.z, H0); o.d = __fmul_rn(da.w, H0);
    o.A = __fadd_rn(__fmul_rn(o.a, o.a), __fmul_rn(o.c, o.c));
    o.B = __fadd_rn(__fmul_rn(o.b, o.b), __fmul_rn(o.d, o.d));
    o.C = __fadd_rn(__fmul_rn(o.a, o.b), __fmul_rn(o.c, o.d));
    o.h = __fmul_rn(__fsub_rn(o.A, o.B), 0.5f);
    o.q = __fsqrt_rn(__fadd_rn(__fmul_rn(o.h, o.h), __fmul_rn(o.C, o.C)));
    o.M = __fadd_rn(__fmul_rn(__fadd_rn(o.A, o.B), 0.5f), o.q);
    o.lam_raw = __fmul_rn(0.5f, tex_log2(o.M));
    const float lam = fminf(fmaxf(o.lam_raw, 0.0f), (float)L);
    const float fl = floorf(lam);
    o.l0 = (int)fl;
    o.f = __fsub_rn(lam, fl);
    o.l1 = min(o.l0 + 1, L);
    return o;
}

// the four taps of one level: element offsets of t00, t10, t01, t11 (texel * C + minibatch offset) and the bilinear fractions
struct Taps { int64_t o00, o10, o01, o11; float fx, fy; };

__device__ __forceinline__ void tex_axis(float u, int n, bool clamp, int &i0, int &i1, float &fr)
{
    const float x = __fsub_rn(__fmul_rn(u, (float)n), 0.5f);
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

__device__ __forceinline__ Taps tex_taps(const mcs_texture_levels &lv, int k, int b, float u, float v, bool clamp)
{
    const int W = lv.w[k], H = lv.h[k], C = lv.C;
    int x0, x1, y0, y1;
    Taps t;
    tex_axis(u, W, clamp, x0, x1, t.fx);
    tex_axis(v, H, clamp, y0, y1, t.fy);
    const int64_t base = (int64_t)b * lv.batch_stride[k];          // elements; stride 0 shares the level over the minibatch
    const int64_t r0 = (int64_t)y0 * W, r1 = (int64_t)y1 * W;      // texels
    t.o00 = base + (r0 + x0) * C; t.o10 = base + (r0 + x1) * C; t.o01 = base + (r1 + x0) * C; t.o11 = base + (r1 + x1) * C;
    return t;
}

template <int VEC> struct Vec { float v[VEC]; };

template <int VEC>
__device__ __forceinline__ Vec<VEC> ld(const float *p)
{
    Vec<VEC> r;
    if (VEC == 4) { const float4 q = __ldg((const float4 *)p); r.v[0] = q.x; r.v[1] = q.y; r.v[2] = q.z; r.v[3] = q.w; }
    else if (VEC == 2) { const float2 q = __ldg((const float2 *)p); r.v[0] = q.x; r.v[1] = q.y; }
    else r.v[0] = __ldg(p);
    return r;
}

template <int VEC>
__device__ __forceinline__ void st(float *p, const Vec<VEC> &r)
{
    if (VEC == 4) *(float4 *)p = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);
    else if (VEC == 2) *(float2 *)p = make_float2(r.v[0], r.v[1]);
    else *p = r.v[0];
}

// the four texels of one channel group
template <int VEC> struct Quad { Vec<VEC> t00, t10, t01, t11; };

template <int VEC>
__device__ __forceinline__ Quad<VEC> ld_quad(const float *p, const Taps &t, int cg)
{
    Quad<VEC> q;
    q.t00 = ld<VEC>(p + t.o00 + cg); q.t10 = ld<VEC>(p + t.o10 + cg); q.t01 = ld<VEC>(p + t.o01 + cg); q.t11 = ld<VEC>(p + t.o11 + cg);
    return q;
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

template <int VEC>
__device__ __forceinline__ void scatter_level(float *grad, const Taps &t, int cg, float wl, const Vec<VEC> &g, bool live)
{
    const float ox = __fsub_rn(1.0f, t.fx), oy = __fsub_rn(1.0f, t.fy);
    const float w[4] = {__fmul_rn(wl, __fmul_rn(oy, ox)), __fmul_rn(wl, __fmul_rn(oy, t.fx)), __fmul_rn(wl, __fmul_rn(t.fy, ox)),
                        __fmul_rn(wl, __fmul_rn(t.fy, t.fx))};
    const int64_t o[4] = {t.o00, t.o10, t.o01, t.o11};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        Vec<VEC> s;
#pragma unroll
        for (int i = 0; i < VEC; ++i) s.v[i] = __fmul_rn(w[j], g.v[i]);
        scatter<VEC>(grad, o[j] + cg, s, live);
    }
}

// pixel of this thread: an 8 x 4 tile per warp
__device__ __forceinline__ bool tex_pixel(const TexArgs &a, int &b, int &y, int &x, int64_t &pix)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t tx = (a.W + 7) / 8, ty = (a.H + 3) / 4, per = tx * ty;
    const int64_t w = i >> 5, lane = i & 31;
    b = (int)(w / per);
    const int64_t t = w - (int64_t)b * per;
    y = (int)(t / tx) * 4 + (int)(lane >> 3);
    x = (int)(t % tx) * 8 + (int)(lane & 7);
    const bool in = b < a.B && y < a.H && x < a.W;
    pix = ((int64_t)b * a.H + y) * a.W + x;
    return in;
}

template <int VEC>
__global__ void __launch_bounds__(256) k_texture_fwd(const TexArgs a)
{
    int b, y, x;
    int64_t pix;
    if (!tex_pixel(a, b, y, x, pix)) return;
    const mcs_texture_levels &lv = a.lv;
    const float2 uv = __ldg((const float2 *)a.uv + pix);
    int l0 = 0, l1 = 0;
    float f = 0.0f;
    if (a.mip) {
        const Lod d = tex_lod(__ldg((const float4 *)a.uv_da + pix), (float)lv.w[0], (float)lv.h[0], lv.n_levels - 1);
        l0 = d.l0; l1 = d.l1; f = d.f;
    }
    const Taps t0 = tex_taps(lv, l0, b, uv.x, uv.y, a.clamp);
    const Taps t1 = tex_taps(lv, l1, b, uv.x, uv.y, a.clamp);
    const float of = __fsub_rn(1.0f, f);
    const int C = lv.C;
    float *out = a.out + pix * C;
    for (int cg = 0; cg < C; cg += VEC) {
        const Quad<VEC> q0 = ld_quad<VEC>(lv.ptr[l0], t0, cg);
        Vec<VEC> r;
#pragma unroll
        for (int j = 0; j < VEC; ++j) r.v[j] = bilerp(q0.t00.v[j], q0.t10.v[j], q0.t01.v[j], q0.t11.v[j], t0.fx, t0.fy);
        if (f != 0.0f) {
            const Quad<VEC> q1 = ld_quad<VEC>(lv.ptr[l1], t1, cg);
#pragma unroll
            for (int j = 0; j < VEC; ++j)
                r.v[j] = __fadd_rn(__fmul_rn(of, r.v[j]), __fmul_rn(f, bilerp(q1.t00.v[j], q1.t10.v[j], q1.t01.v[j], q1.t11.v[j], t1.fx, t1.fy)));
        }
        st<VEC>(out + cg, r);
    }
}

// d uv partial sums of one level and channel group (channels ascending)
template <int VEC>
__device__ __forceinline__ void duv_level(const Quad<VEC> &q, const Taps &t, const Vec<VEC> &g, float &su, float &sv)
{
    const float ox = __fsub_rn(1.0f, t.fx), oy = __fsub_rn(1.0f, t.fy);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
        const float du = __fadd_rn(__fmul_rn(oy, __fsub_rn(q.t10.v[j], q.t00.v[j])), __fmul_rn(t.fy, __fsub_rn(q.t11.v[j], q.t01.v[j])));
        const float dv = __fadd_rn(__fmul_rn(ox, __fsub_rn(q.t01.v[j], q.t00.v[j])), __fmul_rn(t.fx, __fsub_rn(q.t11.v[j], q.t10.v[j])));
        su = __fadd_rn(su, __fmul_rn(g.v[j], du));
        sv = __fadd_rn(sv, __fmul_rn(g.v[j], dv));
    }
}

// One fused backward launch: d tex (float atomics into per-level buffers), d uv and d uv_da (one writer per pixel).
template <int VEC>
__global__ void __launch_bounds__(256) k_texture_bwd(const TexArgs a)
{
    int b, y, x;
    int64_t pix;
    const bool in = tex_pixel(a, b, y, x, pix);
    const int64_t p = in ? pix : 0;
    const mcs_texture_levels &lv = a.lv;
    const int tb = in ? b : 0;
    const float2 uv = in ? __ldg((const float2 *)a.uv + p) : make_float2(0.0f, 0.0f);
    const int L = lv.n_levels - 1;
    Lod d{};
    d.l0 = d.l1 = 0;
    if (a.mip && in) d = tex_lod(__ldg((const float4 *)a.uv_da + p), (float)lv.w[0], (float)lv.h[0], L);
    const float f = a.mip ? d.f : 0.0f;
    const Taps t0 = tex_taps(lv, d.l0, tb, uv.x, uv.y, a.clamp);
    const Taps t1 = tex_taps(lv, d.l1, tb, uv.x, uv.y, a.clamp);
    const float w0 = __fsub_rn(1.0f, f);
    const bool two = f != 0.0f;
    const bool want_da = a.duv_da != nullptr && a.mip && d.lam_raw > 0.0f && d.lam_raw < (float)L && two;
    const bool read = in && (a.duv != nullptr || want_da);
    float *g0 = a.grad[d.l0], *g1 = a.grad[d.l1];
    const int C = lv.C;
    float su0 = 0.0f, sv0 = 0.0f, su1 = 0.0f, sv1 = 0.0f, gl = 0.0f;
    for (int cg = 0; cg < C; cg += VEC) {
        Vec<VEC> g;
        bool live = false;
        if (in) {
            g = ld<VEC>(a.dy + p * C + cg);
#pragma unroll
            for (int j = 0; j < VEC; ++j) live |= g.v[j] != 0.0f;
        } else {
#pragma unroll
            for (int j = 0; j < VEC; ++j) g.v[j] = 0.0f;
        }
        if (read) {
            const Quad<VEC> q0 = ld_quad<VEC>(lv.ptr[d.l0], t0, cg);
            if (a.duv) duv_level<VEC>(q0, t0, g, su0, sv0);
            if (two) {
                const Quad<VEC> q1 = ld_quad<VEC>(lv.ptr[d.l1], t1, cg);
                if (a.duv) duv_level<VEC>(q1, t1, g, su1, sv1);
                if (want_da) {
#pragma unroll
                    for (int j = 0; j < VEC; ++j) {
                        const float s0 = bilerp(q0.t00.v[j], q0.t10.v[j], q0.t01.v[j], q0.t11.v[j], t0.fx, t0.fy);
                        const float s1 = bilerp(q1.t00.v[j], q1.t10.v[j], q1.t01.v[j], q1.t11.v[j], t1.fx, t1.fy);
                        gl = __fadd_rn(gl, __fmul_rn(g.v[j], __fsub_rn(s1, s0)));
                    }
                }
            }
        }
        if (a.want_tex) {
            scatter_level<VEC>(g0, t0, cg, w0, g, live && g0 != nullptr);
            if (a.mip) scatter_level<VEC>(g1, t1, cg, f, g, live && two && g1 != nullptr);
        }
    }
    if (!in) return;
    if (a.duv) {
        float du = __fmul_rn(w0, __fmul_rn((float)lv.w[d.l0], su0)), dv = __fmul_rn(w0, __fmul_rn((float)lv.h[d.l0], sv0));
        if (two) {
            du = __fadd_rn(du, __fmul_rn(f, __fmul_rn((float)lv.w[d.l1], su1)));
            dv = __fadd_rn(dv, __fmul_rn(f, __fmul_rn((float)lv.h[d.l1], sv1)));
        }
        ((float2 *)a.duv)[p] = make_float2(du, dv);
    }
    if (a.duv_da) {
        float4 r = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (want_da) {
            const float gM = __fdiv_rn(gl, __fmul_rn(d.M, 1.38629436f));
            float gA, gB, gC;
            if (d.q > 0.0f) {
                const float rr = __fdiv_rn(d.h, d.q), e = __fdiv_rn(d.C, d.q);
                gA = __fmul_rn(gM, __fadd_rn(0.5f, __fmul_rn(0.5f, rr)));
                gB = __fmul_rn(gM, __fsub_rn(0.5f, __fmul_rn(0.5f, rr)));
                gC = __fmul_rn(gM, e);
            } else {
                gA = gB = __fmul_rn(gM, 0.5f);
                gC = 0.0f;
            }
            const float ga = __fadd_rn(__fmul_rn(__fadd_rn(d.a, d.a), gA), __fmul_rn(d.b, gC));
            const float gb = __fadd_rn(__fmul_rn(__fadd_rn(d.b, d.b), gB), __fmul_rn(d.a, gC));
            const float gc = __fadd_rn(__fmul_rn(__fadd_rn(d.c, d.c), gA), __fmul_rn(d.d, gC));
            const float gd = __fadd_rn(__fmul_rn(__fadd_rn(d.d, d.d), gB), __fmul_rn(d.c, gC));
            const float W0 = (float)lv.w[0], H0 = (float)lv.h[0];
            r = make_float4(__fmul_rn(ga, W0), __fmul_rn(gb, W0), __fmul_rn(gc, H0), __fmul_rn(gd, H0));
        }
        ((float4 *)a.duv_da)[p] = r;
    }
}

int tex_validate(const char *fn, const mcs_texture_levels *lv, const float *uv, const float *uv_da, int32_t B, int32_t H, int32_t W,
                 int32_t filter_mode, int32_t boundary_mode)
{
    MCS_REQUIRE(lv && uv, "%s: null pointer", fn);
    MCS_REQUIRE(filter_mode == MCS_TEX_LINEAR || filter_mode == MCS_TEX_LINEAR_MIPMAP_LINEAR, "%s: unknown filter_mode %d", fn, filter_mode);
    MCS_REQUIRE(boundary_mode == MCS_TEX_WRAP || boundary_mode == MCS_TEX_CLAMP, "%s: unknown boundary_mode %d", fn, boundary_mode);
    MCS_REQUIRE(filter_mode == MCS_TEX_LINEAR || uv_da, "%s: null pointer (uv_da is required with linear-mipmap-linear)", fn);
    MCS_REQUIRE(B >= 0 && H >= 0 && W >= 0, "%s: B, H, W must be >= 0 (got %d, %d, %d)", fn, B, H, W);
    MCS_REQUIRE((int64_t)B * H * W <= (int64_t)INT32_MAX * 64, "%s: too many pixels", fn);
    MCS_REQUIRE(lv->n_levels >= 1 && lv->n_levels <= 16, "%s: n_levels must be in 1..16 (got %d)", fn, lv->n_levels);
    MCS_REQUIRE(lv->C >= 1, "%s: C must be >= 1 (got %d)", fn, lv->C);
    MCS_REQUIRE(((uintptr_t)uv & 7) == 0 && ((uintptr_t)uv_da & 15) == 0, "%s: uv must be 8-byte and uv_da 16-byte aligned", fn);
    for (int k = 0; k < lv->n_levels; ++k) {
        MCS_REQUIRE(lv->ptr[k] != nullptr, "%s: null pointer (level %d)", fn, k);
        MCS_REQUIRE(lv->h[k] >= 1 && lv->w[k] >= 1, "%s: level %d has size %d x %d", fn, k, lv->h[k], lv->w[k]);
        MCS_REQUIRE(k == 0 || (lv->h[k] == max(1, lv->h[0] >> k) && lv->w[k] == max(1, lv->w[0] >> k)),
                    "%s: level %d is %d x %d, expected %d x %d", fn, k, lv->h[k], lv->w[k], max(1, lv->h[0] >> k), max(1, lv->w[0] >> k));
        MCS_REQUIRE(lv->batch_stride[k] == 0 || lv->batch_stride[k] == (int64_t)lv->h[k] * lv->w[k] * lv->C,
                    "%s: level %d batch_stride must be 0 or H*W*C", fn, k);
        MCS_REQUIRE(((uintptr_t)lv->ptr[k] & 3) == 0, "%s: level %d is not 4-byte aligned", fn, k);
    }
    for (int k = 1; k < lv->n_levels; ++k)
        MCS_REQUIRE((lv->batch_stride[k] == 0) == (lv->batch_stride[0] == 0), "%s: every level must share (or not) the minibatch", fn);
    return 0;
}

bool aligned_all(const TexArgs &a, int n_levels, uintptr_t mask)
{
    bool ok = true;
    for (int k = 0; k < n_levels; ++k) ok &= (((uintptr_t)a.lv.ptr[k] | (uintptr_t)a.grad[k]) & mask) == 0;
    return ok && (((uintptr_t)a.out | (uintptr_t)a.dy) & mask) == 0;
}

int tex_launch(const TexArgs &a, cudaStream_t s, bool bwd)
{
    const int C = a.lv.C;
    const int64_t n_threads = (int64_t)a.B * ((a.W + 7) / 8) * ((a.H + 3) / 4) * 32;
    const unsigned blocks = (unsigned)((n_threads + 255) / 256);
    const int n = a.lv.n_levels;
    if (C % 4 == 0 && aligned_all(a, n, 15)) { if (bwd) k_texture_bwd<4><<<blocks, 256, 0, s>>>(a); else k_texture_fwd<4><<<blocks, 256, 0, s>>>(a); }
    else if (C % 2 == 0 && aligned_all(a, n, 7)) { if (bwd) k_texture_bwd<2><<<blocks, 256, 0, s>>>(a); else k_texture_fwd<2><<<blocks, 256, 0, s>>>(a); }
    else { if (bwd) k_texture_bwd<1><<<blocks, 256, 0, s>>>(a); else k_texture_fwd<1><<<blocks, 256, 0, s>>>(a); }
    MCS_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" {

int mcs_texture_fwd(const mcs_texture_levels *tex, const float *uv, const float *uv_da, int32_t B, int32_t H, int32_t W, int32_t filter_mode,
                    int32_t boundary_mode, float *out, mcs_stream stream)
{
    if (int e = tex_validate("mcs_texture_fwd", tex, uv, uv_da, B, H, W, filter_mode, boundary_mode)) return e;
    MCS_REQUIRE(out != nullptr, "mcs_texture_fwd: null pointer");
    if ((int64_t)B * H * W == 0) return 0;
    TexArgs a{};
    a.lv = *tex; a.uv = uv; a.uv_da = uv_da; a.out = out;
    if (filter_mode == MCS_TEX_LINEAR) a.lv.n_levels = 1;
    a.B = B; a.H = H; a.W = W; a.mip = filter_mode == MCS_TEX_LINEAR_MIPMAP_LINEAR; a.clamp = boundary_mode == MCS_TEX_CLAMP;
    return tex_launch(a, (cudaStream_t)stream, false);
}

int mcs_texture_bwd(const mcs_texture_levels *tex, const float *uv, const float *uv_da, int32_t B, int32_t H, int32_t W, int32_t filter_mode,
                    int32_t boundary_mode, const float *d_out, float *const *d_tex, float *d_uv, float *d_uv_da, mcs_stream stream)
{
    if (int e = tex_validate("mcs_texture_bwd", tex, uv, uv_da, B, H, W, filter_mode, boundary_mode)) return e;
    MCS_REQUIRE(d_out != nullptr, "mcs_texture_bwd: null pointer");
    const bool mip = filter_mode == MCS_TEX_LINEAR_MIPMAP_LINEAR;
    const int n = mip ? tex->n_levels : 1;
    bool any_tex = false;
    if (d_tex)
        for (int k = 0; k < n; ++k) any_tex |= d_tex[k] != nullptr;
    MCS_REQUIRE(any_tex || d_uv || (mip && d_uv_da), "mcs_texture_bwd: null pointer (no gradient requested)");
    MCS_REQUIRE(((uintptr_t)d_uv & 7) == 0 && ((uintptr_t)d_uv_da & 15) == 0, "mcs_texture_bwd: d_uv must be 8-byte and d_uv_da 16-byte aligned");
    if ((int64_t)B * H * W == 0) return 0;
    TexArgs a{};
    a.lv = *tex; a.lv.n_levels = n;
    for (int k = 0; k < n; ++k) {
        a.grad[k] = d_tex ? d_tex[k] : nullptr;
        MCS_REQUIRE(((uintptr_t)a.grad[k] & 3) == 0, "mcs_texture_bwd: d_tex[%d] is not 4-byte aligned", k);
    }
    a.uv = uv; a.uv_da = uv_da; a.dy = d_out; a.duv = d_uv; a.duv_da = mip ? d_uv_da : nullptr;
    a.B = B; a.H = H; a.W = W; a.mip = mip; a.clamp = boundary_mode == MCS_TEX_CLAMP; a.want_tex = any_tex;
    return tex_launch(a, (cudaStream_t)stream, true);
}

}  // extern "C"
