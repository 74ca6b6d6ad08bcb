// taps.cu -- the jittered regulariser taps of the reference's shade() (render/render.py:50-97, packed with alpha at :151-153,161-163):
// kd_grad, ks_grad, normal_grad and perturbed_nrm_grad, forward and backward, one launch each way, with no host synchronisation.
// Semantics (the contract; the CPU oracle oracle/taps.c restates it):
//
// Operands are fp32 views of one B, H, W with any non-negative element strides: rast [..,4], jitter [..,2], kd [..,Ckd] (Ckd = 3 or 4),
// ks, gb_normal and perturbed_nrm (optional) [..,3]; the MLP path's kd_jitter [..,Ckd] and ks_jitter [..,3] (both or neither).  fl() is one
// IEEE round-to-nearest operation; sums are evaluated left to right, and every operation is explicitly rounded (never contracted).
//   tap(img)  = the texture look-up of texture.cu, filter 'linear', boundary 'clamp', of image b of img at uv = jitter[p]: the same
//               tex_axis / bilerp (texture.cuh), so a tap equals raster.texture of that image bit for bit.
//   mask[q]   = rast[q].w > 0 ? 1 : 0;  gw = mask[p] * tap(mask).
//   |x|'      = sign(x), with sign(0) = sign(NaN) = 0 (torch's abs backward).
//   sn(x)     = x_c / l, l = sqrtf(clamp(d, 1e-20)), d = (x0 x0 + x1 x1) + x2 x2 (util.safe_normalize; clamp passes NaN).
//   Texture path (render.py:75-78): kd_grad_c = |tap(kd)_c - kd_c| * gw (every channel of kd); ks_grad_c = (|tap(ks)_c - ks_c| * m_c) * gw,
//     m = (0, 1, 1): a multiplication, so a NaN or inf of red stays NaN as in torch.
//   MLP path (render.py:63-68): kd_grad_c = |kd_jitter_c - kd_c|;  ks_grad_c = |ks_jitter_c - ks_c| * m_c;  no gw.
//   normal_grad_c = |tap(n)_c - n_c| * gw (render.py:91-92).
//   perturbed_nrm_grad_c = (1 - sn(a)_2) * gw, a = sn(tap(p)) + sn(p), for c = 0, 1, 2 (render.py:94-97).
//   Each buffer gets alpha appended (render.py:81): kd.w when Ckd = 4, else 1.  Outputs are dense contiguous [B,H,W,Ckd+1] / [B,H,W,4].
// Adjoints (G = the upstream gradient of each buffer; rast and jitter are constants), torch's operation by operation:
//   x * y: d x = g * y.  |t - v|: g_d = g_abs * sign(t - v), d t = g_d, d v = -g_d.
//   kd / normal: g_abs = G_c * gw (texture path) or G_c (MLP path, kd).  ks: g_abs = (G_c * gw) * m_c, or G_c * m_c (MLP path).
//   perturbed: g_z = -((G_0 gw + G_1 gw) + G_2 gw) (repeat sums its copies); sn's adjoint for gy at x:
//     q_c = (x_c / l) / l, g_l = ((-gy_0 q_0) + (-gy_1 q_1)) + (-gy_2 q_2), g_d = d >= 1e-20 ? g_l / (2 l) : 0 (clamp's boundary passes,
//     NaN does not), gx_c = gy_c / l + (g_d x_c + g_d x_c);  g_a = sn'(a; (0, 0, g_z)), then d tap(p) = sn'(tap(p); g_a) and the direct
//     d p = sn'(p; g_a).
//   kd's alpha (Ckd = 4) gets the direct term (((-g_d,3 + G_kd,4) + G_ks,3) + G_n,3) [+ G_p,3].
//   A tap's gradient g_c goes to its four texels as fl(w_ij * g_c), w_00 = oy*ox, w_10 = oy*fx, w_01 = fy*ox, w_11 = fy*fx: d tex of
//     texture.cu's 'linear' look-up, term for term.
// Backward: gradients of kd, ks, gb_normal and perturbed_nrm are dense [B,H,W,4] (channel 3 of a 3-channel operand stays 0), zeroed by
// the caller; each pixel adds its direct terms (one vector reduction) and its four tap terms per tapped image (one each), the
// reductions of k_texture_bwd; a vector of zeros is skipped.  kd_jitter / ks_jitter gradients have one writer per element.
// The forward, every term and every one-writer gradient equal the fp32 oracle bit for bit; the float atomics are the only
// order-dependent result, as for raster.texture.
#include "texture.cuh"

namespace {

constexpr int TP_THREADS = 256;
constexpr float SN_EPS = 1e-20f;

struct Img {                     // one [B,H,W,C] operand
    const float *p;
    int64_t s0, s1, s2, s3;      // element strides
};

struct TapArgs {
    Img rast, jit, kd, ks, nrm, pn, kdj, ksj;
    int B, H, W, ckd, has_pn, mlp;
    float *o_kd, *o_ks, *o_n, *o_p;                          // forward outputs
    const float *g_kd, *g_ks, *g_n, *g_p;                    // upstream gradients (dense)
    float *d_kd, *d_ks, *d_n, *d_p, *d_kdj, *d_ksj;          // backward outputs
};

__device__ __forceinline__ float at(const Img &m, int b, int y, int x, int c)
{
    return __ldg(m.p + (int64_t)b * m.s0 + (int64_t)y * m.s1 + (int64_t)x * m.s2 + (int64_t)c * m.s3);
}

struct Tap { int b, x0, x1, y0, y1; float fx, fy; };

__device__ __forceinline__ float tap(const Img &m, const Tap &t, int c)
{
    return bilerp(at(m, t.b, t.y0, t.x0, c), at(m, t.b, t.y0, t.x1, c), at(m, t.b, t.y1, t.x0, c), at(m, t.b, t.y1, t.x1, c), t.fx, t.fy);
}

__device__ __forceinline__ float mask_at(const Img &r, int b, int y, int x) { return at(r, b, y, x, 3) > 0.0f ? 1.0f : 0.0f; }

__device__ __forceinline__ float sgn(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }     // 0 for +-0 and NaN

// the pixel's taps and gw
__device__ __forceinline__ Tap pixel_tap(const TapArgs &a, int b, int y, int x, float &gw)
{
    Tap t;
    t.b = b;
    tex_axis(at(a.jit, b, y, x, 0), a.W, true, t.x0, t.x1, t.fx);
    tex_axis(at(a.jit, b, y, x, 1), a.H, true, t.y0, t.y1, t.fy);
    const float mt = bilerp(mask_at(a.rast, b, t.y0, t.x0), mask_at(a.rast, b, t.y0, t.x1), mask_at(a.rast, b, t.y1, t.x0),
                            mask_at(a.rast, b, t.y1, t.x1), t.fx, t.fy);
    gw = __fmul_rn(mask_at(a.rast, b, y, x), mt);
    return t;
}

__device__ __forceinline__ float sn_len(const float x[3], float &d)
{
    d = __fadd_rn(__fadd_rn(__fmul_rn(x[0], x[0]), __fmul_rn(x[1], x[1])), __fmul_rn(x[2], x[2]));
    return __fsqrt_rn(d < SN_EPS ? SN_EPS : d);
}

__device__ __forceinline__ void sn(const float x[3], float y[3])
{
    float d;
    const float l = sn_len(x, d);
#pragma unroll
    for (int c = 0; c < 3; ++c) y[c] = __fdiv_rn(x[c], l);
}

__device__ __forceinline__ void sn_bwd(const float x[3], const float gy[3], float gx[3])
{
    float d;
    const float l = sn_len(x, d);
    float gl = 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float t = __fmul_rn(-gy[c], __fdiv_rn(__fdiv_rn(x[c], l), l));
        gl = c == 0 ? t : __fadd_rn(gl, t);
    }
    const float gd = d >= SN_EPS ? __fdiv_rn(gl, __fmul_rn(2.0f, l)) : 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float h = __fmul_rn(gd, x[c]);
        gx[c] = __fadd_rn(__fdiv_rn(gy[c], l), __fadd_rn(h, h));
    }
}

// a = sn(tap(p)) + sn(p); returns sn(a)_2
__device__ __forceinline__ float pert_z(const float tp[3], const float pv[3], float av[3])
{
    float s0[3], s1[3];
    sn(tp, s0);
    sn(pv, s1);
#pragma unroll
    for (int c = 0; c < 3; ++c) av[c] = __fadd_rn(s0[c], s1[c]);
    float d;
    return __fdiv_rn(av[2], sn_len(av, d));
}

__global__ void __launch_bounds__(TP_THREADS) k_taps_fwd(const TapArgs a)
{
    int b, y, x;
    int64_t pix;
    if (!tex_pixel(a.B, a.H, a.W, b, y, x, pix)) return;
    float gw;
    const Tap t = pixel_tap(a, b, y, x, gw);
    const int ckd = a.ckd;
    const float alpha = ckd == 4 ? at(a.kd, b, y, x, 3) : 1.0f;
    float *okd = a.o_kd + pix * (ckd + 1);
    for (int c = 0; c < ckd; ++c) {
        const float v = at(a.kd, b, y, x, c);
        okd[c] = a.mlp ? fabsf(__fsub_rn(at(a.kdj, b, y, x, c), v)) : __fmul_rn(fabsf(__fsub_rn(tap(a.kd, t, c), v)), gw);
    }
    okd[ckd] = alpha;
    float r[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float v = at(a.ks, b, y, x, c), m = c == 0 ? 0.0f : 1.0f;
        r[c] = a.mlp ? __fmul_rn(fabsf(__fsub_rn(at(a.ksj, b, y, x, c), v)), m)
                     : __fmul_rn(__fmul_rn(fabsf(__fsub_rn(tap(a.ks, t, c), v)), m), gw);
    }
    reinterpret_cast<float4 *>(a.o_ks)[pix] = make_float4(r[0], r[1], r[2], alpha);
#pragma unroll
    for (int c = 0; c < 3; ++c) r[c] = __fmul_rn(fabsf(__fsub_rn(tap(a.nrm, t, c), at(a.nrm, b, y, x, c))), gw);
    reinterpret_cast<float4 *>(a.o_n)[pix] = make_float4(r[0], r[1], r[2], alpha);
    if (a.has_pn) {
        float tp[3], pv[3], av[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) { tp[c] = tap(a.pn, t, c); pv[c] = at(a.pn, b, y, x, c); }
        const float g = __fmul_rn(__fsub_rn(1.0f, pert_z(tp, pv, av)), gw);
        reinterpret_cast<float4 *>(a.o_p)[pix] = make_float4(g, g, g, alpha);
    }
}

// the tap terms fl(w_ij * g) of one pixel into the four texels of image t.b, [B,H,W,4] dense
__device__ __forceinline__ void scatter_tap(float *grad, const TapArgs &a, const Tap &t, const Vec<4> &g)
{
    const bool live = g.v[0] != 0.0f || g.v[1] != 0.0f || g.v[2] != 0.0f || g.v[3] != 0.0f;
    if (!live) return;
    const float ox = __fsub_rn(1.0f, t.fx), oy = __fsub_rn(1.0f, t.fy);
    const float w[4] = {__fmul_rn(oy, ox), __fmul_rn(oy, t.fx), __fmul_rn(t.fy, ox), __fmul_rn(t.fy, t.fx)};
    const int ys[4] = {t.y0, t.y0, t.y1, t.y1}, xs[4] = {t.x0, t.x1, t.x0, t.x1};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        Vec<4> s;
#pragma unroll
        for (int i = 0; i < 4; ++i) s.v[i] = __fmul_rn(w[j], g.v[i]);
        scatter<4>(grad, ((((int64_t)t.b * a.H + ys[j]) * a.W) + xs[j]) * 4, s, true);
    }
}

__device__ __forceinline__ void scatter_own(float *grad, int64_t pix, const Vec<4> &g)
{
    scatter<4>(grad, pix * 4, g, g.v[0] != 0.0f || g.v[1] != 0.0f || g.v[2] != 0.0f || g.v[3] != 0.0f);
}

__global__ void __launch_bounds__(TP_THREADS) k_taps_bwd(const TapArgs a)
{
    int b, y, x;
    int64_t pix;
    if (!tex_pixel(a.B, a.H, a.W, b, y, x, pix)) return;
    float gw;
    const Tap t = pixel_tap(a, b, y, x, gw);
    const int ckd = a.ckd;
    const float *Gk = a.g_kd + pix * (ckd + 1);
    const float4 Gs = __ldg(reinterpret_cast<const float4 *>(a.g_ks) + pix), Gn = __ldg(reinterpret_cast<const float4 *>(a.g_n) + pix);
    const float4 Gp = a.has_pn ? __ldg(reinterpret_cast<const float4 *>(a.g_p) + pix) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);

    // kd
    Vec<4> dir{}, tg{};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (c == ckd) break;
        const float v = at(a.kd, b, y, x, c), G = __ldg(Gk + c);
        const float u = a.mlp ? at(a.kdj, b, y, x, c) : tap(a.kd, t, c);
        const float g = __fmul_rn(a.mlp ? G : __fmul_rn(G, gw), sgn(__fsub_rn(u, v)));
        dir.v[c] = -g;
        tg.v[c] = g;
    }
    if (ckd == 4) {
        float s = __fadd_rn(__fadd_rn(__fadd_rn(dir.v[3], __ldg(Gk + 4)), Gs.w), Gn.w);
        if (a.has_pn) s = __fadd_rn(s, Gp.w);
        dir.v[3] = s;
    }
    scatter_own(a.d_kd, pix, dir);
    if (a.mlp) {
#pragma unroll
        for (int c = 0; c < 4; ++c)
            if (c < ckd) a.d_kdj[pix * ckd + c] = tg.v[c];
    } else {
        scatter_tap(a.d_kd, a, t, tg);
    }

    // ks
    const float Gsv[3] = {Gs.x, Gs.y, Gs.z};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float v = at(a.ks, b, y, x, c), m = c == 0 ? 0.0f : 1.0f;
        const float u = a.mlp ? at(a.ksj, b, y, x, c) : tap(a.ks, t, c);
        const float g = __fmul_rn(a.mlp ? __fmul_rn(Gsv[c], m) : __fmul_rn(__fmul_rn(Gsv[c], gw), m), sgn(__fsub_rn(u, v)));
        dir.v[c] = -g;
        tg.v[c] = g;
    }
    dir.v[3] = tg.v[3] = 0.0f;
    scatter_own(a.d_ks, pix, dir);
    if (a.mlp) {
#pragma unroll
        for (int c = 0; c < 3; ++c) a.d_ksj[pix * 3 + c] = tg.v[c];
    } else {
        scatter_tap(a.d_ks, a, t, tg);
    }

    // normal
    const float Gnv[3] = {Gn.x, Gn.y, Gn.z};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float g = __fmul_rn(__fmul_rn(Gnv[c], gw), sgn(__fsub_rn(tap(a.nrm, t, c), at(a.nrm, b, y, x, c))));
        dir.v[c] = -g;
        tg.v[c] = g;
    }
    scatter_own(a.d_n, pix, dir);
    scatter_tap(a.d_n, a, t, tg);

    // perturbed normal
    if (a.has_pn) {
        float tp[3], pv[3], av[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) { tp[c] = tap(a.pn, t, c); pv[c] = at(a.pn, b, y, x, c); }
        pert_z(tp, pv, av);
        const float gz = -__fadd_rn(__fadd_rn(__fmul_rn(Gp.x, gw), __fmul_rn(Gp.y, gw)), __fmul_rn(Gp.z, gw));
        const float gy[3] = {0.0f, 0.0f, gz};
        float ga[3], gt[3], gd[3];
        sn_bwd(av, gy, ga);
        sn_bwd(tp, ga, gt);
        sn_bwd(pv, ga, gd);
#pragma unroll
        for (int c = 0; c < 3; ++c) { dir.v[c] = gd[c]; tg.v[c] = gt[c]; }
        scatter_own(a.d_p, pix, dir);
        scatter_tap(a.d_p, a, t, tg);
    }
}

// Checks one operand view (null when optional and absent) and fills its Img.
int view(const char *fn, const char *name, const mcs_tensor *v, int C, const int32_t *bhw, Img &o)
{
    MCS_REQUIRE(v && v->ptr, "%s: %s is null", fn, name);
    MCS_REQUIRE(v->sizes[3] == C, "%s: %s must have %d channels, got %d", fn, name, C, v->sizes[3]);
    for (int d = 0; d < 3; ++d) MCS_REQUIRE(v->sizes[d] == bhw[d], "%s: %s must have the B, H, W of rast", fn, name);
    for (int d = 0; d < 4; ++d) MCS_REQUIRE(v->strides[d] >= 0, "%s: %s has a negative stride", fn, name);
    o.p = (const float *)v->ptr;
    o.s0 = v->strides[0]; o.s1 = v->strides[1]; o.s2 = v->strides[2]; o.s3 = v->strides[3];
    return 0;
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

int taps_args(const char *fn, const mcs_tensor *rast, const mcs_tensor *jitter, const mcs_tensor *kd, const mcs_tensor *ks, const mcs_tensor *gb_normal,
              const mcs_tensor *perturbed_nrm, const mcs_tensor *kd_jitter, const mcs_tensor *ks_jitter, TapArgs &a)
{
    MCS_REQUIRE(rast && rast->ptr, "%s: rast is null", fn);
    MCS_REQUIRE(kd && (kd->sizes[3] == 3 || kd->sizes[3] == 4), "%s: kd must have 3 or 4 channels", fn);
    MCS_REQUIRE((kd_jitter == nullptr) == (ks_jitter == nullptr), "%s: kd_jitter and ks_jitter go together", fn);
    const int32_t *bhw = rast->sizes;
    a.ckd = kd->sizes[3];
    a.mlp = kd_jitter != nullptr;
    a.has_pn = perturbed_nrm != nullptr;
    if (int e = view(fn, "rast", rast, 4, bhw, a.rast)) return e;
    if (int e = view(fn, "jitter", jitter, 2, bhw, a.jit)) return e;
    if (int e = view(fn, "kd", kd, a.ckd, bhw, a.kd)) return e;
    if (int e = view(fn, "ks", ks, 3, bhw, a.ks)) return e;
    if (int e = view(fn, "gb_normal", gb_normal, 3, bhw, a.nrm)) return e;
    if (a.has_pn)
        if (int e = view(fn, "perturbed_nrm", perturbed_nrm, 3, bhw, a.pn)) return e;
    if (a.mlp) {
        if (int e = view(fn, "kd_jitter", kd_jitter, a.ckd, bhw, a.kdj)) return e;
        if (int e = view(fn, "ks_jitter", ks_jitter, 3, bhw, a.ksj)) return e;
    }
    MCS_REQUIRE(bhw[0] >= 0 && bhw[1] >= 0 && bhw[2] >= 0, "%s: B, H, W must be >= 0", fn);
    MCS_REQUIRE((int64_t)bhw[0] * bhw[1] * bhw[2] < (int64_t)1 << 31, "%s: at most 2^31 - 1 pixels", fn);
    a.B = bhw[0]; a.H = bhw[1]; a.W = bhw[2];
    return 0;
}

unsigned taps_blocks(const TapArgs &a) { return (unsigned)((tex_pixel_threads(a.B, a.H, a.W) + TP_THREADS - 1) / TP_THREADS); }

}  // namespace

extern "C" {

int mcs_jitter_taps_fwd(const mcs_tensor *rast, const mcs_tensor *jitter, const mcs_tensor *kd, const mcs_tensor *ks, const mcs_tensor *gb_normal,
                        const mcs_tensor *perturbed_nrm, const mcs_tensor *kd_jitter, const mcs_tensor *ks_jitter, float *kd_grad, float *ks_grad,
                        float *normal_grad, float *perturbed_nrm_grad, mcs_stream stream)
{
    TapArgs a{};
    if (int e = taps_args("jitter_taps_fwd", rast, jitter, kd, ks, gb_normal, perturbed_nrm, kd_jitter, ks_jitter, a)) return e;
    MCS_REQUIRE(kd_grad && ks_grad && normal_grad && (perturbed_nrm_grad || !a.has_pn), "jitter_taps_fwd: null output pointer");
    MCS_REQUIRE(aligned16(ks_grad) && aligned16(normal_grad) && aligned16(perturbed_nrm_grad), "jitter_taps_fwd: outputs must be 16-byte aligned");
    if ((int64_t)a.B * a.H * a.W == 0) return 0;
    a.o_kd = kd_grad; a.o_ks = ks_grad; a.o_n = normal_grad; a.o_p = perturbed_nrm_grad;
    k_taps_fwd<<<taps_blocks(a), TP_THREADS, 0, (cudaStream_t)stream>>>(a);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_jitter_taps_bwd(const mcs_tensor *rast, const mcs_tensor *jitter, const mcs_tensor *kd, const mcs_tensor *ks, const mcs_tensor *gb_normal,
                        const mcs_tensor *perturbed_nrm, const mcs_tensor *kd_jitter, const mcs_tensor *ks_jitter, const float *d_kd_grad,
                        const float *d_ks_grad, const float *d_normal_grad, const float *d_perturbed_nrm_grad, float *d_kd, float *d_ks,
                        float *d_gb_normal, float *d_perturbed_nrm, float *d_kd_jitter, float *d_ks_jitter, mcs_stream stream)
{
    TapArgs a{};
    if (int e = taps_args("jitter_taps_bwd", rast, jitter, kd, ks, gb_normal, perturbed_nrm, kd_jitter, ks_jitter, a)) return e;
    MCS_REQUIRE(d_kd_grad && d_ks_grad && d_normal_grad && (d_perturbed_nrm_grad || !a.has_pn), "jitter_taps_bwd: null upstream gradient");
    MCS_REQUIRE(d_kd && d_ks && d_gb_normal && (d_perturbed_nrm || !a.has_pn) && ((d_kd_jitter && d_ks_jitter) || !a.mlp),
                "jitter_taps_bwd: null gradient output");
    MCS_REQUIRE(aligned16(d_ks_grad) && aligned16(d_normal_grad) && aligned16(d_perturbed_nrm_grad) && aligned16(d_kd) && aligned16(d_ks) &&
                aligned16(d_gb_normal) && aligned16(d_perturbed_nrm), "jitter_taps_bwd: [..,4] gradients must be 16-byte aligned");
    if ((int64_t)a.B * a.H * a.W == 0) return 0;
    a.g_kd = d_kd_grad; a.g_ks = d_ks_grad; a.g_n = d_normal_grad; a.g_p = d_perturbed_nrm_grad;
    a.d_kd = d_kd; a.d_ks = d_ks; a.d_n = d_gb_normal; a.d_p = d_perturbed_nrm; a.d_kdj = d_kd_jitter; a.d_ksj = d_ks_jitter;
    k_taps_bwd<<<taps_blocks(a), TP_THREADS, 0, (cudaStream_t)stream>>>(a);
    MCS_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
