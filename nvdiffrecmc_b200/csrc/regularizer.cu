// regularizer.cu -- the image-space regularisers of the reference's render/regularizer.py:15-49 on sm_90a: shading_loss,
// material_smoothness_grad and chroma_loss, forward and backward, with no host synchronisation.
//
// Operands are fp32 [B,H,W,4] views (any element strides; float4 loads where a view is dense and 16-byte aligned), all of one
// shape; N = B*H*W pixels.  Gradients are written dense, contiguous [B,H,W,4], one thread per pixel, no atomics.
//
// Forward: one launch; CTA k sums the per-pixel terms of pixels [k*RG_CHUNK, (k+1)*RG_CHUNK) in double, in a fixed order (thread, then
// warp shuffles, then warps in order), and writes them as its partials; a single-CTA finish sums the partials in index order and writes
// the loss.  Two runs give the same bits.  Backward: one launch; it reads the upstream gradient G (one float) from the device.
//
// Contract: the reference's torch composition, operation for operation, with torch's conventions where calculus leaves a choice:
//   luma(x)  = ((x0 + x1) + x2) / 3, value(x) = x[i] with i the FIRST maximal channel of x0..x2 (the first NaN if any), as
//              torch.max(dim) returns it; both are repeated to 3 identical channels, so every mean below over a [B,H,W,3] tensor divides
//              by 3N, and the gradient through `repeat` sums the three copies ((g + g) + g), then luma's / 3 and its sums pass it on.
//   clamp    torch.clamp / torch.clip: NaN passes through; the backward passes the gradient where min <= x <= max (inclusive) and
//              gives 0 elsewhere and at NaN.  eps = 0.001f for value, luma and mean clamps; [0, 65535] in shading_loss.
//   abs'(x)  = sign(x), with sign(0) = sign(NaN) = 0.
//   srgb(f)  = f <= 0.0031308f ? f * 12.92f : powf(max(f, 0.0031308f), E) * 1.055f - 0.055f, E = fl32(1/2.4) (util.py:95-99); only
//              the selected branch has a gradient: 12.92f, or 1.055f * (E * powf(f, fl32(1/2.4 - 1))) where f >= 0.0031308f.
//   means    mean(t) * lambda rounds mean(t) to fp32, then multiplies by fl32(lambda); the backward gives every element of t the
//              gradient fl32(fl32(G * lambda) / fl32(numel)).  A lambda of 0 still evaluates its term (0 * inf = NaN as in the reference).
//   x / y    d x = g / y, d y = -g * ((x / y) / y);  x * y: d x = g * y.
// shading_loss (regularizer.py:27-38), per pixel, all in fp32 except the sums:
//   dl = luma(diffuse), sl = luma(specular), rv = value(ref), a = ref.w, s = dl + sl
//   img = srgb(logf(clamp(s * a, 0, 65535) + 1)), tgt = srgb(logf(clamp(rv * a, 0, 65535) + 1))
//   e = (|img - tgt| * dl) / clamp(s, eps)
//   loss = fl32(mean(e)) * ld + (fl32(mean(sl)) / clamp(fl32(mean(dl)), eps)) * ls       (sums: e, sl, dl; the three means are over 3N)
//   The forward also writes means = (mean(dl), mean(sl)) for the backward, whose ratio term needs both.  logf / powf are the device's
//   (not bit-equal to glibc's); this function's gradients are held to a bound, not to bits.
// material_smoothness_grad (regularizer.py:44-49):
//   loss = ((fl32(mean_N(luma(kd) * kd.w)) * lkd + fl32(mean_3N(ks.rgb * ks.w)) * lks) + fl32(mean_3N(nrm.rgb * nrm.w)) * lnrm
//   kd_grad may also have 5 channels (a 4-channel kd with alpha appended, the transparency configuration): luma reads channels 0..2 and
//   kd.w is the last channel, as the reference's kd_grad[..., -1]; channel 3 gets a gradient of exactly 0 and d kd_grad is [B,H,W,5].
// chroma_loss (regularizer.py:20-24):
//   t_c = (kd_c / clamp(value(kd), eps) - ref_c / clamp(value(ref), eps)) * ref.w,  loss = fl32(mean_3N(|t|)) * lc
//   d kd.w = 0; color_ref is a constant.
// The per-pixel arithmetic of material_smoothness_grad and chroma_loss is + - * / max and abs, every operation explicitly rounded
// (__fadd_rn ...), so their gradients equal the fp32 oracle (oracle/regularizer.c) bit for bit.
#include "common.cuh"

namespace {

constexpr int RG_THREADS = 256;
constexpr int RG_ITEMS = 8;                               // pixels per thread in the forward
constexpr int RG_CHUNK = RG_THREADS * RG_ITEMS;           // pixels per partial
constexpr float EPS = 0.001f;
constexpr float SRGB_T = 0.0031308f;
constexpr float SRGB_E = (float)(1.0 / 2.4);
constexpr float SRGB_EM1 = (float)(1.0 / 2.4 - 1.0);

struct Op {                      // one [B,H,W,4] operand (or a 5-channel kd_grad)
    const float *p;
    int64_t s0, s1, s2, s3;      // element strides
    int64_t sa;                  // element offset of the alpha (last) channel
    int vec;                     // 4 channels, dense and 16-byte aligned: one float4 per pixel
};

struct Grid { int H, W, npx; };

__device__ __forceinline__ float4 ld4(const Op &o, const Grid &g, int px)
{
    if (o.vec) return __ldg(reinterpret_cast<const float4 *>(o.p) + px);
    const int w = px % g.W, t = px / g.W, h = t % g.H, n = t / g.H;
    const float *q = o.p + n * o.s0 + h * o.s1 + w * o.s2;
    return make_float4(__ldg(q), __ldg(q + o.s3), __ldg(q + 2 * o.s3), __ldg(q + o.sa));
}

__device__ __forceinline__ float comp(float4 x, int i) { return i == 0 ? x.x : (i == 1 ? x.y : x.z); }
__device__ __forceinline__ float luma(float4 x) { return __fdiv_rn(__fadd_rn(__fadd_rn(x.x, x.y), x.z), 3.0f); }
__device__ __forceinline__ int argmax3(float4 x)             // torch.max(dim): the first NaN, else the first maximal channel
{
    int i = 0;
    float m = x.x;
    if (x.y > m || (x.y != x.y && m == m)) { i = 1; m = x.y; }
    if (x.z > m || (x.z != x.z && m == m)) i = 2;
    return i;
}
__device__ __forceinline__ float clamp_min(float x, float lo) { return x < lo ? lo : x; }                   // NaN passes
__device__ __forceinline__ float clamp_lh(float x, float lo, float hi) { return x < lo ? lo : (x > hi ? hi : x); }
__device__ __forceinline__ float sgn(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }     // 0 for +-0 and NaN
__device__ __forceinline__ float srgb(float f)
{
    return f <= SRGB_T ? __fmul_rn(f, 12.92f) : __fsub_rn(__fmul_rn(powf(clamp_min(f, SRGB_T), SRGB_E), 1.055f), 0.055f);
}
__device__ __forceinline__ float log_srgb(float x) { return srgb(logf(__fadd_rn(clamp_lh(x, 0.0f, 65535.0f), 1.0f))); }
// upstream gradient of mean(t) * lambda for each of the n elements of t
__device__ __forceinline__ float mean_grad(float G, float lambda, float n) { return __fdiv_rn(__fmul_rn(G, lambda), n); }
// gradient of one luma(x) from the gradient g of ONE of its three repeated copies
__device__ __forceinline__ float luma_grad(float g) { return __fdiv_rn(__fadd_rn(__fadd_rn(g, g), g), 3.0f); }

template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K])                   // fixed order; the result is valid in thread 0
{
    __shared__ double s[K][RG_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) v[k] += __shfl_xor_sync(0xFFFFFFFFu, v[k], d);
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) s[k][warp] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) {
            v[k] = 0.0;
            for (int w = 0; w < RG_THREADS / 32; ++w) v[k] += s[k][w];
        }
}

// ---- per-pixel terms ----
struct ShadingPx { float dl, sl, e; };
__device__ __forceinline__ ShadingPx shading_px(float4 d, float4 s, float4 r)
{
    ShadingPx o;
    o.dl = luma(d); o.sl = luma(s);
    const float a = r.w, sum = __fadd_rn(o.dl, o.sl);
    const float img = log_srgb(__fmul_rn(sum, a)), tgt = log_srgb(__fmul_rn(comp(r, argmax3(r)), a));
    o.e = __fdiv_rn(__fmul_rn(fabsf(__fsub_rn(img, tgt)), o.dl), clamp_min(sum, EPS));
    return o;
}

struct Chroma { float t[3]; };
__device__ __forceinline__ float clipped_value(float4 x) { return clamp_min(comp(x, argmax3(x)), EPS); }
__device__ __forceinline__ Chroma chroma_px(float4 k, float4 r)
{
    const float ck = clipped_value(k), cr = clipped_value(r);
    const float kc[3] = {k.x, k.y, k.z}, rc[3] = {r.x, r.y, r.z};
    Chroma o;
#pragma unroll
    for (int c = 0; c < 3; ++c) o.t[c] = __fmul_rn(__fsub_rn(__fdiv_rn(kc[c], ck), __fdiv_rn(rc[c], cr)), r.w);
    return o;
}

// ---- forward: per-CTA partials ----
enum { FN_SHADING = 0, FN_SMOOTH = 1, FN_CHROMA = 2 };
template <int FN> struct NSums;
template <> struct NSums<FN_SHADING> { static constexpr int K = 3; };
template <> struct NSums<FN_SMOOTH> { static constexpr int K = 3; };
template <> struct NSums<FN_CHROMA> { static constexpr int K = 1; };

template <int FN>
__global__ void __launch_bounds__(RG_THREADS) k_reg_partials(const Op a, const Op b, const Op c, const Grid g, double *__restrict__ part)
{
    constexpr int K = NSums<FN>::K;
    double v[K];
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = 0.0;
#pragma unroll 2
    for (int it = 0; it < RG_ITEMS; ++it) {
        const int px = blockIdx.x * RG_CHUNK + it * RG_THREADS + threadIdx.x;
        if (px >= g.npx) break;
        if constexpr (FN == FN_SHADING) {                     // a diffuse, b specular, c color_ref: sums of e, sl, dl
            const ShadingPx o = shading_px(ld4(a, g, px), ld4(b, g, px), ld4(c, g, px));
            v[0] += (double)o.e; v[1] += (double)o.sl; v[2] += (double)o.dl;
        } else if constexpr (FN == FN_SMOOTH) {               // a kd_grad, b ks_grad, c nrm_grad: one sum per term
            const float4 kd = ld4(a, g, px), ks = ld4(b, g, px), nr = ld4(c, g, px);
            v[0] += (double)__fmul_rn(luma(kd), kd.w);
            v[1] += ((double)__fmul_rn(ks.x, ks.w) + (double)__fmul_rn(ks.y, ks.w)) + (double)__fmul_rn(ks.z, ks.w);
            v[2] += ((double)__fmul_rn(nr.x, nr.w) + (double)__fmul_rn(nr.y, nr.w)) + (double)__fmul_rn(nr.z, nr.w);
        } else {                                              // a kd, b color_ref: sum of |t|
            const Chroma o = chroma_px(ld4(a, g, px), ld4(b, g, px));
            v[0] += ((double)fabsf(o.t[0]) + (double)fabsf(o.t[1])) + (double)fabsf(o.t[2]);
        }
    }
    block_sum<K>(v);
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) part[(int64_t)K * blockIdx.x + k] = v[k];
}

struct Lambdas { float l0, l1, l2; };

template <int FN>
__global__ void __launch_bounds__(RG_THREADS) k_reg_finish(const double *__restrict__ part, int nparts, int64_t npx, Lambdas lam,
                                                           float *__restrict__ loss, float *__restrict__ means)
{
    constexpr int K = NSums<FN>::K;
    double v[K];
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = 0.0;
    for (int i = threadIdx.x; i < nparts; i += RG_THREADS)
#pragma unroll
        for (int k = 0; k < K; ++k) v[k] += part[(int64_t)K * i + k];
    block_sum<K>(v);
    if (threadIdx.x != 0) return;
    const double n = (double)npx;                  // a mean over 3N of three identical copies is the mean over N of one
    if constexpr (FN == FN_SHADING) {
        const float me = (float)(v[0] / n), ms = (float)(v[1] / n), md = (float)(v[2] / n);
        *loss = __fadd_rn(__fmul_rn(me, lam.l0), __fmul_rn(__fdiv_rn(ms, clamp_min(md, EPS)), lam.l1));
        means[0] = md; means[1] = ms;
    } else if constexpr (FN == FN_SMOOTH) {
        const float m0 = (float)(v[0] / n), m1 = (float)(v[1] / (3.0 * n)), m2 = (float)(v[2] / (3.0 * n));
        *loss = __fadd_rn(__fadd_rn(__fmul_rn(m0, lam.l0), __fmul_rn(m1, lam.l1)), __fmul_rn(m2, lam.l2));
    } else {
        *loss = __fmul_rn((float)(v[0] / (3.0 * n)), lam.l0);
    }
}

// ---- backward: one thread per pixel ----
__device__ __forceinline__ void st4(float *p, int px, float x, float y, float z, float w)
{
    reinterpret_cast<float4 *>(p)[px] = make_float4(x, y, z, w);
}

__global__ void __launch_bounds__(RG_THREADS) k_shading_bwd(const Op d, const Op s, const Op r, const Grid g, Lambdas lam,
                                                            const float *__restrict__ means, const float *__restrict__ d_loss,
                                                            float *__restrict__ d_d, float *__restrict__ d_s)
{
    const int px = blockIdx.x * RG_THREADS + threadIdx.x;
    if (px >= g.npx) return;
    const float G = __ldg(d_loss), n3 = (float)(3 * (int64_t)g.npx);
    // global terms: mean(e) * ld and mean(sl) / clamp(mean(dl), eps) * ls
    const float g_e = mean_grad(G, lam.l0, n3);
    const float md = __ldg(means), ms = __ldg(means + 1), cmd = clamp_min(md, EPS), gq = __fmul_rn(G, lam.l1);
    const float g_ms = __fdiv_rn(gq, cmd), g_cmd = __fmul_rn(-gq, __fdiv_rn(__fdiv_rn(ms, cmd), cmd));
    const float g_md = md >= EPS ? g_cmd : 0.0f;
    const float g_slm = __fdiv_rn(g_ms, n3), g_dlm = __fdiv_rn(g_md, n3);

    const float4 D = ld4(d, g, px), S = ld4(s, g, px), R = ld4(r, g, px);
    const float dl = luma(D), sl = luma(S), a = R.w, sum = __fadd_rn(dl, sl), x = __fmul_rn(sum, a);
    const float u = clamp_lh(x, 0.0f, 65535.0f), L = logf(__fadd_rn(u, 1.0f));
    const float img = srgb(L), tgt = log_srgb(__fmul_rn(comp(R, argmax3(R)), a));
    const float diff = __fsub_rn(img, tgt), ad = fabsf(diff), cs = clamp_min(sum, EPS), num = __fmul_rn(ad, dl);
    // e = num / cs, num = ad * dl, cs = clamp(sum, eps)
    const float g_num = __fdiv_rn(g_e, cs), g_cs = __fmul_rn(-g_e, __fdiv_rn(__fdiv_rn(num, cs), cs));
    const float g_ad = __fmul_rn(g_num, dl), g_dl1 = __fmul_rn(g_num, ad);
    const float g_s2 = sum >= EPS ? g_cs : 0.0f;
    // ad = |img - tgt|, img = srgb(L), L = log(u + 1), u = clamp(x, 0, 65535), x = sum * a
    const float g_img = __fmul_rn(g_ad, sgn(diff));
    float g_L;
    if (L <= SRGB_T) g_L = __fmul_rn(g_img, 12.92f);
    else g_L = L >= SRGB_T ? __fmul_rn(__fmul_rn(g_img, 1.055f), __fmul_rn(SRGB_E, powf(L, SRGB_EM1))) : 0.0f;
    const float g_u = __fdiv_rn(g_L, __fadd_rn(u, 1.0f));
    const float g_x = (x >= 0.0f && x <= 65535.0f) ? g_u : 0.0f;
    const float g_s1 = __fmul_rn(g_x, a);
    const float g_dl = __fadd_rn(__fadd_rn(__fadd_rn(g_dl1, g_s2), g_s1), g_dlm);
    const float g_sl = __fadd_rn(__fadd_rn(g_s2, g_s1), g_slm);
    const float gd = luma_grad(g_dl), gs = luma_grad(g_sl);
    st4(d_d, px, gd, gd, gd, 0.0f);
    st4(d_s, px, gs, gs, gs, 0.0f);
}

// ckd: kd_grad's channel count (4 or 5; d_kd is then dense [B,H,W,ckd])
__global__ void __launch_bounds__(RG_THREADS) k_smooth_bwd(const Op kd, const Op ks, const Op nr, const Grid g, Lambdas lam, int ckd,
                                                           const float *__restrict__ d_loss, float *__restrict__ d_kd,
                                                           float *__restrict__ d_ks, float *__restrict__ d_nr)
{
    const int px = blockIdx.x * RG_THREADS + threadIdx.x;
    if (px >= g.npx) return;
    const float G = __ldg(d_loss), n1 = (float)g.npx, n3 = (float)(3 * (int64_t)g.npx);
    const float g1 = mean_grad(G, lam.l0, n1), g2 = mean_grad(G, lam.l1, n3), g3 = mean_grad(G, lam.l2, n3);
    const float4 K = ld4(kd, g, px), S = ld4(ks, g, px), N = ld4(nr, g, px);
    const float gl = __fdiv_rn(__fmul_rn(g1, K.w), 3.0f);
    if (ckd == 4) {
        st4(d_kd, px, gl, gl, gl, __fmul_rn(g1, luma(K)));
    } else {
        float *q = d_kd + (int64_t)px * 5;
        q[0] = gl; q[1] = gl; q[2] = gl; q[3] = 0.0f; q[4] = __fmul_rn(g1, luma(K));
    }
    st4(d_ks, px, __fmul_rn(g2, S.w), __fmul_rn(g2, S.w), __fmul_rn(g2, S.w),
        __fadd_rn(__fadd_rn(__fmul_rn(g2, S.x), __fmul_rn(g2, S.y)), __fmul_rn(g2, S.z)));
    st4(d_nr, px, __fmul_rn(g3, N.w), __fmul_rn(g3, N.w), __fmul_rn(g3, N.w),
        __fadd_rn(__fadd_rn(__fmul_rn(g3, N.x), __fmul_rn(g3, N.y)), __fmul_rn(g3, N.z)));
}

__global__ void __launch_bounds__(RG_THREADS) k_chroma_bwd(const Op kd, const Op ref, const Grid g, Lambdas lam, const float *__restrict__ d_loss,
                                                           float *__restrict__ d_kd)
{
    const int px = blockIdx.x * RG_THREADS + threadIdx.x;
    if (px >= g.npx) return;
    const float G = __ldg(d_loss), n3 = (float)(3 * (int64_t)g.npx);
    const float ge = mean_grad(G, lam.l0, n3);
    const float4 K = ld4(kd, g, px), R = ld4(ref, g, px);
    const int ik = argmax3(K);
    const float vk = comp(K, ik), ck = clamp_min(vk, EPS);
    const Chroma t = chroma_px(K, R);
    const float kc[3] = {K.x, K.y, K.z};
    float gdir[3], gck = 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float g_opt = __fmul_rn(__fmul_rn(ge, sgn(t.t[c])), R.w);     // |.|, then * ref.w; the subtraction passes it on
        gdir[c] = __fdiv_rn(g_opt, ck);
        const float gc = __fmul_rn(-g_opt, __fdiv_rn(__fdiv_rn(kc[c], ck), ck));
        gck = c == 0 ? gc : __fadd_rn(gck, gc);
    }
    const float gv = vk >= EPS ? gck : 0.0f;
    st4(d_kd, px, __fadd_rn(gdir[0], ik == 0 ? gv : 0.0f), __fadd_rn(gdir[1], ik == 1 ? gv : 0.0f), __fadd_rn(gdir[2], ik == 2 ? gv : 0.0f), 0.0f);
}

// ---- host side ----
int npartials(int64_t npx) { return (int)((npx + RG_CHUNK - 1) / RG_CHUNK); }

// Checks the operand views of one entry (non-null, [B,H,W,4] -- operand 0 may have 5 channels when kd5 -- one B, H, W, non-negative
// strides, fewer than 2^31 pixels) and fills ops.
int views(const char *fn, int n, const mcs_tensor *const *v, const char *const *names, Op *ops, Grid &g, bool kd5 = false)
{
    for (int i = 0; i < n; ++i) {
        MCS_REQUIRE(v[i] && v[i]->ptr, "%s: %s is null", fn, names[i]);
        if (i == 0 && kd5)
            MCS_REQUIRE(v[i]->sizes[3] == 4 || v[i]->sizes[3] == 5, "%s: %s must have 4 or 5 channels, got %d", fn, names[i], v[i]->sizes[3]);
        else
            MCS_REQUIRE(v[i]->sizes[3] == 4, "%s: %s must have 4 channels, got %d", fn, names[i], v[i]->sizes[3]);
        for (int d = 0; d < 3; ++d)
            MCS_REQUIRE(v[i]->sizes[d] == v[0]->sizes[d], "%s: %s must have the shape of %s", fn, names[i], names[0]);
        for (int d = 0; d < 4; ++d) MCS_REQUIRE(v[i]->strides[d] >= 0, "%s: %s has a negative stride", fn, names[i]);
    }
    const int B = v[0]->sizes[0], H = v[0]->sizes[1], W = v[0]->sizes[2];
    MCS_REQUIRE(B > 0 && H > 0 && W > 0, "%s: empty operands", fn);
    const int64_t npx = (int64_t)B * H * W;
    MCS_REQUIRE(npx < (int64_t)1 << 31, "%s: %lld pixels, at most 2^31 - 1", fn, (long long)npx);
    g.H = H; g.W = W; g.npx = (int)npx;
    for (int i = 0; i < n; ++i) {
        const int32_t *sz = v[i]->sizes, *st = v[i]->strides;
        Op &o = ops[i];
        o.p = (const float *)v[i]->ptr;
        o.s0 = st[0]; o.s1 = st[1]; o.s2 = st[2]; o.s3 = st[3];
        o.sa = (int64_t)(sz[3] - 1) * st[3];
        o.vec = sz[3] == 4 && ((uintptr_t)o.p & 15) == 0 && st[3] == 1 && (sz[2] == 1 || st[2] == 4) && (sz[1] == 1 || st[1] == 4 * W) &&
                (sz[0] == 1 || st[0] == 4 * (int64_t)H * W);
    }
    return 0;
}

bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

template <int FN>
int reg_fwd(const char *fn, int n, const mcs_tensor *const *v, const char *const *names, Lambdas lam, double *partials, float *loss, float *means,
            mcs_stream stream)
{
    Op ops[3] = {};
    Grid g{};
    if (int e = views(fn, n, v, names, ops, g, FN == FN_SMOOTH)) return e;
    MCS_REQUIRE(partials && loss && (means || FN != FN_SHADING), "%s: null output pointer", fn);
    const cudaStream_t s = (cudaStream_t)stream;
    const int np = npartials(g.npx);
    k_reg_partials<FN><<<np, RG_THREADS, 0, s>>>(ops[0], ops[1], ops[2], g, partials);
    MCS_LAUNCH_CHECK();
    k_reg_finish<FN><<<1, RG_THREADS, 0, s>>>(partials, np, g.npx, lam, loss, means);
    MCS_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" {

int32_t mcs_shading_loss_num_partials(int32_t B, int32_t H, int32_t W) { return npartials((int64_t)B * H * W); }
int32_t mcs_material_smoothness_grad_num_partials(int32_t B, int32_t H, int32_t W) { return npartials((int64_t)B * H * W); }
int32_t mcs_chroma_loss_num_partials(int32_t B, int32_t H, int32_t W) { return npartials((int64_t)B * H * W); }

int mcs_shading_loss_fwd(const mcs_tensor *diffuse_light, const mcs_tensor *specular_light, const mcs_tensor *color_ref, float lambda_diffuse,
                         float lambda_specular, double *partials, float *loss, float *means, mcs_stream stream)
{
    const mcs_tensor *v[3] = {diffuse_light, specular_light, color_ref};
    const char *names[3] = {"diffuse_light", "specular_light", "color_ref"};
    return reg_fwd<FN_SHADING>("shading_loss_fwd", 3, v, names, Lambdas{lambda_diffuse, lambda_specular, 0.0f}, partials, loss, means, stream);
}

int mcs_shading_loss_bwd(const mcs_tensor *diffuse_light, const mcs_tensor *specular_light, const mcs_tensor *color_ref, float lambda_diffuse,
                         float lambda_specular, const float *means, const float *d_loss, float *d_diffuse_light, float *d_specular_light,
                         mcs_stream stream)
{
    const mcs_tensor *v[3] = {diffuse_light, specular_light, color_ref};
    const char *names[3] = {"diffuse_light", "specular_light", "color_ref"};
    Op ops[3] = {};
    Grid g{};
    if (int e = views("shading_loss_bwd", 3, v, names, ops, g)) return e;
    MCS_REQUIRE(means && d_loss && d_diffuse_light && d_specular_light, "shading_loss_bwd: null pointer argument");
    MCS_REQUIRE(aligned16(d_diffuse_light) && aligned16(d_specular_light), "shading_loss_bwd: gradient outputs must be 16-byte aligned");
    k_shading_bwd<<<(g.npx + RG_THREADS - 1) / RG_THREADS, RG_THREADS, 0, (cudaStream_t)stream>>>(
        ops[0], ops[1], ops[2], g, Lambdas{lambda_diffuse, lambda_specular, 0.0f}, means, d_loss, d_diffuse_light, d_specular_light);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_material_smoothness_grad_fwd(const mcs_tensor *kd_grad, const mcs_tensor *ks_grad, const mcs_tensor *nrm_grad, float lambda_kd,
                                     float lambda_ks, float lambda_nrm, double *partials, float *loss, mcs_stream stream)
{
    const mcs_tensor *v[3] = {kd_grad, ks_grad, nrm_grad};
    const char *names[3] = {"kd_grad", "ks_grad", "nrm_grad"};
    return reg_fwd<FN_SMOOTH>("material_smoothness_grad_fwd", 3, v, names, Lambdas{lambda_kd, lambda_ks, lambda_nrm}, partials, loss, nullptr,
                              stream);
}

int mcs_material_smoothness_grad_bwd(const mcs_tensor *kd_grad, const mcs_tensor *ks_grad, const mcs_tensor *nrm_grad, float lambda_kd,
                                     float lambda_ks, float lambda_nrm, const float *d_loss, float *d_kd_grad, float *d_ks_grad,
                                     float *d_nrm_grad, mcs_stream stream)
{
    const mcs_tensor *v[3] = {kd_grad, ks_grad, nrm_grad};
    const char *names[3] = {"kd_grad", "ks_grad", "nrm_grad"};
    Op ops[3] = {};
    Grid g{};
    if (int e = views("material_smoothness_grad_bwd", 3, v, names, ops, g, true)) return e;
    const int ckd = kd_grad->sizes[3];
    MCS_REQUIRE(d_loss && d_kd_grad && d_ks_grad && d_nrm_grad, "material_smoothness_grad_bwd: null pointer argument");
    MCS_REQUIRE((aligned16(d_kd_grad) || ckd == 5) && aligned16(d_ks_grad) && aligned16(d_nrm_grad),
                "material_smoothness_grad_bwd: gradient outputs must be 16-byte aligned (d_kd_grad: when 4-channel)");
    k_smooth_bwd<<<(g.npx + RG_THREADS - 1) / RG_THREADS, RG_THREADS, 0, (cudaStream_t)stream>>>(
        ops[0], ops[1], ops[2], g, Lambdas{lambda_kd, lambda_ks, lambda_nrm}, ckd, d_loss, d_kd_grad, d_ks_grad, d_nrm_grad);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_chroma_loss_fwd(const mcs_tensor *kd, const mcs_tensor *color_ref, float lambda_chroma, double *partials, float *loss, mcs_stream stream)
{
    const mcs_tensor *v[2] = {kd, color_ref};
    const char *names[2] = {"kd", "color_ref"};
    return reg_fwd<FN_CHROMA>("chroma_loss_fwd", 2, v, names, Lambdas{lambda_chroma, 0.0f, 0.0f}, partials, loss, nullptr, stream);
}

int mcs_chroma_loss_bwd(const mcs_tensor *kd, const mcs_tensor *color_ref, float lambda_chroma, const float *d_loss, float *d_kd, mcs_stream stream)
{
    const mcs_tensor *v[2] = {kd, color_ref};
    const char *names[2] = {"kd", "color_ref"};
    Op ops[3] = {};
    Grid g{};
    if (int e = views("chroma_loss_bwd", 2, v, names, ops, g)) return e;
    MCS_REQUIRE(d_loss && d_kd, "chroma_loss_bwd: null pointer argument");
    MCS_REQUIRE(aligned16(d_kd), "chroma_loss_bwd: the gradient output must be 16-byte aligned");
    k_chroma_bwd<<<(g.npx + RG_THREADS - 1) / RG_THREADS, RG_THREADS, 0, (cudaStream_t)stream>>>(ops[0], ops[1], g, Lambdas{lambda_chroma, 0.0f, 0.0f},
                                                                                                   d_loss, d_kd);
    MCS_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
