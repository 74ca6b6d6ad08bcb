// lossmesh.cu -- the two cheap brackets of the hot path (SURVEY.md section 8 row f3), H100 versions:
//   * image_loss  : tonemap (log-sRGB) + {L1, MSE, RELMSE, SMAPE, N2N} per pixel with a deterministic two-level reduction
//                   (replaces imgLossFwdKernel / imgLossBwdKernel, render/renderutils/c_src/loss.cu:105-227, and
//                   image_loss_fwd/_bwd, torch_bindings.cpp:739-800).  FIX: "n2n" is honoured (the reference's strToLoss,
//                   torch_bindings.cpp:727-737, has no "n2n" case and silently computes L1 on the CUDA path).
//   * xfm_points / xfm_vectors : batched 4x4 transform of [1|B, V, 3] points (replaces xfmPointsFwd/BwdKernel,
//                   render/renderutils/c_src/mesh.cu:19-90, and xfm_fwd/_bwd, torch_bindings.cpp:803-864).
//   * coverage_loss : the geometry passes' whole image loss (geometry/dmtet.py:229-230, geometry/dlmesh.py:75-76),
//                       mse(shaded.a, ref.a) + image_loss(shaded.rgb * ref.a, ref.rgb * ref.a), in one launch each way (+ a one-CTA finish).
// All are HBM-streaming: image_loss reads 24 B/px (fwd) / writes 24 B/px more (bwd); coverage_loss reads 32 B/px (fwd) and writes 16 B/px
// more (bwd); xfm reads 12 B and writes 16 B per vertex.
//
// coverage_loss contract.  N = B*H*W pixels of shaded and ref ([B,H,W,4] fp32, any strides); per pixel, in fp32:
//   img_c = shaded_c * ref.a, tgt_c = ref_c * ref.a (c = rgb, each product rounded once, as torch's mul)
//   colour = image_loss's per-pixel value of (img, tgt): the clamps, the tonemap and loss_fwd1 of k_image_loss_fwd, summed over c, * (1/3)
//   coverage = (shaded.a - ref.a)^2, the difference and the square each rounded once
// Forward: CTA k covers pixels [256k, 256k + 256) and sums each term in k_image_loss_fwd's order (butterfly shuffles in each warp, then the
// eight warp sums in warp order from 0, all fp32); it writes coverage to partials[k] and colour to partials[P + k], P = num_partials.  The
// colour partials are therefore image_loss's partials of (img, tgt) bit for bit.  The finish (one CTA) sums each half of partials in double,
// thread t taking partials t, t + 256, ... in index order, then shuffles and warps as above, and writes
//   loss = fl32(coverage_sum / N + colour_sum / N)          (both quotients and their sum in double, one rounding to fp32)
// Backward: one thread per pixel reads the upstream gradient G from the device and writes d shaded [B,H,W,4] (dense, 16-byte aligned),
// every value as autograd forms it through the two torch lines:
//   rgb:   dv = fl(G * fl(1 / fl32(N))) * (1/3) -- torch's CUDA division of sum(partials) by the host scalar N multiplies by the rounded
//          reciprocal; the sum passes it to every partial, and k_image_loss_bwd takes a third -- then image_loss's channel backward on
//          (img_c, tgt_c) and d shaded_c = fl(d img_c * ref.a), mul's backward.
//   alpha: fl(fl(fl32(2 / N) * fl(shaded.a - ref.a)) * G), mse_loss's backward (alpha * (input - target) * grad, alpha = 2 / numel).
//   Each value is then added to +0, as autograd adds the two slices' zero-filled gradients: -0 becomes +0.  d ref is not formed.
// k_image_loss_fwd / _bwd keep their own inline copy of the per-channel loop so that their SASS is what it was; image_loss_px and
// image_loss_ch_bwd restate it line for line, and tests/test_gpu_coverage_loss.py holds the two to the same bits.
#include "common.cuh"

namespace {

enum { LOSS_L1 = 0, LOSS_MSE = 1, LOSS_RELMSE = 2, LOSS_SMAPE = 3, LOSS_N2N = 4 };
constexpr int LOSS_BLOCK = 256;

__device__ __forceinline__ float bwd_abs(float x) { return x == 0.0f ? 0.0f : (x < 0.0f ? -1.0f : 1.0f); }        // loss.cu:17
// loss.cu:28-41
__device__ __forceinline__ float fwd_srgb(float x) { return x > 0.0031308f ? powf(fmaxf(x, 0.0031308f), 1.0f / 2.4f) * 1.055f - 0.055f : 12.92f * fmaxf(x, 0.0f); }
__device__ __forceinline__ float bwd_srgb(float x, float d_out)
{
    if (x > 0.0031308f) return d_out * 0.439583f / powf(x, 0.583333f);
    if (x > 0.0f) return d_out * 12.92f;
    return 0.0f;
}
__device__ __forceinline__ float fwd_tonemap(float x) { return fwd_srgb(logf(x + 1.0f)); }                          // loss.cu:43-46
__device__ __forceinline__ float bwd_tonemap(float x, float d_out)                                                  // loss.cu:48-65
{
    if (x > 0.0f && x < 65535.0f) return bwd_srgb(logf(x + 1.0f), d_out) * (1.0f / (x + 1.0f));
    return 0.0f;
}

__device__ __forceinline__ float loss_fwd1(int loss, float img, float tgt)
{
    const float eps = 0.01f;
    const float d = img - tgt;
    switch (loss) {
    case LOSS_MSE: return d * d;
    case LOSS_RELMSE: return d * d / (img * img + tgt * tgt + eps);             // loss.cu:67-70
    case LOSS_N2N: return d * d / (img * img + eps);                            // loss.cu:79-82
    case LOSS_SMAPE: return fabsf(d) / (img + tgt + eps);                       // loss.cu:92-95
    default: return fabsf(d);
    }
}
__device__ __forceinline__ void loss_bwd1(int loss, float img, float tgt, float dv, float &d_img, float &d_tgt)
{
    const float eps = 0.01f;
    const float d = img - tgt;
    switch (loss) {
    case LOSS_MSE: d_img = dv * 2.0f * d; d_tgt = -d_img; break;                                            // loss.cu:181-185
    case LOSS_RELMSE: {                                                                                     // loss.cu:72-77
        const float den = tgt * tgt + img * img + eps;
        d_img = dv * 2.0f * d * (tgt * (tgt + img) + eps) / (den * den);
        d_tgt = -dv * 2.0f * d * (img * (tgt + img) + eps) / (den * den);
    } break;
    case LOSS_N2N: {                                                                                        // loss.cu:84-89
        const float den = img * img + eps;
        d_img = dv * 2.0f * d / den; d_tgt = -d_img;
    } break;
    case LOSS_SMAPE: {                                                                                      // loss.cu:97-102
        const float den = tgt + img + eps;
        d_img = dv * bwd_abs(d) * (2.0f * tgt + eps) / (den * den);
        d_tgt = -dv * bwd_abs(d) * (2.0f * img + eps) / (den * den);
    } break;
    default: d_img = dv * bwd_abs(d); d_tgt = -d_img; break;
    }
}

struct LossParams {
    TView img, tgt;
    int N, H, W; int64_t npx;
    int loss, tonemap;
    float *partial;              // fwd: [nblocks] per-CTA sums of (sum_c loss)/3
    TView dout; int dout_n;      // bwd: upstream gradient per CTA partial (or a single broadcast value)
    float *d_img, *d_tgt;        // bwd: contiguous [N,H,W,3]
};

__global__ void __launch_bounds__(LOSS_BLOCK) k_image_loss_fwd(LossParams p)
{
    __shared__ float s_part[LOSS_BLOCK / 32];
    const int64_t px = (int64_t)blockIdx.x * LOSS_BLOCK + threadIdx.x;
    float v = 0.0f;
    if (px < p.npx) {
        const int w = (int)(px % p.W); const int64_t t = px / p.W; const int h = (int)(t % p.H), n = (int)(t / p.H);
        f3 a = p.img.ld3(n, h, w), b = p.tgt.ld3(n, h, w);
        float ia[3] = {a.x, a.y, a.z}, tb[3] = {b.x, b.y, b.z};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float x = clampf(ia[c], 0.0f, 65535.0f), y = clampf(tb[c], 0.0f, 65535.0f);       // loss.cu:118-119 (always, not only when tonemapping)
            if (p.tonemap) { x = fwd_tonemap(x); y = fwd_tonemap(y); }
            v += loss_fwd1(p.loss, x, y);
        }
        v *= (1.0f / 3.0f);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.0f;
#pragma unroll
        for (int i = 0; i < LOSS_BLOCK / 32; ++i) s += s_part[i];
        p.partial[blockIdx.x] = s;              // fixed order: deterministic
    }
}

__global__ void __launch_bounds__(LOSS_BLOCK) k_image_loss_bwd(LossParams p)
{
    const int64_t px = (int64_t)blockIdx.x * LOSS_BLOCK + threadIdx.x;
    if (px >= p.npx) return;
    const int w = (int)(px % p.W); const int64_t t = px / p.W; const int h = (int)(t % p.H), n = (int)(t / p.H);
    const float d_out = __ldg(p.dout.p + (p.dout_n == 1 ? 0 : (int64_t)blockIdx.x * p.dout.s0));
    f3 a = p.img.ld3(n, h, w), b = p.tgt.ld3(n, h, w);
    float ia[3] = {a.x, a.y, a.z}, tb[3] = {b.x, b.y, b.z}, gi[3], gt[3];
    const float dv = d_out * (1.0f / 3.0f);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float x = ia[c], y = tb[c];
        if (p.tonemap) { x = fwd_tonemap(x); y = fwd_tonemap(y); }                 // loss.cu:163-167 (no clamp in the replay, as in the reference)
        float di, dt;
        loss_bwd1(p.loss, x, y, dv, di, dt);
        if (p.tonemap) { di = bwd_tonemap(ia[c], di); dt = bwd_tonemap(tb[c], dt); }
        if (ia[c] <= 0.0f || ia[c] >= 65535.0f) di = 0.0f;                          // loss.cu:217-222
        if (tb[c] <= 0.0f || tb[c] >= 65535.0f) dt = 0.0f;
        gi[c] = di; gt[c] = dt;
    }
    float *o1 = p.d_img + px * 3, *o2 = p.d_tgt + px * 3;
    o1[0] = gi[0]; o1[1] = gi[1]; o1[2] = gi[2];
    o2[0] = gt[0]; o2[1] = gt[1]; o2[2] = gt[2];
}

// ---- coverage_loss (contract in the file header) ----
// image_loss's per-pixel value, k_image_loss_fwd's loop
__device__ __forceinline__ float image_loss_px(int loss, int tonemap, const float (&ia)[3], const float (&tb)[3])
{
    float v = 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float x = clampf(ia[c], 0.0f, 65535.0f), y = clampf(tb[c], 0.0f, 65535.0f);
        if (tonemap) { x = fwd_tonemap(x); y = fwd_tonemap(y); }
        v += loss_fwd1(loss, x, y);
    }
    return v * (1.0f / 3.0f);
}

// d img of one channel, k_image_loss_bwd's loop body (d tgt is not formed)
__device__ __forceinline__ float image_loss_ch_bwd(int loss, int tonemap, float img, float tgt, float dv)
{
    float x = img, y = tgt;
    if (tonemap) { x = fwd_tonemap(x); y = fwd_tonemap(y); }
    float di, dt;
    loss_bwd1(loss, x, y, dv, di, dt);
    if (tonemap) di = bwd_tonemap(img, di);
    if (img <= 0.0f || img >= 65535.0f) di = 0.0f;
    return di;
}

// sums v[k] over the CTA in k_image_loss_fwd's order; the sums are valid in thread 0
template <typename T, int K>
__device__ __forceinline__ void cta_sum(T (&v)[K])
{
    __shared__ T s_part[K][LOSS_BLOCK / 32];
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xFFFFFFFFu, v[k], o);
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) s_part[k][threadIdx.x >> 5] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) {
            T s = 0;
#pragma unroll
            for (int i = 0; i < LOSS_BLOCK / 32; ++i) s += s_part[k][i];
            v[k] = s;
        }
}

struct CoverageParams {
    TView img, ref;                 // [B,H,W,4]
    int img_vec, ref_vec;           // dense and 16-byte aligned: one float4 per pixel
    int H, W; int64_t npx;
    int loss, tonemap;
    float *partial;                 // fwd: [2P], coverage then colour
    const float *d_loss;            // bwd: G, one float
    float inv_npx, two_over_npx;    // bwd: fl32(1 / fl32(N)), fl32(2 / N)
    float *d_img;                   // bwd: dense [B,H,W,4]
};

__device__ __forceinline__ float4 ld_rgba(const TView &v, int vec, int64_t px, int n, int h, int w)
{
    if (vec) return __ldg(reinterpret_cast<const float4 *>(v.p) + px);
    const float *q = v.p + v.off(n, h, w);
    return make_float4(__ldg(q), __ldg(q + v.s3), __ldg(q + 2 * v.s3), __ldg(q + 3 * v.s3));
}

__device__ __forceinline__ void premultiply(float4 s, float4 r, float (&ia)[3], float (&tb)[3])
{
    ia[0] = __fmul_rn(s.x, r.w); ia[1] = __fmul_rn(s.y, r.w); ia[2] = __fmul_rn(s.z, r.w);
    tb[0] = __fmul_rn(r.x, r.w); tb[1] = __fmul_rn(r.y, r.w); tb[2] = __fmul_rn(r.z, r.w);
}

__global__ void __launch_bounds__(LOSS_BLOCK) k_coverage_loss_fwd(CoverageParams p)
{
    const int64_t px = (int64_t)blockIdx.x * LOSS_BLOCK + threadIdx.x;
    float v[2] = {0.0f, 0.0f};                                  // coverage, colour
    if (px < p.npx) {
        const int w = (int)(px % p.W); const int64_t t = px / p.W; const int h = (int)(t % p.H), n = (int)(t / p.H);
        const float4 s = ld_rgba(p.img, p.img_vec, px, n, h, w), r = ld_rgba(p.ref, p.ref_vec, px, n, h, w);
        float ia[3], tb[3];
        premultiply(s, r, ia, tb);
        const float e = __fsub_rn(s.w, r.w);
        v[0] = __fmul_rn(e, e);
        v[1] = image_loss_px(p.loss, p.tonemap, ia, tb);
    }
    cta_sum(v);
    if (threadIdx.x == 0) {
        p.partial[blockIdx.x] = v[0];
        p.partial[gridDim.x + blockIdx.x] = v[1];
    }
}

__global__ void __launch_bounds__(LOSS_BLOCK) k_coverage_loss_finish(const float *__restrict__ part, int nparts, int64_t npx, float *__restrict__ loss)
{
    double v[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < nparts; i += LOSS_BLOCK) {
        v[0] += (double)part[i];
        v[1] += (double)part[nparts + i];
    }
    cta_sum(v);
    if (threadIdx.x == 0) *loss = (float)(v[0] / (double)npx + v[1] / (double)npx);
}

__global__ void __launch_bounds__(LOSS_BLOCK) k_coverage_loss_bwd(CoverageParams p)
{
    const int64_t px = (int64_t)blockIdx.x * LOSS_BLOCK + threadIdx.x;
    if (px >= p.npx) return;
    const int w = (int)(px % p.W); const int64_t t = px / p.W; const int h = (int)(t % p.H), n = (int)(t / p.H);
    const float G = __ldg(p.d_loss);
    const float dv = __fmul_rn(G, p.inv_npx) * (1.0f / 3.0f);
    const float4 s = ld_rgba(p.img, p.img_vec, px, n, h, w), r = ld_rgba(p.ref, p.ref_vec, px, n, h, w);
    float ia[3], tb[3], g[3];
    premultiply(s, r, ia, tb);
#pragma unroll
    for (int c = 0; c < 3; ++c) g[c] = __fadd_rn(__fmul_rn(image_loss_ch_bwd(p.loss, p.tonemap, ia[c], tb[c], dv), r.w), 0.0f);
    const float ga = __fadd_rn(__fmul_rn(__fmul_rn(p.two_over_npx, __fsub_rn(s.w, r.w)), G), 0.0f);
    reinterpret_cast<float4 *>(p.d_img)[px] = make_float4(g[0], g[1], g[2], ga);
}

struct XfmParams {
    const float *points; int p_s0, p_s1, p_s2; int p_b;     // [1|B, V, 3]
    const float *matrix; int m_s0, m_s1, m_s2;              // [B, 4, 4]
    const float *dout; int d_s0, d_s1, d_s2;                // bwd: [B, V, 4|3]
    float *out;                                             // fwd: contiguous [B,V,4] (points) or [B,V,3] (vectors); bwd: [B,V,3]
    int B, V, is_points;
};

__global__ void __launch_bounds__(256) k_xfm_fwd(XfmParams p)
{
    __shared__ float m[4][4];       // m[r][c] = matrix[b][r][c]
    const int b = blockIdx.y;
    if (threadIdx.x < 16) m[threadIdx.x / 4][threadIdx.x % 4] = __ldg(p.matrix + (int64_t)b * p.m_s0 + (threadIdx.x / 4) * p.m_s1 + (threadIdx.x % 4) * p.m_s2);
    __syncthreads();
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= p.V) return;
    const float *q = p.points + (int64_t)(p.p_b == 1 ? 0 : b) * p.p_s0 + (int64_t)v * p.p_s1;
    const float x = __ldg(q), y = __ldg(q + p.p_s2), z = __ldg(q + 2 * p.p_s2);
    // out = [x y z w] * M^T  (ops.py:515: matmul(pad(points), transpose(matrix)))
    if (p.is_points) {
        float4 o;
        o.x = x * m[0][0] + y * m[0][1] + z * m[0][2] + m[0][3];
        o.y = x * m[1][0] + y * m[1][1] + z * m[1][2] + m[1][3];
        o.z = x * m[2][0] + y * m[2][1] + z * m[2][2] + m[2][3];
        o.w = x * m[3][0] + y * m[3][1] + z * m[3][2] + m[3][3];
        reinterpret_cast<float4 *>(p.out)[(int64_t)b * p.V + v] = o;
    } else {
        float *o = p.out + ((int64_t)b * p.V + v) * 3;
        o[0] = x * m[0][0] + y * m[0][1] + z * m[0][2];
        o[1] = x * m[1][0] + y * m[1][1] + z * m[1][2];
        o[2] = x * m[2][0] + y * m[2][1] + z * m[2][2];
    }
}

__global__ void __launch_bounds__(256) k_xfm_bwd(XfmParams p)
{
    __shared__ float m[4][4];
    const int b = blockIdx.y;
    if (threadIdx.x < 16) m[threadIdx.x / 4][threadIdx.x % 4] = __ldg(p.matrix + (int64_t)b * p.m_s0 + (threadIdx.x / 4) * p.m_s1 + (threadIdx.x % 4) * p.m_s2);
    __syncthreads();
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= p.V) return;
    const float *g = p.dout + (int64_t)b * p.d_s0 + (int64_t)v * p.d_s1;
    const float gx = __ldg(g), gy = __ldg(g + p.d_s2), gz = __ldg(g + 2 * p.d_s2), gw = p.is_points ? __ldg(g + 3 * p.d_s2) : 0.0f;
    float *o = p.out + ((int64_t)b * p.V + v) * 3;                   // full-batch gradient; a broadcast input is reduced by the caller
    o[0] = gx * m[0][0] + gy * m[1][0] + gz * m[2][0] + gw * m[3][0];
    o[1] = gx * m[0][1] + gy * m[1][1] + gz * m[2][1] + gw * m[3][1];
    o[2] = gx * m[0][2] + gy * m[1][2] + gz * m[2][2] + gw * m[3][2];
}

static int loss_common(LossParams &p, const mcs_tensor *img, const mcs_tensor *target, int32_t loss, int32_t tonemapper)
{
    MCS_REQUIRE(view_ok(img) && view_ok(target), "image_loss: null / empty tensor argument");
    MCS_REQUIRE((img->sizes[3] == 3 || img->sizes[3] == 1) && (target->sizes[3] == 3 || target->sizes[3] == 1), "image_loss: img/target must have 3 channels");
    MCS_REQUIRE(loss >= 0 && loss <= 4, "image_loss: unknown loss id %d (0 l1, 1 mse, 2 relmse, 3 smape, 4 n2n)", loss);
    p.N = img->sizes[0] > target->sizes[0] ? img->sizes[0] : target->sizes[0];
    p.H = img->sizes[1] > target->sizes[1] ? img->sizes[1] : target->sizes[1];
    p.W = img->sizes[2] > target->sizes[2] ? img->sizes[2] : target->sizes[2];
    for (int d = 0; d < 3; ++d) {
        const int full = d == 0 ? p.N : (d == 1 ? p.H : p.W);
        MCS_REQUIRE((img->sizes[d] == full || img->sizes[d] == 1) && (target->sizes[d] == full || target->sizes[d] == 1), "image_loss: shapes are not broadcastable");
    }
    p.npx = (int64_t)p.N * p.H * p.W;
    p.img = make_view(img); p.tgt = make_view(target);
    p.loss = loss; p.tonemap = tonemapper;
    return 0;
}

static bool dense_rgba(const mcs_tensor *t)
{
    const int32_t *sz = t->sizes, *st = t->strides;
    return ((uintptr_t)t->ptr & 15) == 0 && st[3] == 1 && (sz[2] == 1 || st[2] == 4) && (sz[1] == 1 || st[1] == 4 * sz[2]) &&
           (sz[0] == 1 || (int64_t)st[0] == 4 * (int64_t)sz[1] * sz[2]);
}

static int coverage_common(const char *fn, CoverageParams &p, const mcs_tensor *img, const mcs_tensor *ref, int32_t loss, int32_t tonemapper)
{
    MCS_REQUIRE(loss >= 0 && loss <= 4, "%s: unknown loss id %d (0 l1, 1 mse, 2 relmse, 3 smape, 4 n2n)", fn, loss);
    MCS_REQUIRE(tonemapper == 0 || tonemapper == 1, "%s: unknown tonemapper id %d (0 none, 1 log_srgb)", fn, tonemapper);
    const mcs_tensor *v[2] = {img, ref};
    const char *names[2] = {"img", "ref"};
    for (int i = 0; i < 2; ++i) {
        MCS_REQUIRE(v[i] && v[i]->ptr, "%s: %s is null", fn, names[i]);
        MCS_REQUIRE(v[i]->sizes[3] == 4, "%s: %s must have 4 channels, got %d", fn, names[i], v[i]->sizes[3]);
        for (int d = 0; d < 3; ++d) MCS_REQUIRE(v[i]->sizes[d] == img->sizes[d], "%s: ref must have the shape of img", fn);
        for (int d = 0; d < 4; ++d) MCS_REQUIRE(v[i]->strides[d] >= 0, "%s: %s has a negative stride", fn, names[i]);
    }
    MCS_REQUIRE(img->sizes[0] > 0 && img->sizes[1] > 0 && img->sizes[2] > 0, "%s: empty operands", fn);
    p.npx = (int64_t)img->sizes[0] * img->sizes[1] * img->sizes[2];
    MCS_REQUIRE(p.npx < (int64_t)1 << 31, "%s: %lld pixels, at most 2^31 - 1", fn, (long long)p.npx);
    p.H = img->sizes[1]; p.W = img->sizes[2];
    p.img = make_view(img); p.ref = make_view(ref);
    p.img_vec = dense_rgba(img); p.ref_vec = dense_rgba(ref);
    p.loss = loss; p.tonemap = tonemapper;
    return 0;
}

}  // namespace

extern "C" {

int mcs_image_loss_num_partials(int32_t N, int32_t H, int32_t W) { return (int)(((int64_t)N * H * W + LOSS_BLOCK - 1) / LOSS_BLOCK); }

int mcs_image_loss_fwd(const mcs_tensor *img, const mcs_tensor *target, int32_t loss, int32_t tonemapper, float *partials, mcs_stream s)
{
    LossParams p{};
    if (int e = loss_common(p, img, target, loss, tonemapper)) return e;
    MCS_REQUIRE(partials != nullptr, "image_loss_fwd: null output");
    p.partial = partials;
    const int nb = mcs_image_loss_num_partials(p.N, p.H, p.W);
    k_image_loss_fwd<<<nb, LOSS_BLOCK, 0, (cudaStream_t)s>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_image_loss_bwd(const mcs_tensor *img, const mcs_tensor *target, int32_t loss, int32_t tonemapper, const mcs_tensor *d_partials,
                       float *d_img, float *d_target, mcs_stream s)
{
    LossParams p{};
    if (int e = loss_common(p, img, target, loss, tonemapper)) return e;
    MCS_REQUIRE(view_ok(d_partials) && d_img && d_target, "image_loss_bwd: null argument");
    const int nb = mcs_image_loss_num_partials(p.N, p.H, p.W);
    MCS_REQUIRE(d_partials->sizes[0] == nb || d_partials->sizes[0] == 1, "image_loss_bwd: gradient must have one value per partial sum (%d)", nb);
    p.dout = make_view(d_partials); p.dout_n = d_partials->sizes[0];
    p.d_img = d_img; p.d_tgt = d_target;
    k_image_loss_bwd<<<nb, LOSS_BLOCK, 0, (cudaStream_t)s>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_coverage_loss_num_partials(int32_t B, int32_t H, int32_t W) { return mcs_image_loss_num_partials(B, H, W); }

int mcs_coverage_loss_fwd(const mcs_tensor *img, const mcs_tensor *ref, int32_t loss, int32_t tonemapper, float *partials, float *loss_out,
                          mcs_stream s)
{
    CoverageParams p{};
    if (int e = coverage_common("coverage_loss_fwd", p, img, ref, loss, tonemapper)) return e;
    MCS_REQUIRE(partials && loss_out, "coverage_loss_fwd: null output pointer");
    p.partial = partials;
    const int nb = mcs_coverage_loss_num_partials(img->sizes[0], p.H, p.W);
    k_coverage_loss_fwd<<<nb, LOSS_BLOCK, 0, (cudaStream_t)s>>>(p);
    MCS_LAUNCH_CHECK();
    k_coverage_loss_finish<<<1, LOSS_BLOCK, 0, (cudaStream_t)s>>>(partials, nb, p.npx, loss_out);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_coverage_loss_bwd(const mcs_tensor *img, const mcs_tensor *ref, int32_t loss, int32_t tonemapper, const float *d_loss, float *d_img,
                          mcs_stream s)
{
    CoverageParams p{};
    if (int e = coverage_common("coverage_loss_bwd", p, img, ref, loss, tonemapper)) return e;
    MCS_REQUIRE(d_loss && d_img, "coverage_loss_bwd: null pointer argument");
    MCS_REQUIRE(((uintptr_t)d_img & 15) == 0, "coverage_loss_bwd: d_img must be 16-byte aligned");
    p.d_loss = d_loss; p.d_img = d_img;
    p.inv_npx = 1.0f / (float)p.npx;
    p.two_over_npx = (float)(2.0 / (double)p.npx);
    k_coverage_loss_bwd<<<mcs_coverage_loss_num_partials(img->sizes[0], p.H, p.W), LOSS_BLOCK, 0, (cudaStream_t)s>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

static int xfm_common(XfmParams &p, const mcs_tensor *points, const mcs_tensor *matrix)
{
    MCS_REQUIRE(view_ok(points) && view_ok(matrix), "xfm: null / empty tensor argument");
    // points: sizes (1|B, V, 3, 1); matrix: (B, 4, 4, 1)
    MCS_REQUIRE(points->sizes[2] == 3 && matrix->sizes[1] == 4 && matrix->sizes[2] == 4, "xfm: points must be [1|B,V,3] and matrix [B,4,4]");
    MCS_REQUIRE(points->sizes[0] == 1 || points->sizes[0] == matrix->sizes[0], "xfm: points batch must be 1 or match the matrix batch");
    p.points = (const float *)points->ptr; p.p_s0 = points->strides[0]; p.p_s1 = points->strides[1]; p.p_s2 = points->strides[2]; p.p_b = points->sizes[0];
    p.matrix = (const float *)matrix->ptr; p.m_s0 = matrix->strides[0]; p.m_s1 = matrix->strides[1]; p.m_s2 = matrix->strides[2];
    p.B = matrix->sizes[0]; p.V = points->sizes[1];
    MCS_REQUIRE(p.B <= 65535, "xfm: batch too large");
    return 0;
}

int mcs_xfm_fwd(const mcs_tensor *points, const mcs_tensor *matrix, int32_t is_points, float *out, mcs_stream s)
{
    XfmParams p{};
    if (int e = xfm_common(p, points, matrix)) return e;
    MCS_REQUIRE(out != nullptr, "xfm_fwd: null output");
    p.out = out; p.is_points = is_points;
    k_xfm_fwd<<<dim3((p.V + 255) / 256, p.B), 256, 0, (cudaStream_t)s>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_xfm_bwd(const mcs_tensor *points, const mcs_tensor *matrix, const mcs_tensor *d_out, int32_t is_points, float *d_points, mcs_stream s)
{
    XfmParams p{};
    if (int e = xfm_common(p, points, matrix)) return e;
    MCS_REQUIRE(view_ok(d_out) && d_points, "xfm_bwd: null argument");
    MCS_REQUIRE(d_out->sizes[0] == p.B && d_out->sizes[1] == p.V && d_out->sizes[2] == (is_points ? 4 : 3), "xfm_bwd: upstream gradient shape mismatch");
    p.dout = (const float *)d_out->ptr; p.d_s0 = d_out->strides[0]; p.d_s1 = d_out->strides[1]; p.d_s2 = d_out->strides[2];
    p.out = d_points; p.is_points = is_points;
    k_xfm_bwd<<<dim3((p.V + 255) / 256, p.B), 256, 0, (cudaStream_t)s>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
