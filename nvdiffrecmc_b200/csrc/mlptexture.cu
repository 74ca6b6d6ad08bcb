// mlptexture.cu -- the reference's MLPTexture3D.sample (render/mlptexture.py:86-96) as one forward and one backward kernel: AABB
// normalisation, clamp, the hash-grid encoding of hashgrid.cu (16 levels -> 32 features), a bias-free MLP of `hidden` (1..4) ReLU
// layers of width 32 and an output layer of C (1..8) channels, sigmoid scaled into min_max.  Semantics (the contract; the CPU oracle
// oracle/mlptexture.c restates it), per point t [3], with aabb [2,3] and min_max [2,C] read from device memory:
//   xn_d = (t_d - a0_d) / (a1_d - a0_d);  x_d = 0 if xn_d < 0, 1 if xn_d > 1, else xn_d (NaN stays NaN, as torch.clamp);
//   e [32] = the encoding of x (hashgrid.cu's contract, bit for bit);
//   layer l < hidden: h_j = relu(sum over k ascending of W_l[j,k] * in_k), in = e for l = 0, relu(a) = 0 if a <= 0 else a;
//   output: z_c = sum over k ascending of W_hidden[c,k] * h_k;  s = 1 / (1 + exp(-z));  out_c = s * (hi_c - lo_c) + lo_c.
//   Every sum over k is an fmaf chain from +0 (acc = fmaf(W, in, acc)); every other operation is one IEEE round-to-nearest operation in
//   the order written, never contracted.  W_l is torch's Linear.weight [out, in], row-major.
//   exp is mt_exp below (Cephes expf's range reduction and polynomial, within 2 ulp of exp; NaN -> NaN, x > 88.72283935546875 -> +inf,
//   x < -103.27892990343185 -> 0; 2^n is applied as two normal powers of two so that only the last product rounds).
// Adjoints (g = d out [C]):
//   dz_c = (g_c * (hi_c - lo_c)) * ((1 - s_c) * s_c);  d h_k = sum over c ascending of dz_c * W_hidden[c,k] (fmaf chain from +0), then
//   for each hidden layer from the top: d pre_j = d h_j if h_j > 0 else 0, d in_k = sum over j ascending of d pre_j * W_l[j,k] (fmaf
//   chain from +0); d e = d in of layer 0.
//   d W (deterministic, independent of the launch shape): the points are split into chunks of MCS_MLPTEX_CHUNK consecutive points; the
//   chunk partial of W_l[j,k] is an fmaf chain from +0 over the chunk's points ascending, of d pre_j * in_k (dz_c * h_k for the output
//   layer); d W = the partials summed from +0 in ascending chunk order.
//   d params, d x (of the clamped x) = hashgrid.cu's adjoints of d e (float atomics for d params, grouped on the dense levels; the
//   deterministic ascending-level sum for d x; a level whose two gradients are exactly zero is skipped by both);
//   d t_d = (0 <= xn_d <= 1 ? d x_d : 0) / (a1_d - a0_d).  aabb and min_max get no gradient.
// Every index is reduced modulo its level's size, so every access stays in bounds for every input; NaN inputs give NaN outputs.
// The pair (render.py:63-64's two samples of every pixel; the kernels' kPair instances): per pixel i the plain point t_i and the
// jittered point __fadd_rn(t_i, off_i), each evaluated exactly as above (out / enc and out_jit / enc_jit); d t = fl(d_plain + d_jit),
// d off = d_jit; d W keeps one chunk-partial set per kind of point, each summed in chunk order as above, then d W = fl(d W plain +
// d W jit); d params takes both points' atomics.  So everything but d params equals two single calls and autograd's sums bit for bit.
#include "hashgrid.cuh"

namespace {

constexpr int kThreads = 128;                       // one thread per point; the backward walks its chunk in sub-batches of kThreads
constexpr int kChunk = MCS_MLPTEX_CHUNK;
constexpr int kStride = kThreads + 1;               // feature-major sub-batch rows [32][kThreads + 1]: conflict-free both ways
static_assert(kChunk % kThreads == 0, "a chunk is a whole number of sub-batches");

struct MtArgs {
    const float *t;            // [n,3]
    int64_t n;
    const float *aabb;         // [2,3]
    const float *mm;           // [2,C]
    const float2 *params;
    mcs_hashgrid_levels lv;
    const float *w[5];         // layer l < hidden: [32,32]; layer hidden: [C,32]
    int hidden, C;
    float *out;                // [n,C]
    float *enc;                // [n,32]: written by the forward when non-null, read by the backward
    const float *dout;         // [n,C]
    float2 *dparams;
    float *dt;                 // [n,3]
    float *ws;                 // [chunks, n_weights] chunk partials of d W (null: no d W); the pair: [2, chunks, n_weights]
    // the pair (the jittered point of pixel i is t_i + off_i): its output, saved encoding and upstream gradient, and d off
    const float *off;          // [n,3]
    float *out_jit;            // [n,C]
    float *enc_jit;            // [n,32]
    const float *dout_jit;     // [n,C] (pair backward: either dout may be null, meaning zero)
    float *doff;               // [n,3] (null: not requested)
};

__host__ __device__ __forceinline__ int mt_n_weights(int hidden, int C) { return hidden * 1024 + C * 32; }

__device__ __forceinline__ float mt_exp(float x)
{
    if (x != x) return x;
    if (x > 88.72283935546875f) return INFINITY;
    if (x < -103.27892990343185f) return 0.0f;
    const float z = floorf(__fadd_rn(__fmul_rn(1.44269504088896341f, x), 0.5f));
    const int n = (int)z;
    float r = __fsub_rn(x, __fmul_rn(z, 0.693359375f));
    r = __fsub_rn(r, __fmul_rn(z, -2.12194440e-4f));
    const float rr = __fmul_rn(r, r);
    float p = 1.9875691500e-4f;
    p = __fadd_rn(__fmul_rn(p, r), 1.3981999507e-3f);
    p = __fadd_rn(__fmul_rn(p, r), 8.3334519073e-3f);
    p = __fadd_rn(__fmul_rn(p, r), 4.1665795894e-2f);
    p = __fadd_rn(__fmul_rn(p, r), 1.6666665459e-1f);
    p = __fadd_rn(__fmul_rn(p, r), 5.0000001201e-1f);
    p = __fadd_rn(__fadd_rn(__fmul_rn(p, rr), r), 1.0f);
    const int n1 = n / 2, n2 = n - n1;
    return __fmul_rn(__fmul_rn(p, __int_as_float((n1 + 127) << 23)), __int_as_float((n2 + 127) << 23));
}

// weights of every layer into shared memory, layer l at l * 1024 (read as broadcasts)
__device__ __forceinline__ void mt_load_weights(const MtArgs &a, float *sw)
{
    const int nW = mt_n_weights(a.hidden, a.C);
    for (int e = threadIdx.x; e < nW; e += blockDim.x) {
        const int l = min(e >> 10, a.hidden);
        sw[e] = a.w[l][e - l * 1024];
    }
}

// normalised (xn) and clamped (x) point: t_i, or with jit the jittered point t_i + off_i (one fp32 add per component, as torch's)
__device__ __forceinline__ void mt_point(const MtArgs &a, int64_t i, bool jit, float xn[3], float x[3])
{
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float a0 = __ldg(a.aabb + d), a1 = __ldg(a.aabb + 3 + d);
        float td = __ldg(a.t + 3 * i + d);
        if (jit) td = __fadd_rn(td, __ldg(a.off + 3 * i + d));
        xn[d] = __fdiv_rn(__fsub_rn(td, a0), __fsub_rn(a1, a0));
        x[d] = xn[d] < 0.0f ? 0.0f : (xn[d] > 1.0f ? 1.0f : xn[d]);
    }
}

__device__ __forceinline__ void mt_encode(const MtArgs &a, const float x[3], float e[32])
{
#pragma unroll
    for (int l = 0; l < 16; ++l) {
        const uint32_t off = a.lv.offset[l], size = a.lv.offset[l + 1] - off, res = a.lv.res[l];
        const bool dense = (a.lv.dense_mask >> l) & 1u;
        const Cell cl = hg_cell(a.lv.scale[l], x);
        float y0 = 0.0f, y1 = 0.0f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float w1[3];
            hg_weights(cl, c, w1);
            const float w = __fmul_rn(__fmul_rn(w1[0], w1[1]), w1[2]);
            const float2 v = __ldg(a.params + off + hg_index(cl, c, dense, res, size));
            y0 = __fadd_rn(y0, __fmul_rn(w, v.x));
            y1 = __fadd_rn(y1, __fmul_rn(w, v.y));
        }
        e[2 * l] = y0;
        e[2 * l + 1] = y1;
    }
}

__device__ __forceinline__ float mt_dot32(const float *W, const float v[32])
{
    float acc = 0.0f;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const float4 w = reinterpret_cast<const float4 *>(W)[q];
        acc = fmaf(w.x, v[4 * q], acc);
        acc = fmaf(w.y, v[4 * q + 1], acc);
        acc = fmaf(w.z, v[4 * q + 2], acc);
        acc = fmaf(w.w, v[4 * q + 3], acc);
    }
    return acc;
}

// one hidden layer in place: v <- relu(W v)
__device__ __forceinline__ void mt_hidden(const float *W, float v[32])
{
    float h[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const float acc = mt_dot32(W + 32 * j, v);
        h[j] = acc <= 0.0f ? 0.0f : acc;
    }
#pragma unroll
    for (int k = 0; k < 32; ++k) v[k] = h[k];
}

// sigmoid of z: s
__device__ __forceinline__ float mt_sigmoid(float z) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, mt_exp(-z))); }

// the forward of one point (jit: the jittered point of pixel i) into out [n,C] and, when non-null, enc [n,32]
__device__ __forceinline__ void mt_fwd_point(const MtArgs &a, const float *sw, int64_t i, bool jit, float *out, float *enc)
{
    float xn[3], x[3], v[32];
    mt_point(a, i, jit, xn, x);
    mt_encode(a, x, v);
    if (enc) {
        float4 *e4 = reinterpret_cast<float4 *>(enc + 32 * i);
#pragma unroll
        for (int q = 0; q < 8; ++q) e4[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    }
    for (int l = 0; l < a.hidden; ++l) mt_hidden(sw + 1024 * l, v);
    const float *Wo = sw + 1024 * a.hidden;
    for (int c = 0; c < a.C; ++c) {
        const float s = mt_sigmoid(mt_dot32(Wo + 32 * c, v));
        const float lo = __ldg(a.mm + c), hi = __ldg(a.mm + a.C + c);
        out[i * a.C + c] = __fadd_rn(__fmul_rn(s, __fsub_rn(hi, lo)), lo);
    }
}

// kPair: thread 2i evaluates pixel i's plain point and thread 2i + 1 its jittered one, so the two points' coarse-level gathers (the same
// cells, within N(0, 0.01) of each other) are issued by one warp instruction.  (One thread evaluating both points back to back was
// slower than two launches: 3.57 against 2.26 ms at 8 x 512^2, H100 80GB HBM3 at 700 W.)
template <bool kPair>
__global__ void __launch_bounds__(kThreads) k_mlptex_fwd(const MtArgs a)
{
    extern __shared__ float4 smem[];
    float *sw = reinterpret_cast<float *>(smem);
    mt_load_weights(a, sw);
    __syncthreads();
    const int64_t k = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    const int64_t i = kPair ? k >> 1 : k;
    if (i >= a.n) return;
    const bool jit = kPair && (k & 1);
    mt_fwd_point(a, sw, i, jit, jit ? a.out_jit : a.out, jit ? a.enc_jit : a.enc);
}

// One pass of the backward over a sub-batch (point i = base + threadIdx.x, live when in; cnt live points) -- the plain points (jit false)
// or, in the pair, the jittered ones -- extending the d W chunk partials sp:
//   1. the hidden activations are recomputed from the saved encoding and kept feature-major in shared memory (act[l] = input of layer l);
//   2. the MLP's backward runs per thread, top layer first; before each layer's input gradient, the block extends the chunk partials of
//      that layer's d W over the sub-batch (thread t owns 8 consecutive weights of each 32 x 32 layer and 2 of the output layer; the
//      partials stay in shared memory across sub-batches);
//   3. d e goes to shared memory, and each thread runs the hash-grid adjoints of its point, point-major over the levels.
// With want_t, d t of a live point goes to a.dt, or in the pair to gt.  kPair: dout may be null (zero).
template <bool kPair>
__device__ __forceinline__ void mt_bwd_pass(const MtArgs &a, bool jit, const float *sw, float *sp, float *dp, float *act, int64_t i, bool in,
                                            int cnt, bool want_t, float gt[3])
{
    const int H = a.hidden, C = a.C, nW = mt_n_weights(H, C);
    const bool want_dw = a.ws != nullptr;
    const int t = threadIdx.x;
    const float *Wo = sw + 1024 * H;
    const float *enc = jit ? a.enc_jit : a.enc, *dout = jit ? a.dout_jit : a.dout;
    __syncthreads();                                                                // weights loaded; previous pass done with act
    float v[32];
    if (in) {
        const float4 *e4 = reinterpret_cast<const float4 *>(enc + 32 * i);
#pragma unroll
        for (int q = 0; q < 8; ++q) { const float4 e = e4[q]; v[4 * q] = e.x; v[4 * q + 1] = e.y; v[4 * q + 2] = e.z; v[4 * q + 3] = e.w; }
    } else {
#pragma unroll
        for (int k = 0; k < 32; ++k) v[k] = 0.0f;
    }
#pragma unroll
    for (int k = 0; k < 32; ++k) act[k * kStride + t] = v[k];
    for (int l = 0; l < H; ++l) {
        mt_hidden(sw + 1024 * l, v);
#pragma unroll
        for (int k = 0; k < 32; ++k) act[((l + 1) * 32 + k) * kStride + t] = v[k];
    }
    // output layer: dz, and d h = W_out^T dz
    float dh[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) dh[k] = 0.0f;
    for (int c = 0; c < C; ++c) {
        float dz = 0.0f;
        if (in) {
            const float s = mt_sigmoid(mt_dot32(Wo + 32 * c, v));
            const float lo = __ldg(a.mm + c), hi = __ldg(a.mm + C + c);
            const float gs = __fmul_rn((!kPair || dout) ? __ldg(dout + i * C + c) : 0.0f, __fsub_rn(hi, lo));
            dz = __fmul_rn(gs, __fmul_rn(__fsub_rn(1.0f, s), s));
        }
        dp[c * kStride + t] = dz;
        const float4 *r = reinterpret_cast<const float4 *>(Wo + 32 * c);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float4 w = r[q];
            dh[4 * q] = fmaf(dz, w.x, dh[4 * q]);
            dh[4 * q + 1] = fmaf(dz, w.y, dh[4 * q + 1]);
            dh[4 * q + 2] = fmaf(dz, w.z, dh[4 * q + 2]);
            dh[4 * q + 3] = fmaf(dz, w.w, dh[4 * q + 3]);
        }
    }
    __syncthreads();
    if (want_dw) {
        for (int w = H * 1024 + t; w < nW; w += kThreads) {
            const int c = (w - H * 1024) >> 5, k = w & 31;
            const float *pa = act + (H * 32 + k) * kStride, *pd = dp + c * kStride;
            float p = sp[w];
            for (int ii = 0; ii < cnt; ++ii) p = fmaf(pd[ii], pa[ii], p);
            sp[w] = p;
        }
    }
    // hidden layers, top first: dh -> d pre (ReLU mask of the layer's output) -> d W partials -> d of the layer's input
#pragma unroll
    for (int k = 0; k < 32; ++k) dh[k] = v[k] > 0.0f ? dh[k] : 0.0f;
    for (int l = H - 1; l >= 0; --l) {
        __syncthreads();                                                            // everyone done reading dp
#pragma unroll
        for (int k = 0; k < 32; ++k) dp[k * kStride + t] = dh[k];
        __syncthreads();
        if (want_dw) {
            const int j = t >> 2, k0 = (t & 3) * 8;
            float *ps = sp + l * 1024 + 8 * t;                                      // = W_l[j, k0 .. k0 + 7]
            float p[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) p[q] = ps[q];
            const float *pd = dp + j * kStride, *pa = act + (l * 32 + k0) * kStride;
            for (int ii = 0; ii < cnt; ++ii) {
                const float d = pd[ii];
#pragma unroll
                for (int q = 0; q < 8; ++q) p[q] = fmaf(d, pa[q * kStride + ii], p[q]);
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) ps[q] = p[q];
        }
        float dv[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) dv[k] = 0.0f;
        const float *W = sw + 1024 * l;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const float4 *r = reinterpret_cast<const float4 *>(W + 32 * j);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 w = r[q];
                dv[4 * q] = fmaf(dh[j], w.x, dv[4 * q]);
                dv[4 * q + 1] = fmaf(dh[j], w.y, dv[4 * q + 1]);
                dv[4 * q + 2] = fmaf(dh[j], w.z, dv[4 * q + 2]);
                dv[4 * q + 3] = fmaf(dh[j], w.w, dv[4 * q + 3]);
            }
        }
        if (l > 0) {
#pragma unroll
            for (int k = 0; k < 32; ++k) dh[k] = act[(l * 32 + k) * kStride + t] > 0.0f ? dv[k] : 0.0f;
        } else {
#pragma unroll
            for (int k = 0; k < 32; ++k) dh[k] = dv[k];
        }
    }
    if (!a.dparams && !want_t) return;
    __syncthreads();                                                                // d W readers done with dp
#pragma unroll
    for (int k = 0; k < 32; ++k) dp[k * kStride + t] = dh[k];                     // d e; each thread reads back its own column
    float xn[3] = {0.0f, 0.0f, 0.0f}, x[3] = {0.0f, 0.0f, 0.0f}, dx[3] = {0.0f, 0.0f, 0.0f};
    if (in) mt_point(a, i, jit, xn, x);
    for (int l = 0; l < 16; ++l) {
        const uint32_t off = a.lv.offset[l], size = a.lv.offset[l + 1] - off, res = a.lv.res[l];
        const bool dense = (a.lv.dense_mask >> l) & 1u;
        const float s = a.lv.scale[l];
        const Cell cl = hg_cell(s, x);
        const float2 dy = make_float2(dp[2 * l * kStride + t], dp[(2 * l + 1) * kStride + t]);
        const bool live = in && (dy.x != 0.0f || dy.y != 0.0f);
        if (a.dparams && (dense || live)) {
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float w1[3];
                hg_weights(cl, c, w1);
                const float w = __fmul_rn(__fmul_rn(w1[0], w1[1]), w1[2]);
                hg_scatter(a.dparams + off, hg_index(cl, c, dense, res, size), make_float2(__fmul_rn(w, dy.x), __fmul_rn(w, dy.y)), live,
                           dense);
            }
        }
        if (want_t && live) {
            float ad[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float w1[3];
                hg_weights(cl, c, w1);
                const float2 pv = __ldg(a.params + off + hg_index(cl, c, dense, res, size));
                const float sc = __fadd_rn(__fmul_rn(dy.x, pv.x), __fmul_rn(dy.y, pv.y));
                const float dw[3] = {__fmul_rn(w1[1], w1[2]), __fmul_rn(w1[0], w1[2]), __fmul_rn(w1[0], w1[1])};
#pragma unroll
                for (int d = 0; d < 3; ++d) ad[d] = __fadd_rn(ad[d], __fmul_rn(((c >> d) & 1) ? dw[d] : -dw[d], sc));
            }
#pragma unroll
            for (int d = 0; d < 3; ++d) dx[d] = __fadd_rn(dx[d], __fmul_rn(s, ad[d]));
        }
    }
    if (want_t && in) {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float g = (xn[d] >= 0.0f && xn[d] <= 1.0f) ? dx[d] : 0.0f;
            const float v = __fdiv_rn(g, __fsub_rn(__ldg(a.aabb + 3 + d), __ldg(a.aabb + d)));
            if (kPair) gt[d] = v;
            else a.dt[3 * i + d] = v;
        }
    }
}

// One block per chunk of kChunk points (the pair: pixels), walked in sub-batches of kThreads, one mt_bwd_pass per sub-batch (the pair:
// the plain points, then the jittered ones, each set with its own chunk partials; a thread holds its pixel's plain d t in registers until
// the jittered one is done).  The chunk partials are written to the workspace at the end; k_mlptex_dw_sum adds them in chunk order.
template <bool kPair>
__global__ void __launch_bounds__(kThreads) k_mlptex_bwd(const MtArgs a)
{
    extern __shared__ float4 smem[];
    const int nW = mt_n_weights(a.hidden, a.C), nW4 = (nW + 3) & ~3;
    float *sw = reinterpret_cast<float *>(smem);            // [nW4] weights
    float *sp = sw + nW4;                                   // [1 + kPair][nW4] chunk partials of d W (plain, jittered)
    float *dp = sp + (kPair ? 2 : 1) * nW4;                 // [32][kStride] d pre of the current layer, then d e
    float *act = dp + 32 * kStride;                         // [H + 1][32][kStride] layer inputs
    mt_load_weights(a, sw);
    for (int e = threadIdx.x; e < (kPair ? nW4 + nW : nW); e += kThreads) sp[e] = 0.0f;
    const int t = threadIdx.x;
    for (int sb = 0; sb < kChunk / kThreads; ++sb) {
        const int64_t base = (int64_t)blockIdx.x * kChunk + (int64_t)sb * kThreads;
        if (base >= a.n) break;                                                     // block-uniform
        const int cnt = (int)min((int64_t)kThreads, a.n - base);
        const int64_t i = base + t;
        const bool in = t < cnt;
        float g[3];
        mt_bwd_pass<kPair>(a, false, sw, sp, dp, act, i, in, cnt, a.dt != nullptr, g);
        if (kPair) {
            float gj[3];
            mt_bwd_pass<kPair>(a, true, sw, sp + nW4, dp, act, i, in, cnt, a.dt || a.doff, gj);
            if (in && a.dt)
#pragma unroll
                for (int d = 0; d < 3; ++d) a.dt[3 * i + d] = __fadd_rn(g[d], gj[d]);
            if (in && a.doff)
#pragma unroll
                for (int d = 0; d < 3; ++d) a.doff[3 * i + d] = gj[d];
        }
    }
    if (a.ws) {
        __syncthreads();
        float *wsb = a.ws + (int64_t)blockIdx.x * nW;
        for (int e = t; e < nW; e += kThreads) wsb[e] = sp[e];
        if (kPair) {
            wsb += (int64_t)gridDim.x * nW;
            for (int e = t; e < nW; e += kThreads) wsb[e] = sp[nW4 + e];
        }
    }
}

struct DwOut { float *d[5]; };

// sum from +0 in ascending chunk order of the chunk partials ws [chunks, nW] of weight e
__device__ __forceinline__ float mt_chunk_sum(const float *ws, int64_t chunks, int nW, int e)
{
    float s = 0.0f;
    int64_t ch = 0;
    for (; ch + 8 <= chunks; ch += 8) {
        float p[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) p[q] = __ldg(ws + (ch + q) * nW + e);
#pragma unroll
        for (int q = 0; q < 8; ++q) s = __fadd_rn(s, p[q]);
    }
    for (; ch < chunks; ++ch) s = __fadd_rn(s, __ldg(ws + ch * nW + e));
    return s;
}

// d W = the chunk partials summed from +0 in ascending chunk order (the pair: each set so, then plain + jittered); one thread per weight
// (consecutive threads read consecutive weights)
template <bool kPair>
__global__ void __launch_bounds__(128) k_mlptex_dw_sum(const float *ws, int64_t chunks, int hidden, int C, DwOut o)
{
    const int nW = mt_n_weights(hidden, C);
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nW) return;
    float s = mt_chunk_sum(ws, chunks, nW, e);
    if (kPair) s = __fadd_rn(s, mt_chunk_sum(ws + chunks * nW, chunks, nW, e));
    const int l = min(e >> 10, hidden);
    if (o.d[l]) o.d[l][e - l * 1024] = s;
}

size_t mt_bwd_smem(int hidden, int C, bool pair)
{
    const int nW4 = (mt_n_weights(hidden, C) + 3) & ~3;
    return sizeof(float) * ((size_t)(pair ? 3 : 2) * nW4 + (size_t)(hidden + 2) * 32 * kStride);
}

int mt_validate(const char *fn, const float *t, int64_t n, const float *aabb, const float *min_max, const float *params,
                const mcs_hashgrid_levels *lv, int32_t hidden, int32_t C, const float *const *weights)
{
    MCS_REQUIRE(t && aabb && min_max && params && lv && weights, "%s: null pointer", fn);
    MCS_REQUIRE(n >= 0, "%s: n must be >= 0 (got %lld)", fn, (long long)n);
    MCS_REQUIRE(n <= (int64_t)INT32_MAX * kThreads, "%s: n too large", fn);
    MCS_REQUIRE(hidden >= 1 && hidden <= 4, "%s: hidden must be in 1..4 (got %d)", fn, hidden);
    MCS_REQUIRE(C >= 1 && C <= 8, "%s: channels must be in 1..8 (got %d)", fn, C);
    MCS_REQUIRE(lv->n_levels == 16, "%s: the encoding must have 16 levels (32 features; got %d)", fn, lv->n_levels);
    MCS_REQUIRE(((uintptr_t)params & 7) == 0, "%s: params must be 8-byte aligned", fn);
    for (int l = 0; l <= hidden; ++l) MCS_REQUIRE(weights[l] != nullptr, "%s: null pointer (weights[%d])", fn, l);
    for (int l = 0; l <= 16; ++l) {
        MCS_REQUIRE(lv->offset[l] % 8 == 0, "%s: offset[%d] = %u is not a multiple of 8", fn, l, lv->offset[l]);
        if (l > 0) MCS_REQUIRE(lv->offset[l] > lv->offset[l - 1], "%s: offsets not increasing at level %d", fn, l - 1);
    }
    return 0;
}

MtArgs mt_args(const float *t, int64_t n, const float *aabb, const float *min_max, const float *params, const mcs_hashgrid_levels *lv,
               int32_t hidden, int32_t C, const float *const *weights)
{
    MtArgs a{};
    a.t = t; a.n = n; a.aabb = aabb; a.mm = min_max; a.params = (const float2 *)params; a.lv = *lv;
    for (int l = 0; l <= hidden; ++l) a.w[l] = weights[l];
    a.hidden = hidden; a.C = C;
    return a;
}

// the checks of a backward entry after mt_validate: -> 0, with want_dw set, or the error status
int mt_validate_bwd(const char *fn, int32_t hidden, const float *enc, bool want_grad, float *const *d_weights, bool *want_dw,
                    const float *d_params, const void *workspace)
{
    *want_dw = false;
    if (d_weights)
        for (int l = 0; l <= hidden; ++l) *want_dw |= d_weights[l] != nullptr;
    MCS_REQUIRE(want_grad || *want_dw, "%s: null pointer (no gradient requested)", fn);
    MCS_REQUIRE(!*want_dw || workspace, "%s: null pointer (workspace)", fn);
    MCS_REQUIRE(((uintptr_t)enc & 15) == 0 && ((uintptr_t)d_params & 7) == 0 && ((uintptr_t)workspace & 15) == 0,
                "%s: enc and workspace must be 16-byte aligned, d_params 8-byte aligned", fn);
    return 0;
}

template <bool kPair>
int mt_launch_fwd(const MtArgs &a, mcs_stream stream)
{
    if (a.n == 0) return 0;
    const size_t smem = sizeof(float) * mt_n_weights(a.hidden, a.C);
    const int64_t threads = kPair ? 2 * a.n : a.n;
    k_mlptex_fwd<kPair><<<(unsigned)((threads + kThreads - 1) / kThreads), kThreads, smem, (cudaStream_t)stream>>>(a);
    MCS_LAUNCH_CHECK();
    return 0;
}

template <bool kPair>
int mt_launch_bwd(const MtArgs &a, float *const *d_weights, mcs_stream stream)
{
    const int hidden = a.hidden, channels = a.C;
    const cudaStream_t s = (cudaStream_t)stream;
    if (a.n == 0) {
        if (a.ws)
            for (int l = 0; l <= hidden; ++l)
                if (d_weights[l]) MCS_CUDA(cudaMemsetAsync(d_weights[l], 0, sizeof(float) * (l < hidden ? 1024 : 32 * channels), s));
        return 0;
    }
    const size_t smem = mt_bwd_smem(hidden, channels, kPair);
    MCS_CUDA(cudaFuncSetAttribute(k_mlptex_bwd<kPair>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t chunks = (a.n + kChunk - 1) / kChunk;
    k_mlptex_bwd<kPair><<<(unsigned)chunks, kThreads, smem, s>>>(a);
    MCS_LAUNCH_CHECK();
    if (a.ws) {
        DwOut o{};
        for (int l = 0; l <= hidden; ++l) o.d[l] = d_weights[l];
        const int nW = mt_n_weights(hidden, channels);
        k_mlptex_dw_sum<kPair><<<(nW + 127) / 128, 128, 0, s>>>(a.ws, chunks, hidden, channels, o);
        MCS_LAUNCH_CHECK();
    }
    return 0;
}

}  // namespace

extern "C" {

int64_t mcs_mlptex_workspace_bytes(int64_t n, int32_t hidden, int32_t channels)
{
    if (n < 0 || hidden < 1 || hidden > 4 || channels < 1 || channels > 8) return -1;
    return (int64_t)sizeof(float) * ((n + kChunk - 1) / kChunk) * mt_n_weights(hidden, channels);
}

int mcs_mlptex_fwd(const float *t, int64_t n, const float *aabb, const float *min_max, const float *params, const mcs_hashgrid_levels *lv,
                   int32_t hidden, int32_t channels, const float *const *weights, float *out, float *enc, mcs_stream stream)
{
    if (int e = mt_validate("mcs_mlptex_fwd", t, n, aabb, min_max, params, lv, hidden, channels, weights)) return e;
    MCS_REQUIRE(out != nullptr, "mcs_mlptex_fwd: null pointer (out)");
    MCS_REQUIRE(((uintptr_t)enc & 15) == 0, "mcs_mlptex_fwd: enc must be 16-byte aligned");
    MtArgs a = mt_args(t, n, aabb, min_max, params, lv, hidden, channels, weights);
    a.out = out; a.enc = enc;
    return mt_launch_fwd<false>(a, stream);
}

int mcs_mlptex_bwd(const float *t, int64_t n, const float *aabb, const float *min_max, const float *params, const mcs_hashgrid_levels *lv,
                   int32_t hidden, int32_t channels, const float *const *weights, const float *enc, const float *d_out, float *d_params,
                   float *d_t, float *const *d_weights, void *workspace, mcs_stream stream)
{
    const char *fn = "mcs_mlptex_bwd";
    if (int e = mt_validate(fn, t, n, aabb, min_max, params, lv, hidden, channels, weights)) return e;
    MCS_REQUIRE(enc && d_out, "%s: null pointer (enc / d_out)", fn);
    bool want_dw;
    if (int e = mt_validate_bwd(fn, hidden, enc, d_params || d_t, d_weights, &want_dw, d_params, workspace)) return e;
    MtArgs a = mt_args(t, n, aabb, min_max, params, lv, hidden, channels, weights);
    a.enc = const_cast<float *>(enc); a.dout = d_out; a.dparams = (float2 *)d_params; a.dt = d_t; a.ws = want_dw ? (float *)workspace : nullptr;
    return mt_launch_bwd<false>(a, d_weights, stream);
}

int mcs_mlptex_pair_fwd(const float *t, const float *offset, int64_t n, const float *aabb, const float *min_max, const float *params,
                        const mcs_hashgrid_levels *lv, int32_t hidden, int32_t channels, const float *const *weights, float *out, float *out_jit,
                        float *enc, float *enc_jit, mcs_stream stream)
{
    const char *fn = "mcs_mlptex_pair_fwd";
    if (int e = mt_validate(fn, t, n, aabb, min_max, params, lv, hidden, channels, weights)) return e;
    MCS_REQUIRE(n <= (int64_t)INT32_MAX * (kThreads / 2), "%s: n too large", fn);            // two threads per pixel
    MCS_REQUIRE(offset != nullptr, "%s: null pointer (offset)", fn);
    MCS_REQUIRE(out && out_jit, "%s: null pointer (out / out_jit)", fn);
    MCS_REQUIRE(((uintptr_t)enc & 15) == 0 && ((uintptr_t)enc_jit & 15) == 0, "%s: enc and enc_jit must be 16-byte aligned", fn);
    MtArgs a = mt_args(t, n, aabb, min_max, params, lv, hidden, channels, weights);
    a.off = offset; a.out = out; a.out_jit = out_jit; a.enc = enc; a.enc_jit = enc_jit;
    return mt_launch_fwd<true>(a, stream);
}

int mcs_mlptex_pair_bwd(const float *t, const float *offset, int64_t n, const float *aabb, const float *min_max, const float *params,
                        const mcs_hashgrid_levels *lv, int32_t hidden, int32_t channels, const float *const *weights, const float *enc,
                        const float *enc_jit, const float *d_out, const float *d_out_jit, float *d_params, float *d_t, float *d_offset,
                        float *const *d_weights, void *workspace, mcs_stream stream)
{
    const char *fn = "mcs_mlptex_pair_bwd";
    if (int e = mt_validate(fn, t, n, aabb, min_max, params, lv, hidden, channels, weights)) return e;
    MCS_REQUIRE(offset != nullptr, "%s: null pointer (offset)", fn);
    MCS_REQUIRE(enc && enc_jit, "%s: null pointer (enc / enc_jit)", fn);
    MCS_REQUIRE(((uintptr_t)enc_jit & 15) == 0, "%s: enc_jit must be 16-byte aligned", fn);
    bool want_dw;
    if (int e = mt_validate_bwd(fn, hidden, enc, d_params || d_t || d_offset, d_weights, &want_dw, d_params, workspace)) return e;
    MtArgs a = mt_args(t, n, aabb, min_max, params, lv, hidden, channels, weights);
    a.off = offset; a.enc = const_cast<float *>(enc); a.enc_jit = const_cast<float *>(enc_jit); a.dout = d_out; a.dout_jit = d_out_jit;
    a.dparams = (float2 *)d_params; a.dt = d_t; a.doff = d_offset; a.ws = want_dw ? (float *)workspace : nullptr;
    return mt_launch_bwd<true>(a, d_weights, stream);
}

}  // extern "C"
