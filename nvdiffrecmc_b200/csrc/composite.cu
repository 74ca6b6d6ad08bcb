// composite.cu -- render_mesh's layer compositing (the reference's composite_buffer, render/render.py:284-291, run for every buffer key at
// :321-330) for every buffer of one depth-peel layer in one launch, forward and backward, with no host synchronisation.
// Semantics (the contract):
//
// A layer holds n buffers (1 <= n <= MCS_COMPOSITE_MAX_BUFFERS), buffer k an fp32 [B,H,W,C_k] view (C_k >= 1, any non-negative element
// strides), and its rast [B,H,W,4] (contiguous).  Layers are given front to back and composited back to front; for every key k, starting
// from accum_k = background_k (zeros when none is given):
//   mask    = rast.w > 0 ? 1 : 0, alpha_k = fl(mask * buf_k[C_k - 1])      (a multiplication: a NaN or inf alpha gives NaN even where uncovered)
//   end_k   = (buf_k[0 .. C_k - 2], 1)
//   lerped  = torch.lerp(accum_k, end_k, alpha_k): |w| < 0.5 ? fma(w, e - s, s) : fma(w - 1, e - s, e), e - s rounded once (torch's branch
//             rule and rounding; a NaN weight takes the second branch)
//   accum_k = antialias(lerped, rast, pos, tris, adj): raster.antialias's semantics (csrc/raster.cu header rules 1-6), bit for bit: the pairs
//             come from antialias.cuh, and v = c_p, then per pair p gains, in the order left, right, up, down, v = v + w (c_q - c_p), each
//             operation rounded.
// One launch per layer (mcs_composite_fwd): a thread per pixel searches its antialias pairs once and applies their weights to every
// channel of every buffer.  Only the lerp of a neighbour this pixel gains from is recomputed there, from that neighbour's accumulator and
// buffers; nothing is staged between the lerp and the antialias.  accum_in is the previous (deeper) layer's accum_out, or the backgrounds.
//
// Backward (mcs_composite_bwd), one launch per layer, front to back; G = d accum_out (the upstream gradient of this layer's output), and
// in torch's operation order:
//   d lerped  = k_antialias<true>'s gather: v = G_p, then per pair in pair order v = fma(-w, G_p, v) when p gains, fma(w, G_q, v) when q gains;
//   d accum_in_c = fl(d lerped_c * fl(1 - alpha)),  d buf_c = fl(d lerped_c * alpha) for c < C_k - 1 (the ones channel gets nothing),
//   d buf alpha  = fl(mask * sum_c fl(d lerped_c * fl(e_c - s_c))), summed in channel order over all C_k channels;
//   d pos     = per pair this pixel owns (right, down), one dL/dt = sum over the channels of every buffer of G_gain (lerped_other -
//               lerped_gain) (fmaf, buffer then channel order), then one set of float atomics through the crossing edge (antialias.cuh).
// The deepest layer's d accum_in is d background.  Every output except d pos has one writer per element and is bit-reproducible; d pos is
// an order-dependent float-atomic sum.  A null accum_in entry reads as zeros; a null d accum_in or d buffers entry is not written.
#include "antialias.cuh"

namespace {

struct SV {                      // [B,H,W,C] view, element strides; p null: zeros (input) or not written (output)
    float *p;
    int s0, s1, s2, s3;
};

__device__ __forceinline__ int64_t sv_off(const SV &v, int b, int y, int x, int c)
{
    return (int64_t)b * v.s0 + (int64_t)y * v.s1 + (int64_t)x * v.s2 + (int64_t)c * v.s3;
}
__device__ __forceinline__ float sv_ld(const SV &v, int b, int y, int x, int c) { return __ldg(v.p + sv_off(v, b, y, x, c)); }
__device__ __forceinline__ void sv_st(const SV &v, int b, int y, int x, int c, float x_) { v.p[sv_off(v, b, y, x, c)] = x_; }

struct CompKey {
    SV buf, acc, out;            // forward: this layer's buffer, accum_in, accum_out
    SV dout, dacc, dbuf;         // backward: d accum_out (read), d accum_in and d buf (written when non-null)
    int C;
};

struct CompParams {
    AAGeom g;
    int n;
    int64_t npx;
    float *dpos;
    CompKey k[MCS_COMPOSITE_MAX_BUFFERS];
};

// torch.lerp(s, e, w) (ATen's lerp: branch on |w| < 0.5, each branch one fused multiply-add)
__device__ __forceinline__ float lerp_t(float s, float e, float w)
{
    const float d = __fsub_rn(e, s);
    return fabsf(w) < 0.5f ? __fmaf_rn(w, d, s) : __fmaf_rn(__fsub_rn(w, 1.0f), d, e);
}

__device__ __forceinline__ float mask_of(float4 r) { return r.w > 0.0f ? 1.0f : 0.0f; }

__device__ __forceinline__ float alpha_at(const CompKey &K, int b, int y, int x, float m) { return __fmul_rn(m, sv_ld(K.buf, b, y, x, K.C - 1)); }

__device__ __forceinline__ float acc_at(const CompKey &K, int b, int y, int x, int c) { return K.acc.p ? sv_ld(K.acc, b, y, x, c) : 0.0f; }
__device__ __forceinline__ float end_at(const CompKey &K, int b, int y, int x, int c) { return c == K.C - 1 ? 1.0f : sv_ld(K.buf, b, y, x, c); }

__device__ __forceinline__ float lerped_at(const CompKey &K, int b, int y, int x, int c, float a)
{
    return lerp_t(acc_at(K, b, y, x, c), end_at(K, b, y, x, c), a);
}

__global__ void __launch_bounds__(256) k_composite_fwd(const CompParams p)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.npx) return;
    int b, iy, ix;
    px_decode(i, p.g.H, p.g.W, b, iy, ix);
    const float4 r = __ldg(p.g.rast + i);
    const AAPairs pr = aa_pixel_pairs<false>(p.g, i, b, iy, ix, r, nullptr, [](bool, int, int64_t) { return 0.0f; });
    bool gain[4];
    float mq[4];
#pragma unroll
    for (int d = 0; d < 4; ++d) {
        gain[d] = pr.on[d] && pr.self[d];
        mq[d] = gain[d] ? mask_of(__ldg(p.g.rast + pr.j[d])) : 0.0f;
    }
    const float mp = mask_of(r);
    for (int k = 0; k < p.n; ++k) {
        const CompKey &K = p.k[k];
        const int C = K.C;
        const float ap = alpha_at(K, b, iy, ix, mp);
        float aq[4];
#pragma unroll
        for (int d = 0; d < 4; ++d) aq[d] = gain[d] ? alpha_at(K, b, aa_nby(d, iy), aa_nbx(d, ix), mq[d]) : 0.0f;
        for (int c = 0; c < C; ++c) {
            const float cs = lerped_at(K, b, iy, ix, c, ap);
            float v = cs;
#pragma unroll
            for (int d = 0; d < 4; ++d)
                if (gain[d]) v = __fadd_rn(v, __fmul_rn(pr.w[d], __fsub_rn(lerped_at(K, b, aa_nby(d, iy), aa_nbx(d, ix), c, aq[d]), cs)));
            sv_st(K.out, b, iy, ix, c, v);
        }
    }
}

__global__ void __launch_bounds__(256) k_composite_bwd(const CompParams p)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.npx) return;
    int b, iy, ix;
    px_decode(i, p.g.H, p.g.W, b, iy, ix);
    const float4 r = __ldg(p.g.rast + i);
    const float mp = mask_of(r);
    const AAPairs pr = aa_pixel_pairs<true>(p.g, i, b, iy, ix, r, p.dpos, [&](bool gain_self, int d, int64_t j) {
        const int ny = aa_nby(d, iy), nx = aa_nbx(d, ix);
        const float mj = mask_of(__ldg(p.g.rast + j));
        const int gy = gain_self ? iy : ny, gx = gain_self ? ix : nx, oy = gain_self ? ny : iy, ox = gain_self ? nx : ix;
        const float mg = gain_self ? mp : mj, mo = gain_self ? mj : mp;
        float s = 0.0f;
        for (int k = 0; k < p.n; ++k) {
            const CompKey &K = p.k[k];
            const float ag = alpha_at(K, b, gy, gx, mg), ao = alpha_at(K, b, oy, ox, mo);
            for (int c = 0; c < K.C; ++c)
                s = fmaf(sv_ld(K.dout, b, gy, gx, c), lerped_at(K, b, oy, ox, c, ao) - lerped_at(K, b, gy, gx, c, ag), s);
        }
        return s;
    });
    for (int k = 0; k < p.n; ++k) {
        const CompKey &K = p.k[k];
        const int C = K.C;
        const float ap = alpha_at(K, b, iy, ix, mp), om = __fsub_rn(1.0f, ap);
        float sa = 0.0f;
        for (int c = 0; c < C; ++c) {
            const float g = sv_ld(K.dout, b, iy, ix, c);
            float v = g;
#pragma unroll
            for (int d = 0; d < 4; ++d)
                if (pr.on[d]) v = pr.self[d] ? __fmaf_rn(-pr.w[d], g, v) : __fmaf_rn(pr.w[d], sv_ld(K.dout, b, aa_nby(d, iy), aa_nbx(d, ix), c), v);
            if (K.dacc.p) sv_st(K.dacc, b, iy, ix, c, __fmul_rn(v, om));
            if (K.dbuf.p && c < C - 1) sv_st(K.dbuf, b, iy, ix, c, __fmul_rn(v, ap));
            const float t = __fmul_rn(v, __fsub_rn(end_at(K, b, iy, ix, c), acc_at(K, b, iy, ix, c)));
            sa = c == 0 ? t : __fadd_rn(sa, t);
        }
        if (K.dbuf.p) sv_st(K.dbuf, b, iy, ix, C - 1, __fmul_rn(mp, sa));
    }
}

// Checks entry k of the descriptor table `what` against B, H, W and C (a null table entry is allowed when `optional`) and fills v.
int sv_view(const char *fn, const char *what, int k, const mcs_tensor *t, int B, int H, int W, int C, bool optional, SV &v)
{
    v = SV{};
    if (!t->ptr) {
        MCS_REQUIRE(optional, "%s: %s[%d] is null", fn, what, k);
        return 0;
    }
    MCS_REQUIRE(t->sizes[0] == B && t->sizes[1] == H && t->sizes[2] == W && t->sizes[3] == C,
                "%s: %s[%d] is [%d,%d,%d,%d], expected [%d,%d,%d,%d]", fn, what, k, t->sizes[0], t->sizes[1], t->sizes[2], t->sizes[3], B, H, W, C);
    for (int d = 0; d < 4; ++d) MCS_REQUIRE(t->strides[d] >= 0, "%s: %s[%d] has a negative stride", fn, what, k);
    v.p = (float *)t->ptr;
    v.s0 = t->strides[0]; v.s1 = t->strides[1]; v.s2 = t->strides[2]; v.s3 = t->strides[3];
    return 0;
}

int comp_args(const char *fn, int32_t n, const mcs_tensor *buffers, const mcs_tensor *accum_in, const float *rast, const float *pos,
              int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, CompParams &p)
{
    MCS_REQUIRE(n >= 1 && n <= MCS_COMPOSITE_MAX_BUFFERS, "%s: %d buffers (1 to %d allowed)", fn, n, MCS_COMPOSITE_MAX_BUFFERS);
    MCS_REQUIRE(buffers && accum_in && rast && pos && tris && adj && V > 0 && T > 0 && pos_batch_stride >= 0, "%s: bad arguments", fn);
    const int B = buffers[0].sizes[0], H = buffers[0].sizes[1], W = buffers[0].sizes[2];
    MCS_REQUIRE(B > 0 && H > 0 && W > 0, "%s: empty buffers", fn);
    p.n = n;
    p.npx = (int64_t)B * H * W;
    p.g = AAGeom{(const float4 *)rast, B, H, W, pos, pos_batch_stride, V, tris, T, adj};
    for (int k = 0; k < n; ++k) {
        const int C = buffers[k].sizes[3];
        if (int e = sv_view(fn, "buffers", k, buffers + k, B, H, W, C, false, p.k[k].buf)) return e;
        MCS_REQUIRE(C >= 1, "%s: buffers[%d] has no channels", fn, k);
        p.k[k].C = C;
        if (int e = sv_view(fn, "accum_in", k, accum_in + k, B, H, W, C, true, p.k[k].acc)) return e;
    }
    return 0;
}

}  // namespace

extern "C" {

int mcs_composite_fwd(int32_t n_buffers, const mcs_tensor *buffers, const mcs_tensor *accum_in, const mcs_tensor *accum_out, const float *rast,
                      const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, mcs_stream stream)
{
    const char *fn = "mcs_composite_fwd";
    CompParams p{};
    if (int e = comp_args(fn, n_buffers, buffers, accum_in, rast, pos, pos_batch_stride, V, tris, T, adj, p)) return e;
    MCS_REQUIRE(accum_out, "%s: null accum_out", fn);
    for (int k = 0; k < p.n; ++k)
        if (int e = sv_view(fn, "accum_out", k, accum_out + k, p.g.B, p.g.H, p.g.W, p.k[k].C, false, p.k[k].out)) return e;
    k_composite_fwd<<<(unsigned)((p.npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

int mcs_composite_bwd(int32_t n_buffers, const mcs_tensor *buffers, const mcs_tensor *accum_in, const mcs_tensor *d_accum_out,
                      const mcs_tensor *d_accum_in, const mcs_tensor *d_buffers, const float *rast, const float *pos, int64_t pos_batch_stride,
                      int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, float *d_pos, mcs_stream stream)
{
    const char *fn = "mcs_composite_bwd";
    CompParams p{};
    if (int e = comp_args(fn, n_buffers, buffers, accum_in, rast, pos, pos_batch_stride, V, tris, T, adj, p)) return e;
    MCS_REQUIRE(d_accum_out && d_accum_in && d_buffers, "%s: null gradient table", fn);
    for (int k = 0; k < p.n; ++k) {
        const int B = p.g.B, H = p.g.H, W = p.g.W, C = p.k[k].C;
        if (int e = sv_view(fn, "d_accum_out", k, d_accum_out + k, B, H, W, C, false, p.k[k].dout)) return e;
        if (int e = sv_view(fn, "d_accum_in", k, d_accum_in + k, B, H, W, C, true, p.k[k].dacc)) return e;
        if (int e = sv_view(fn, "d_buffers", k, d_buffers + k, B, H, W, C, true, p.k[k].dbuf)) return e;
    }
    p.dpos = d_pos;
    k_composite_bwd<<<(unsigned)((p.npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p);
    MCS_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
