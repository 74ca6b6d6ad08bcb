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
//
// Supersampling (mcs_composite_ss_fwd / _bwd, render_mesh with spp > 1, render.py:247-250 and 313-330): rast is at full resolution
// [B,H,W,4] with H and W multiples of spp, and every pixel runs the rules above.  Each descriptor table is at full resolution [B,H,W,C_k]
// or at output resolution [B,H/spp,W/spp,C_k], uniform within the table:
//   - an output-resolution input (buffers, accum_in, i.e. MSAA-shaded buffers and the backgrounds) is read by full-resolution pixel (y, x)
//     at (y / spp, x / spp): scale_img_nhwc(..., mag='nearest'), without the full-resolution copy;
//   - an output-resolution accum_out is avg_pool_nhwc(accum, spp): the fp32 sum, from 0, of its spp x spp block in row-major order
//     (rows outer), divided by spp^2 (ATen's avg_pool2d);
//   - an output-resolution d accum_out gives every pixel of its block the upstream gradient fl(g / spp^2) (avg_pool2d's backward);
//   - an output-resolution d accum_in or d buffers entry is the fp32 sum, from 0, of its block's per-pixel gradients in row-major order
//     (upsample_nearest2d's backward).
// A thread then takes one output-resolution pixel and walks its block in row-major order, so every output still has one writer and a
// fixed summation order; the running sums live in the output element itself.  mcs_composite_fwd / _bwd are the spp = 1 case.
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

struct CompKey {
    SV buf, acc, out;            // forward: this layer's buffer, accum_in, accum_out
    SV dout, dacc, dbuf;         // backward: d accum_out (read), d accum_in and d buf (written when non-null)
    int C;
};

// Resolution of each table: 1 (full, pixel (y, x) is element (y, x)) or spp (output, pixel (y, x) is element (y / spp, x / spp)).
struct CompRes {
    int buf, acc, out, dout, dacc, dbuf;
};

struct CompParams {
    AAGeom g;
    int n;
    int64_t npx;                 // threads: full-resolution pixels (spp 1) or output-resolution pixels
    int spp, nsub, Ho, Wo;       // nsub = spp^2, Ho x Wo = the output resolution
    CompRes r;
    float *dpos;
    CompKey k[MCS_COMPOSITE_MAX_BUFFERS];
};

// Offset of full-resolution pixel (y, x) in view v at resolution sc; SS: the supersampled kernels, where sc may be spp.
template <bool SS>
__device__ __forceinline__ int64_t px_off(const SV &v, int sc, int b, int y, int x, int c)
{
    if (SS && sc != 1) { y = (int)((unsigned)y / (unsigned)sc); x = (int)((unsigned)x / (unsigned)sc); }
    return sv_off(v, b, y, x, c);
}
template <bool SS>
__device__ __forceinline__ float ld_at(const SV &v, int sc, int b, int y, int x, int c) { return __ldg(v.p + px_off<SS>(v, sc, b, y, x, c)); }

// Writes full-resolution pixel (y, x)'s value x_, step s of its block walk: directly at full resolution; at output resolution into the
// element's running sum (from 0 at s = 0), divided by spp^2 at the block's last step when `mean`.
template <bool SS>
__device__ __forceinline__ void st_at(const CompParams &p, const SV &v, int sc, int b, int y, int x, int c, float x_, int s, bool mean)
{
    float *q = v.p + px_off<SS>(v, sc, b, y, x, c);
    if (!SS || sc == 1) { *q = x_; return; }
    const float sum = __fadd_rn(s == 0 ? 0.0f : *q, x_);
    *q = mean && s == p.nsub - 1 ? __fdiv_rn(sum, (float)p.nsub) : sum;
}

// torch.lerp(s, e, w) (ATen's lerp: branch on |w| < 0.5, each branch one fused multiply-add)
__device__ __forceinline__ float lerp_t(float s, float e, float w)
{
    const float d = __fsub_rn(e, s);
    return fabsf(w) < 0.5f ? __fmaf_rn(w, d, s) : __fmaf_rn(__fsub_rn(w, 1.0f), d, e);
}

__device__ __forceinline__ float mask_of(float4 r) { return r.w > 0.0f ? 1.0f : 0.0f; }

template <bool SS>
__device__ __forceinline__ float alpha_at(const CompParams &p, const CompKey &K, int b, int y, int x, float m)
{
    return __fmul_rn(m, ld_at<SS>(K.buf, p.r.buf, b, y, x, K.C - 1));
}
template <bool SS>
__device__ __forceinline__ float acc_at(const CompParams &p, const CompKey &K, int b, int y, int x, int c)
{
    return K.acc.p ? ld_at<SS>(K.acc, p.r.acc, b, y, x, c) : 0.0f;
}
template <bool SS>
__device__ __forceinline__ float end_at(const CompParams &p, const CompKey &K, int b, int y, int x, int c)
{
    return c == K.C - 1 ? 1.0f : ld_at<SS>(K.buf, p.r.buf, b, y, x, c);
}
template <bool SS>
__device__ __forceinline__ float lerped_at(const CompParams &p, const CompKey &K, int b, int y, int x, int c, float a)
{
    return lerp_t(acc_at<SS>(p, K, b, y, x, c), end_at<SS>(p, K, b, y, x, c), a);
}
// upstream gradient of full-resolution pixel (y, x): d accum_out there, or fl(g / spp^2) of its output-resolution pixel
template <bool SS>
__device__ __forceinline__ float dout_at(const CompParams &p, const CompKey &K, int b, int y, int x, int c)
{
    const float g = ld_at<SS>(K.dout, p.r.dout, b, y, x, c);
    return SS && p.r.dout != 1 ? __fdiv_rn(g, (float)p.nsub) : g;
}

// The forward of full-resolution pixel i = (b, iy, ix), step s of its thread's block walk.
template <bool SS>
__device__ __forceinline__ void comp_fwd_px(const CompParams &p, int64_t i, int b, int iy, int ix, int s)
{
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
        const float ap = alpha_at<SS>(p, K, b, iy, ix, mp);
        float aq[4];
#pragma unroll
        for (int d = 0; d < 4; ++d) aq[d] = gain[d] ? alpha_at<SS>(p, K, b, aa_nby(d, iy), aa_nbx(d, ix), mq[d]) : 0.0f;
        for (int c = 0; c < C; ++c) {
            const float cs = lerped_at<SS>(p, K, b, iy, ix, c, ap);
            float v = cs;
#pragma unroll
            for (int d = 0; d < 4; ++d)
                if (gain[d]) v = __fadd_rn(v, __fmul_rn(pr.w[d], __fsub_rn(lerped_at<SS>(p, K, b, aa_nby(d, iy), aa_nbx(d, ix), c, aq[d]), cs)));
            st_at<SS>(p, K.out, p.r.out, b, iy, ix, c, v, s, true);
        }
    }
}

// The backward of full-resolution pixel i = (b, iy, ix), step s of its thread's block walk.
template <bool SS>
__device__ __forceinline__ void comp_bwd_px(const CompParams &p, int64_t i, int b, int iy, int ix, int s)
{
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
            const float ag = alpha_at<SS>(p, K, b, gy, gx, mg), ao = alpha_at<SS>(p, K, b, oy, ox, mo);
            for (int c = 0; c < K.C; ++c)
                s = fmaf(dout_at<SS>(p, K, b, gy, gx, c), lerped_at<SS>(p, K, b, oy, ox, c, ao) - lerped_at<SS>(p, K, b, gy, gx, c, ag), s);
        }
        return s;
    });
    for (int k = 0; k < p.n; ++k) {
        const CompKey &K = p.k[k];
        const int C = K.C;
        const float ap = alpha_at<SS>(p, K, b, iy, ix, mp), om = __fsub_rn(1.0f, ap);
        float sa = 0.0f;
        for (int c = 0; c < C; ++c) {
            const float g = dout_at<SS>(p, K, b, iy, ix, c);
            float v = g;
#pragma unroll
            for (int d = 0; d < 4; ++d)
                if (pr.on[d]) v = pr.self[d] ? __fmaf_rn(-pr.w[d], g, v) : __fmaf_rn(pr.w[d], dout_at<SS>(p, K, b, aa_nby(d, iy), aa_nbx(d, ix), c), v);
            if (K.dacc.p) st_at<SS>(p, K.dacc, p.r.dacc, b, iy, ix, c, __fmul_rn(v, om), s, false);
            if (K.dbuf.p && c < C - 1) st_at<SS>(p, K.dbuf, p.r.dbuf, b, iy, ix, c, __fmul_rn(v, ap), s, false);
            const float t = __fmul_rn(v, __fsub_rn(end_at<SS>(p, K, b, iy, ix, c), acc_at<SS>(p, K, b, iy, ix, c)));
            sa = c == 0 ? t : __fadd_rn(sa, t);
        }
        if (K.dbuf.p) st_at<SS>(p, K.dbuf, p.r.dbuf, b, iy, ix, C - 1, __fmul_rn(mp, sa), s, false);
    }
}

// One kernel body per direction: without SS a thread per full-resolution pixel, with SS a thread per output-resolution pixel that walks
// its spp x spp block in row-major order.
template <bool BWD, bool SS>
__global__ void __launch_bounds__(256) k_composite(const CompParams p)
{
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= p.npx) return;
    int b, y, x;
    if (!SS) {
        px_decode(t, p.g.H, p.g.W, b, y, x);
        if (BWD) comp_bwd_px<false>(p, t, b, y, x, 0);
        else comp_fwd_px<false>(p, t, b, y, x, 0);
        return;
    }
    px_decode(t, p.Ho, p.Wo, b, y, x);
    int s = 0;
    for (int sy = 0; sy < p.spp; ++sy)
        for (int sx = 0; sx < p.spp; ++sx, ++s) {
            const int iy = y * p.spp + sy, ix = x * p.spp + sx;
            const int64_t i = ((int64_t)b * p.g.H + iy) * p.g.W + ix;
            if (BWD) comp_bwd_px<true>(p, i, b, iy, ix, s);
            else comp_fwd_px<true>(p, i, b, iy, ix, s);
        }
}

// Checks entry k of the descriptor table `what` against B, H, W and C (a null table entry is allowed when `optional`) and fills v.  The
// table is at full resolution [B,H,W,C] or, with spp > 1, at output resolution [B,H/spp,W/spp,C]: sc is 0 until the table's first
// non-null entry sets it to 1 or spp, and every later entry must match it.
int sv_view(const char *fn, const char *what, int k, const mcs_tensor *t, int B, int H, int W, int spp, int C, bool optional, int &sc, SV &v)
{
    v = SV{};
    if (!t->ptr) {
        MCS_REQUIRE(optional, "%s: %s[%d] is null", fn, what, k);
        return 0;
    }
    const bool full = t->sizes[0] == B && t->sizes[1] == H && t->sizes[2] == W && t->sizes[3] == C;
    const bool outr = spp > 1 && t->sizes[0] == B && t->sizes[1] == H / spp && t->sizes[2] == W / spp && t->sizes[3] == C;
    if (spp == 1)
        MCS_REQUIRE(full, "%s: %s[%d] is [%d,%d,%d,%d], expected [%d,%d,%d,%d]", fn, what, k, t->sizes[0], t->sizes[1], t->sizes[2], t->sizes[3],
                    B, H, W, C);
    else
        MCS_REQUIRE(full || outr, "%s: %s[%d] is [%d,%d,%d,%d], expected [%d,%d,%d,%d] or [%d,%d,%d,%d]", fn, what, k, t->sizes[0], t->sizes[1],
                    t->sizes[2], t->sizes[3], B, H, W, C, B, H / spp, W / spp, C);
    const int s = full ? 1 : spp;
    MCS_REQUIRE(sc == 0 || sc == s, "%s: %s[%d] is at %s resolution, an earlier entry at %s resolution", fn, what, k, s == 1 ? "full" : "output",
                s == 1 ? "output" : "full");
    sc = s;
    for (int d = 0; d < 4; ++d) MCS_REQUIRE(t->strides[d] >= 0, "%s: %s[%d] has a negative stride", fn, what, k);
    v.p = (float *)t->ptr;
    v.s0 = t->strides[0]; v.s1 = t->strides[1]; v.s2 = t->strides[2]; v.s3 = t->strides[3];
    return 0;
}

int comp_args(const char *fn, int32_t n, const mcs_tensor *buffers, const mcs_tensor *accum_in, int B, int H, int W, int spp, const float *rast,
              const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, CompParams &p)
{
    MCS_REQUIRE(n >= 1 && n <= MCS_COMPOSITE_MAX_BUFFERS, "%s: %d buffers (1 to %d allowed)", fn, n, MCS_COMPOSITE_MAX_BUFFERS);
    MCS_REQUIRE(buffers && accum_in && rast && pos && tris && adj && V > 0 && T > 0 && pos_batch_stride >= 0, "%s: bad arguments", fn);
    MCS_REQUIRE(B > 0 && H > 0 && W > 0, "%s: empty buffers", fn);
    MCS_REQUIRE(spp >= 1, "%s: spp %d (1 or more allowed)", fn, spp);
    MCS_REQUIRE(H % spp == 0 && W % spp == 0, "%s: H x W = %d x %d is not a multiple of spp %d", fn, H, W, spp);
    p.n = n;
    p.spp = spp;
    p.nsub = spp * spp;
    p.Ho = H / spp;
    p.Wo = W / spp;
    p.npx = (int64_t)B * p.Ho * p.Wo;
    p.g = AAGeom{(const float4 *)rast, B, H, W, pos, pos_batch_stride, V, tris, T, adj};
    p.r = CompRes{};
    for (int k = 0; k < n; ++k) {
        const int C = buffers[k].sizes[3];
        if (int e = sv_view(fn, "buffers", k, buffers + k, B, H, W, spp, C, false, p.r.buf, p.k[k].buf)) return e;
        MCS_REQUIRE(C >= 1, "%s: buffers[%d] has no channels", fn, k);
        p.k[k].C = C;
        if (int e = sv_view(fn, "accum_in", k, accum_in + k, B, H, W, spp, C, true, p.r.acc, p.k[k].acc)) return e;
    }
    return 0;
}

// Reads the table `what` into the views of field `f` of every key; its resolution goes to sc (0 when every entry is null).
template <class F>
int comp_table(const char *fn, const char *what, const mcs_tensor *t, bool optional, CompParams &p, int &sc, F f)
{
    sc = 0;
    for (int k = 0; k < p.n; ++k)
        if (int e = sv_view(fn, what, k, t + k, p.g.B, p.g.H, p.g.W, p.spp, p.k[k].C, optional, sc, f(p.k[k]))) return e;
    return 0;
}

int comp_launch(bool bwd, CompParams &p, mcs_stream stream)
{
    for (int *sc : {&p.r.buf, &p.r.acc, &p.r.out, &p.r.dout, &p.r.dacc, &p.r.dbuf})
        if (*sc == 0) *sc = 1;                    // an all-null table: never read or written
    const unsigned grid = (unsigned)((p.npx + 255) / 256);
    const cudaStream_t s = (cudaStream_t)stream;
    if (p.spp == 1) {
        if (bwd) k_composite<true, false><<<grid, 256, 0, s>>>(p);
        else k_composite<false, false><<<grid, 256, 0, s>>>(p);
    } else {
        if (bwd) k_composite<true, true><<<grid, 256, 0, s>>>(p);
        else k_composite<false, true><<<grid, 256, 0, s>>>(p);
    }
    MCS_LAUNCH_CHECK();
    return 0;
}

int comp_fwd(const char *fn, int32_t n, const mcs_tensor *buffers, const mcs_tensor *accum_in, const mcs_tensor *accum_out, int B, int H, int W,
             int spp, const float *rast, const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const int32_t *adj,
             mcs_stream stream)
{
    CompParams p{};
    if (int e = comp_args(fn, n, buffers, accum_in, B, H, W, spp, rast, pos, pos_batch_stride, V, tris, T, adj, p)) return e;
    MCS_REQUIRE(accum_out, "%s: null accum_out", fn);
    if (int e = comp_table(fn, "accum_out", accum_out, false, p, p.r.out, [](CompKey &K) -> SV & { return K.out; })) return e;
    return comp_launch(false, p, stream);
}

int comp_bwd(const char *fn, int32_t n, const mcs_tensor *buffers, const mcs_tensor *accum_in, const mcs_tensor *d_accum_out,
             const mcs_tensor *d_accum_in, const mcs_tensor *d_buffers, int B, int H, int W, int spp, const float *rast, const float *pos,
             int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, float *d_pos, mcs_stream stream)
{
    CompParams p{};
    if (int e = comp_args(fn, n, buffers, accum_in, B, H, W, spp, rast, pos, pos_batch_stride, V, tris, T, adj, p)) return e;
    MCS_REQUIRE(d_accum_out && d_accum_in && d_buffers, "%s: null gradient table", fn);
    if (int e = comp_table(fn, "d_accum_out", d_accum_out, false, p, p.r.dout, [](CompKey &K) -> SV & { return K.dout; })) return e;
    if (int e = comp_table(fn, "d_accum_in", d_accum_in, true, p, p.r.dacc, [](CompKey &K) -> SV & { return K.dacc; })) return e;
    if (int e = comp_table(fn, "d_buffers", d_buffers, true, p, p.r.dbuf, [](CompKey &K) -> SV & { return K.dbuf; })) return e;
    // a gradient is at its input's resolution (a table whose entries are all null has none)
    auto res = [](int sc) { return sc > 1 ? "output" : "full"; };
    MCS_REQUIRE(!p.r.dbuf || p.r.dbuf == p.r.buf, "%s: d_buffers is at %s resolution, buffers at %s", fn, res(p.r.dbuf), res(p.r.buf));
    MCS_REQUIRE(!p.r.dacc || !p.r.acc || p.r.dacc == p.r.acc, "%s: d_accum_in is at %s resolution, accum_in at %s", fn, res(p.r.dacc),
                res(p.r.acc));
    p.dpos = d_pos;
    return comp_launch(true, p, stream);
}

}  // namespace

extern "C" {

int mcs_composite_fwd(int32_t n_buffers, const mcs_tensor *buffers, const mcs_tensor *accum_in, const mcs_tensor *accum_out, const float *rast,
                      const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, mcs_stream stream)
{
    const bool ok = n_buffers >= 1 && n_buffers <= MCS_COMPOSITE_MAX_BUFFERS && buffers;
    return comp_fwd("mcs_composite_fwd", n_buffers, buffers, accum_in, accum_out, ok ? buffers[0].sizes[0] : 0, ok ? buffers[0].sizes[1] : 0,
                    ok ? buffers[0].sizes[2] : 0, 1, rast, pos, pos_batch_stride, V, tris, T, adj, stream);
}

int mcs_composite_bwd(int32_t n_buffers, const mcs_tensor *buffers, const mcs_tensor *accum_in, const mcs_tensor *d_accum_out,
                      const mcs_tensor *d_accum_in, const mcs_tensor *d_buffers, const float *rast, const float *pos, int64_t pos_batch_stride,
                      int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, float *d_pos, mcs_stream stream)
{
    const bool ok = n_buffers >= 1 && n_buffers <= MCS_COMPOSITE_MAX_BUFFERS && buffers;
    return comp_bwd("mcs_composite_bwd", n_buffers, buffers, accum_in, d_accum_out, d_accum_in, d_buffers, ok ? buffers[0].sizes[0] : 0,
                    ok ? buffers[0].sizes[1] : 0, ok ? buffers[0].sizes[2] : 0, 1, rast, pos, pos_batch_stride, V, tris, T, adj, d_pos, stream);
}

int mcs_composite_ss_fwd(int32_t n_buffers, const mcs_tensor *buffers, const mcs_tensor *accum_in, const mcs_tensor *accum_out, int32_t B,
                         int32_t H, int32_t W, int32_t spp, const float *rast, const float *pos, int64_t pos_batch_stride, int32_t V,
                         const int32_t *tris, int32_t T, const int32_t *adj, mcs_stream stream)
{
    return comp_fwd("mcs_composite_ss_fwd", n_buffers, buffers, accum_in, accum_out, B, H, W, spp, rast, pos, pos_batch_stride, V, tris, T, adj,
                    stream);
}

int mcs_composite_ss_bwd(int32_t n_buffers, const mcs_tensor *buffers, const mcs_tensor *accum_in, const mcs_tensor *d_accum_out,
                         const mcs_tensor *d_accum_in, const mcs_tensor *d_buffers, int32_t B, int32_t H, int32_t W, int32_t spp, const float *rast,
                         const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, float *d_pos,
                         mcs_stream stream)
{
    return comp_bwd("mcs_composite_ss_bwd", n_buffers, buffers, accum_in, d_accum_out, d_accum_in, d_buffers, B, H, W, spp, rast, pos,
                    pos_batch_stride, V, tris, T, adj, d_pos, stream);
}

}  // extern "C"
