// elementwise.cu -- H100 kernels for the renderutils streaming ops:
//   lambert / frostbite_diffuse / fresnel_shlick / ndf_ggx / lambda_ggx / masking_smith /
//   pbr_specular / pbr_bsdf / prepare_shading_normal / shade_combine, forward and backward.
// Replaces render/renderutils/c_src/bsdf.cu:382-707, normal.cu:95-178 and their launchers in
// render/renderutils/c_src/torch_bindings.cpp (8x8 blocks, one scalar-load pixel per thread).
//
// These ops are pure HBM streaming (84 B/px fwd, 156 B/px bwd for pbr_bsdf, SURVEY.md section 8d).
// Design: each thread owns FOUR consecutive pixels so that every contiguous [.,3] fp32 operand is
// moved with three 128-bit loads/stores (48 B per thread, 1536 B per warp-instruction group, fully
// coalesced), broadcast operands (e.g. view_pos [B,1,1,3]) fall back to strided scalar loads that
// hit L1; grid = enough 256-thread CTAs to cover the pixels (>= several waves over 132 SMs at
// 512x512), no shared memory, no divergence except the BSDF's own branches.
#include <utility>

#include "bsdf.cuh"

namespace {

struct Grid { int N, H, W; int64_t npx; };

struct TIn {
    TView v;
    int fast;      // contiguous, full grid, 16B aligned -> vector path
};

struct Px4 {
    int64_t p0;
    int cnt;
};

__device__ __forceinline__ void px_decode(const Grid &g, int64_t p, int &n, int &h, int &w)
{
    w = (int)(p % g.W);
    int64_t t = p / g.W;
    h = (int)(t % g.H);
    n = (int)(t / g.H);
}

// FULL = all four pixels valid: every loop bound and array index is a compile-time constant, so the pixel
// registers never spill to local memory (the ragged tail is a separate, rarely executed instantiation).
template <int C, bool FULL>
__device__ __forceinline__ void ew_load(const TIn &t, const Grid &g, const Px4 &q, float (&out)[4][C])
{
    if (FULL && t.fast) {
        const float4 *src = reinterpret_cast<const float4 *>(t.v.p + q.p0 * C);
        float buf[4 * C];
#pragma unroll
        for (int i = 0; i < C; ++i) {
            float4 x = __ldg(src + i);
            buf[4 * i + 0] = x.x; buf[4 * i + 1] = x.y; buf[4 * i + 2] = x.z; buf[4 * i + 3] = x.w;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int c = 0; c < C; ++c) out[k][c] = buf[k * C + c];
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (FULL || k < q.cnt) {
                int n, h, w;
                px_decode(g, q.p0 + k, n, h, w);
                const float *src = t.v.p + t.v.off(n, h, w);
#pragma unroll
                for (int c = 0; c < C; ++c) out[k][c] = __ldg(src + (t.v.n3 == 1 ? 0 : c * t.v.s3));
            } else {
#pragma unroll
                for (int c = 0; c < C; ++c) out[k][c] = 0.0f;
            }
        }
    }
}

template <int C, bool FULL>
__device__ __forceinline__ void ew_store(float *dst, const Px4 &q, const float (&v)[4][C])
{
    if (FULL) {
        float buf[4 * C];
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int c = 0; c < C; ++c) buf[k * C + c] = v[k][c];
        float4 *d = reinterpret_cast<float4 *>(dst + q.p0 * C);
#pragma unroll
        for (int i = 0; i < C; ++i) d[i] = make_float4(buf[4 * i], buf[4 * i + 1], buf[4 * i + 2], buf[4 * i + 3]);
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (k < q.cnt) {
#pragma unroll
                for (int c = 0; c < C; ++c) dst[(q.p0 + k) * C + c] = v[k][c];
            }
    }
}

__device__ __forceinline__ f3 to3(const float (&a)[3]) { return F3(a[0], a[1], a[2]); }
__device__ __forceinline__ void from3(float (&a)[3], f3 v) { a[0] = v.x; a[1] = v.y; a[2] = v.z; }

#ifndef MCS_EW_MINB
#define MCS_EW_MINB 2          // caps the heaviest op (pbr_bsdf backward, 139 regs) at 128 so two CTAs fit: 0.32 -> 0.21 ms at 16x512x512
#endif
template <class Op>
__global__ void __launch_bounds__(256, MCS_EW_MINB) ew_kernel(Op op, Grid g)
{
    int64_t q4 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    Px4 q;
    q.p0 = q4 * 4;
    if (q.p0 >= g.npx) return;
    int64_t rem = g.npx - q.p0;
    q.cnt = rem >= 4 ? 4 : (int)rem;
    if (q.cnt == 4) op.template run<true>(g, q);
    else op.template run<false>(g, q);
}

// ---------------------------------------------------------------------------------------------
// Ops
// ---------------------------------------------------------------------------------------------
// Each op is one declaration: its operands' names and channel counts (arg), its forward output's channel count (OUT), its scalar
// members, and two per-pixel bodies, fwd(operands..., out) and bwd(operands..., d_operands..., d_out).  The backward writes one
// gradient per operand, with that operand's channel count.  Ew<Op, BWD> loads, runs and stores them, and ew() checks the entry's
// tensors with the same channel counts; a body whose parameters disagree with arg does not compile.
struct Arg {
    const char *name;
    int C;
    bool opt = false;   // read, and its gradient written, only while opt_on(op) holds
};
template <class Op> __host__ __device__ __forceinline__ bool opt_on(const Op &) { return true; }
template <int C> using In = const float (&)[C];
template <int C> using Out = float (&)[C];

struct Lambert {
    static constexpr Arg arg[] = {{"nrm", 3}, {"wi", 3}};
    static constexpr int OUT = 1;
    __device__ void fwd(In<3> n, In<3> wi, Out<1> o) const { o[0] = fwd_lambert(to3(n), to3(wi)); }
    __device__ void bwd(In<3> n, In<3> wi, Out<3> g_n, Out<3> g_wi, In<1> d) const
    {
        f3 x = F3(0.0f), y = F3(0.0f);
        bwd_lambert(to3(n), to3(wi), x, y, d[0]);
        from3(g_n, x); from3(g_wi, y);
    }
};
struct Frostbite {
    static constexpr Arg arg[] = {{"nrm", 3}, {"wi", 3}, {"wo", 3}, {"lin_rough", 1}};
    static constexpr int OUT = 1;
    __device__ void fwd(In<3> n, In<3> wi, In<3> wo, In<1> lr, Out<1> o) const { o[0] = fwd_frostbite(to3(n), to3(wi), to3(wo), lr[0]); }
    __device__ void bwd(In<3> n, In<3> wi, In<3> wo, In<1> lr, Out<3> g_n, Out<3> g_wi, Out<3> g_wo, Out<1> g_lr, In<1> d) const
    {
        f3 x = F3(0.0f), y = F3(0.0f), z = F3(0.0f); float dl = 0.0f;
        bwd_frostbite(to3(n), to3(wi), to3(wo), lr[0], x, y, z, dl, d[0]);
        from3(g_n, x); from3(g_wi, y); from3(g_wo, z); g_lr[0] = dl;
    }
};
struct Fresnel {
    static constexpr Arg arg[] = {{"f0", 3}, {"f90", 3}, {"cos_theta", 1}};
    static constexpr int OUT = 3;
    __device__ void fwd(In<3> f0, In<3> f90, In<1> c, Out<3> o) const { from3(o, fwd_fresnel3(to3(f0), to3(f90), c[0])); }
    __device__ void bwd(In<3> f0, In<3> f90, In<1> c, Out<3> g_f0, Out<3> g_f90, Out<1> g_c, In<3> d) const
    {
        f3 x = F3(0.0f), y = F3(0.0f); float z = 0.0f;
        bwd_fresnel3(to3(f0), to3(f90), c[0], x, y, z, to3(d));
        from3(g_f0, x); from3(g_f90, y); g_c[0] = z;
    }
};
template <int WHICH>   // 0 ndf, 1 lambda
struct Ggx2 {
    static constexpr Arg arg[] = {{"alpha_sqr", 1}, {"cos_theta", 1}};
    static constexpr int OUT = 1;
    __device__ void fwd(In<1> a2, In<1> c, Out<1> o) const { o[0] = WHICH == 0 ? fwd_ndf_ggx(a2[0], c[0]) : fwd_lambda_ggx(a2[0], c[0]); }
    __device__ void bwd(In<1> a2, In<1> c, Out<1> g_a2, Out<1> g_c, In<1> d) const
    {
        float x = 0.0f, y = 0.0f;
        if (WHICH == 0) bwd_ndf_ggx(a2[0], c[0], x, y, d[0]);
        else bwd_lambda_ggx(a2[0], c[0], x, y, d[0]);
        g_a2[0] = x; g_c[0] = y;
    }
};
struct Masking {
    static constexpr Arg arg[] = {{"alpha_sqr", 1}, {"cos_i", 1}, {"cos_o", 1}};
    static constexpr int OUT = 1;
    __device__ void fwd(In<1> a2, In<1> ci, In<1> co, Out<1> o) const { o[0] = fwd_masking_smith(a2[0], ci[0], co[0]); }
    __device__ void bwd(In<1> a2, In<1> ci, In<1> co, Out<1> g_a2, Out<1> g_ci, Out<1> g_co, In<1> d) const
    {
        float x = 0.0f, y = 0.0f, z = 0.0f;
        bwd_masking_smith(a2[0], ci[0], co[0], x, y, z, d[0]);
        g_a2[0] = x; g_ci[0] = y; g_co[0] = z;
    }
};
struct Spec {
    float min_roughness;
    static constexpr Arg arg[] = {{"col", 3}, {"nrm", 3}, {"wo", 3}, {"wi", 3}, {"alpha", 1}};
    static constexpr int OUT = 3;
    __device__ void fwd(In<3> col, In<3> n, In<3> wo, In<3> wi, In<1> al, Out<3> o) const
    {
        from3(o, fwd_pbr_specular(to3(col), to3(n), to3(wo), to3(wi), al[0], min_roughness));
    }
    __device__ void bwd(In<3> col, In<3> n, In<3> wo, In<3> wi, In<1> al, Out<3> g_col, Out<3> g_n, Out<3> g_wo, Out<3> g_wi, Out<1> g_al,
                        In<3> d) const
    {
        f3 x = F3(0.0f), y = F3(0.0f), z = F3(0.0f), w = F3(0.0f); float da = 0.0f;
        bwd_pbr_specular(to3(col), to3(n), to3(wo), to3(wi), al[0], min_roughness, x, y, z, w, da, to3(d));
        from3(g_col, x); from3(g_n, y); from3(g_wo, z); from3(g_wi, w); g_al[0] = da;
    }
};
struct Pbr {
    float min_roughness; int bsdf;
    static constexpr Arg arg[] = {{"kd", 3}, {"arm", 3}, {"pos", 3}, {"nrm", 3}, {"view_pos", 3}, {"light_pos", 3}};
    static constexpr int OUT = 3;
    __device__ void fwd(In<3> kd, In<3> arm, In<3> pos, In<3> n, In<3> view, In<3> light, Out<3> o) const
    {
        from3(o, ru_fwd_pbr_bsdf(to3(kd), to3(arm), to3(pos), to3(n), to3(view), to3(light), min_roughness, bsdf));
    }
    __device__ void bwd(In<3> kd, In<3> arm, In<3> pos, In<3> n, In<3> view, In<3> light,
                        Out<3> g_kd, Out<3> g_arm, Out<3> g_pos, Out<3> g_n, Out<3> g_view, Out<3> g_light, In<3> d) const
    {
        f3 x0 = F3(0.0f), x1 = F3(0.0f), x2 = F3(0.0f), x3 = F3(0.0f), x4 = F3(0.0f), x5 = F3(0.0f);
        ru_bwd_pbr_bsdf(to3(kd), to3(arm), to3(pos), to3(n), to3(view), to3(light), min_roughness, bsdf, x0, x1, x2, x3, x4, x5, to3(d));
        from3(g_kd, x0); from3(g_arm, x1); from3(g_pos, x2); from3(g_n, x3); from3(g_view, x4); from3(g_light, x5);
    }
};
struct Psn {
    int two_sided, opengl;
    static constexpr Arg arg[] = {{"pos", 3}, {"view_pos", 3}, {"perturbed_nrm", 3}, {"smooth_nrm", 3}, {"smooth_tng", 3}, {"geom_nrm", 3}};
    static constexpr int OUT = 3;
    __device__ void fwd(In<3> pos, In<3> view, In<3> pn, In<3> sn, In<3> st, In<3> gn, Out<3> o) const
    {
        f3 smooth_nrm = safe_normalize(to3(sn)), smooth_tng = safe_normalize(to3(st));
        f3 view_vec = safe_normalize(to3(view) - to3(pos));
        f3 geom = to3(gn);
        f3 sh = fwd_perturb_normal(to3(pn), smooth_nrm, smooth_tng, opengl != 0);
        f3 res = (two_sided && dot(view_vec, geom) < 0.0f) ? fwd_bend_normal(view_vec, -sh, -geom) : fwd_bend_normal(view_vec, sh, geom);
        from3(o, res);
    }
    __device__ void bwd(In<3> pos, In<3> view, In<3> pn, In<3> sn, In<3> st, In<3> gn,
                        Out<3> g_pos, Out<3> g_view, Out<3> g_pn, Out<3> g_sn, Out<3> g_st, Out<3> g_gn, In<3> d) const
    {
        f3 _sn = to3(sn), _st = to3(st);
        f3 smooth_nrm = safe_normalize(_sn), smooth_tng = safe_normalize(_st);
        f3 _vv = to3(view) - to3(pos);
        f3 view_vec = safe_normalize(_vv);
        f3 geom = to3(gn), p = to3(pn);
        f3 sh = fwd_perturb_normal(p, smooth_nrm, smooth_tng, opengl != 0);
        f3 d_vv = F3(0.0f), d_sh = F3(0.0f), d_geom = F3(0.0f);
        if (two_sided && dot(view_vec, geom) < 0.0f) {
            bwd_bend_normal(view_vec, -sh, -geom, d_vv, d_sh, d_geom, to3(d));
            d_sh = -d_sh; d_geom = -d_geom;
        } else bwd_bend_normal(view_vec, sh, geom, d_vv, d_sh, d_geom, to3(d));
        f3 dp = F3(0.0f), dsn = F3(0.0f), dst = F3(0.0f);
        bwd_perturb_normal(p, smooth_nrm, smooth_tng, dp, dsn, dst, d_sh, opengl != 0);
        f3 d__vv = F3(0.0f), d__sn = F3(0.0f), d__st = F3(0.0f);
        bwd_safe_normalize(_vv, d__vv, d_vv);
        bwd_safe_normalize(_sn, d__sn, dsn);
        bwd_safe_normalize(_st, d__st, dst);
        from3(g_pos, -d__vv); from3(g_view, d__vv); from3(g_pn, dp); from3(g_sn, d__sn); from3(g_st, d__st); from3(g_gn, d_geom);
    }
};
// Tail of render.shade(), render/render.py:119-131 (row f3): normalise the two denoiser outputs (rgb weighted sum, weight) and recombine
// the demodulated signals:  shaded = (A.rgb / A.w) * kd * (1 - ks.z) + B.rgb / B.w   ('pbr');   shaded = (A.rgb / A.w) * kd   ('diffuse' / 'white').
// One launch instead of ~8 torch element-wise kernels forward and ~14 backward.  In 'diffuse', b4 / ks are not read and d_b4 / d_ks
// are not written: the Python op passes d_a4 / d_kd in their place.
struct Combine {
    int pbr;
    static constexpr Arg arg[] = {{"a4", 4}, {"b4", 4, true}, {"kd", 3}, {"ks", 3, true}};
    static constexpr int OUT = 3;
    __device__ void fwd(In<4> A, In<4> B, In<3> d, In<3> s, Out<3> o) const
    {
        const float ia = 1.0f / A[3], m = pbr ? 1.0f - s[2] : 1.0f, ib = pbr ? 1.0f / B[3] : 0.0f;
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c] = A[c] * ia * d[c] * m + (pbr ? B[c] * ib : 0.0f);
    }
    __device__ void bwd(In<4> A, In<4> B, In<3> d, In<3> s, Out<4> gA, Out<4> gB, Out<3> gd, Out<3> gs, In<3> go) const
    {
        const float ia = 1.0f / A[3], m = pbr ? 1.0f - s[2] : 1.0f, ib = pbr ? 1.0f / B[3] : 0.0f;
        float gaw = 0.0f, gbw = 0.0f, gm = 0.0f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float da = A[c] * ia;                       // demodulated diffuse
            gA[c] = go[c] * d[c] * m * ia;
            gaw -= go[c] * d[c] * m * da * ia;
            gd[c] = go[c] * da * m;
            gm += go[c] * da * d[c];
            gB[c] = pbr ? go[c] * ib : 0.0f;
            gbw -= pbr ? go[c] * B[c] * ib * ib : 0.0f;
        }
        gA[3] = gaw; gB[3] = gbw;
        gs[0] = 0.0f; gs[1] = 0.0f; gs[2] = pbr ? -gm : 0.0f;
    }
};
__host__ __device__ __forceinline__ bool opt_on(const Combine &op) { return op.pbr != 0; }

// pick<I>(x...): the I-th element of the pack x.
template <size_t I, class A, class... B> __device__ __forceinline__ decltype(auto) pick(A &a, B &...b)
{
    if constexpr (I == 0) return (a); else return pick<I - 1>(b...);
}

// ew_kernel's parameter for Op's forward (BWD = false) or backward: one TIn per operand (then d_out in the backward), the op's scalars
// and its output pointers.  A thread's pixel values sit in one float[4][C] per slot: the operands, then the output (forward) or d_out
// (backward), then one gradient per operand.  Loads and stores take required operands first, then d_out, then the optional ones.
template <class Op, bool BWD>
struct Ew {
    static constexpr size_t NIN = sizeof(Op::arg) / sizeof(Arg);
    static constexpr size_t NSLOT = BWD ? 2 * NIN + 1 : NIN + 1;
    TIn in[NIN + BWD];
    Op op;
    float *out[BWD ? NIN : 1];

    template <size_t S> static constexpr int CH = S < NIN ? Op::arg[S].C : S == NIN ? Op::OUT : Op::arg[S - NIN - 1].C;
    template <size_t I> static constexpr bool IS_OPT = I < NIN && Op::arg[I].opt;
    template <bool FULL, bool OPT, size_t I, int C> __device__ __forceinline__ void load(const Grid &g, const Px4 &q, float (&x)[4][C]) const
    {
        if constexpr (IS_OPT<I> == OPT) ew_load<C, FULL>(in[I], g, q, x);
    }
    template <bool FULL, bool OPT, size_t I, int C> __device__ __forceinline__ void store(const Px4 &q, float (&x)[4][C]) const
    {
        if constexpr (IS_OPT<I> == OPT) ew_store<C, FULL>(out[I], q, x);
    }
    // Declares the slots one call level each, so that each is a local array of its own: nvcc then emits the code it emits for
    // hand-declared arrays, which one struct holding every slot does not get.
    template <bool FULL, class... X> __device__ __forceinline__ void run(const Grid &g, const Px4 &q, X &...x) const
    {
        if constexpr (sizeof...(X) < NSLOT) {
            float v[4][CH<sizeof...(X)>];
            run<FULL>(g, q, x..., v);
        } else run_slots<FULL>(g, q, std::make_index_sequence<NIN>(), x...);
    }
    template <bool FULL, size_t... I, class... X>
    __device__ __forceinline__ void run_slots(const Grid &g, const Px4 &q, std::index_sequence<I...>, X &...x) const
    {
        (load<FULL, false, I>(g, q, pick<I>(x...)), ...);
        if constexpr (BWD) load<FULL, false, NIN>(g, q, pick<NIN>(x...));
        if (opt_on(op)) (load<FULL, true, I>(g, q, pick<I>(x...)), ...);
        if constexpr (!BWD) {
#pragma unroll
            for (int k = 0; k < 4; ++k) op.fwd(pick<I>(x...)[k]..., pick<NIN>(x...)[k]);
            ew_store<Op::OUT, FULL>(out[0], q, pick<NIN>(x...));
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) op.bwd(pick<I>(x...)[k]..., pick<NIN + 1 + I>(x...)[k]..., pick<NIN>(x...)[k]);
            (store<FULL, false, I>(q, pick<NIN + 1 + I>(x...)), ...);
            if (opt_on(op)) (store<FULL, true, I>(q, pick<NIN + 1 + I>(x...)), ...);
        }
    }
};

static bool mk_in(const mcs_tensor *t, const Grid &g, int C, TIn &out, const char *name)
{
    if (!(t->sizes[3] == C || t->sizes[3] == 1)) { mcs_set_error("%s must have %d channels (got %d)", name, C, t->sizes[3]); return false; }
    for (int d = 0; d < 3; ++d) {
        int full = d == 0 ? g.N : (d == 1 ? g.H : g.W);
        if (!(t->sizes[d] == full || t->sizes[d] == 1)) { mcs_set_error("%s: dim %d = %d not broadcastable to %d", name, d, t->sizes[d], full); return false; }
    }
    out.v = make_view(t);
    bool contig = t->sizes[0] == g.N && t->sizes[1] == g.H && t->sizes[2] == g.W && t->sizes[3] == C &&
                  (C == 1 || t->strides[3] == 1) && t->strides[2] == C && t->strides[1] == C * g.W && t->strides[0] == C * g.W * g.H;
    out.fast = contig && ((uintptr_t)t->ptr % 16 == 0);
    return true;
}

// Check the entry's tensors (Op's operands, then d_out in the backward) and output pointers against Op's declaration, broadcast the
// operands to their common grid (update_grid, torch_bindings.cpp:87-101), and launch one thread per 4 pixels.
template <bool BWD, class Op, size_t NT, size_t NO>
static int ew(const char *entry, mcs_stream s, const Op &decl, const mcs_tensor *const (&ts)[NT], float *const (&outs)[NO])
{
    using E = Ew<Op, BWD>;
    static_assert(NT == E::NIN + BWD && NO == (BWD ? E::NIN : 1), "one tensor per operand (and d_out), one pointer per output");
    Grid g{1, 1, 1, 0};
    for (const mcs_tensor *t : ts) {
        MCS_REQUIRE(view_ok(t), "%s: null / empty tensor argument", entry);
        g.N = t->sizes[0] > g.N ? t->sizes[0] : g.N;
        g.H = t->sizes[1] > g.H ? t->sizes[1] : g.H;
        g.W = t->sizes[2] > g.W ? t->sizes[2] : g.W;
    }
    g.npx = (int64_t)g.N * g.H * g.W;
    E op;
    op.op = decl;
    for (size_t i = 0; i < NT; ++i)
        if (!mk_in(ts[i], g, i < E::NIN ? Op::arg[i].C : Op::OUT, op.in[i], i < E::NIN ? Op::arg[i].name : "d_out")) return 1;
    for (size_t i = 0; i < NO; ++i) {
        MCS_REQUIRE(outs[i] || (BWD && Op::arg[i].opt && !opt_on(decl)), "%s: null output pointer %s%s", entry, BWD ? "d_" : "out",
                    BWD ? Op::arg[i].name : "");
        op.out[i] = outs[i];
    }
    int64_t nblocks = ((g.npx + 3) / 4 + 255) / 256;
    MCS_REQUIRE(nblocks < (1ll << 31), "elementwise grid too large");
    ew_kernel<E><<<(unsigned)nblocks, 256, 0, (cudaStream_t)s>>>(op, g);
    MCS_LAUNCH_CHECK();
    return 0;
}

// shade_combine writes its outputs at a4's [N,H,W] (and d_b4 at b4's in 'pbr') while ew() launches over the broadcast grid of every
// operand: an output operand that spans less than that grid would let the kernel write past the end of its buffers.
template <size_t N>
static bool spans_grid(const char *entry, const mcs_tensor *t, const char *name, const mcs_tensor *const (&all)[N])
{
    if (!view_ok(t)) return true;                     // ew() reports null / empty operands
    for (const mcs_tensor *o : all) {
        if (!view_ok(o)) continue;
        for (int d = 0; d < 3; ++d)
            if (o->sizes[d] > t->sizes[d]) {
                mcs_set_error("%s: %s must span the operands' grid (dim %d is %d, another operand has %d): the outputs take its shape",
                              entry, name, d, t->sizes[d], o->sizes[d]);
                return false;
            }
    }
    return true;
}

}  // namespace

extern "C" {

int mcs_lambert_fwd(const mcs_tensor *nrm, const mcs_tensor *wi, float *out, mcs_stream s)
{
    return ew<false>(__func__, s, Lambert{}, {nrm, wi}, {out});
}
int mcs_lambert_bwd(const mcs_tensor *nrm, const mcs_tensor *wi, const mcs_tensor *d_out, float *d_nrm, float *d_wi, mcs_stream s)
{
    return ew<true>(__func__, s, Lambert{}, {nrm, wi, d_out}, {d_nrm, d_wi});
}
int mcs_frostbite_fwd(const mcs_tensor *nrm, const mcs_tensor *wi, const mcs_tensor *wo, const mcs_tensor *lin_rough, float *out, mcs_stream s)
{
    return ew<false>(__func__, s, Frostbite{}, {nrm, wi, wo, lin_rough}, {out});
}
int mcs_frostbite_bwd(const mcs_tensor *nrm, const mcs_tensor *wi, const mcs_tensor *wo, const mcs_tensor *lin_rough, const mcs_tensor *d_out,
                      float *d_nrm, float *d_wi, float *d_wo, float *d_lin_rough, mcs_stream s)
{
    return ew<true>(__func__, s, Frostbite{}, {nrm, wi, wo, lin_rough, d_out}, {d_nrm, d_wi, d_wo, d_lin_rough});
}
int mcs_fresnel_shlick_fwd(const mcs_tensor *f0, const mcs_tensor *f90, const mcs_tensor *cos_theta, float *out, mcs_stream s)
{
    return ew<false>(__func__, s, Fresnel{}, {f0, f90, cos_theta}, {out});
}
int mcs_fresnel_shlick_bwd(const mcs_tensor *f0, const mcs_tensor *f90, const mcs_tensor *cos_theta, const mcs_tensor *d_out,
                           float *d_f0, float *d_f90, float *d_cos, mcs_stream s)
{
    return ew<true>(__func__, s, Fresnel{}, {f0, f90, cos_theta, d_out}, {d_f0, d_f90, d_cos});
}
int mcs_ndf_ggx_fwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_theta, float *out, mcs_stream s)
{
    return ew<false>(__func__, s, Ggx2<0>{}, {alpha_sqr, cos_theta}, {out});
}
int mcs_ndf_ggx_bwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_theta, const mcs_tensor *d_out, float *d_alpha_sqr, float *d_cos, mcs_stream s)
{
    return ew<true>(__func__, s, Ggx2<0>{}, {alpha_sqr, cos_theta, d_out}, {d_alpha_sqr, d_cos});
}
int mcs_lambda_ggx_fwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_theta, float *out, mcs_stream s)
{
    return ew<false>(__func__, s, Ggx2<1>{}, {alpha_sqr, cos_theta}, {out});
}
int mcs_lambda_ggx_bwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_theta, const mcs_tensor *d_out, float *d_alpha_sqr, float *d_cos, mcs_stream s)
{
    return ew<true>(__func__, s, Ggx2<1>{}, {alpha_sqr, cos_theta, d_out}, {d_alpha_sqr, d_cos});
}
int mcs_masking_smith_fwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_i, const mcs_tensor *cos_o, float *out, mcs_stream s)
{
    return ew<false>(__func__, s, Masking{}, {alpha_sqr, cos_i, cos_o}, {out});
}
int mcs_masking_smith_bwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_i, const mcs_tensor *cos_o, const mcs_tensor *d_out,
                          float *d_alpha_sqr, float *d_cos_i, float *d_cos_o, mcs_stream s)
{
    return ew<true>(__func__, s, Masking{}, {alpha_sqr, cos_i, cos_o, d_out}, {d_alpha_sqr, d_cos_i, d_cos_o});
}
int mcs_pbr_specular_fwd(const mcs_tensor *col, const mcs_tensor *nrm, const mcs_tensor *wo, const mcs_tensor *wi, const mcs_tensor *alpha,
                         float min_roughness, float *out, mcs_stream s)
{
    return ew<false>(__func__, s, Spec{min_roughness}, {col, nrm, wo, wi, alpha}, {out});
}
int mcs_pbr_specular_bwd(const mcs_tensor *col, const mcs_tensor *nrm, const mcs_tensor *wo, const mcs_tensor *wi, const mcs_tensor *alpha,
                         float min_roughness, const mcs_tensor *d_out,
                         float *d_col, float *d_nrm, float *d_wo, float *d_wi, float *d_alpha, mcs_stream s)
{
    return ew<true>(__func__, s, Spec{min_roughness}, {col, nrm, wo, wi, alpha, d_out}, {d_col, d_nrm, d_wo, d_wi, d_alpha});
}
int mcs_pbr_bsdf_fwd(const mcs_tensor *kd, const mcs_tensor *arm, const mcs_tensor *pos, const mcs_tensor *nrm, const mcs_tensor *view_pos,
                     const mcs_tensor *light_pos, float min_roughness, int32_t bsdf, float *out, mcs_stream s)
{
    return ew<false>(__func__, s, Pbr{min_roughness, bsdf}, {kd, arm, pos, nrm, view_pos, light_pos}, {out});
}
int mcs_pbr_bsdf_bwd(const mcs_tensor *kd, const mcs_tensor *arm, const mcs_tensor *pos, const mcs_tensor *nrm, const mcs_tensor *view_pos,
                     const mcs_tensor *light_pos, float min_roughness, int32_t bsdf, const mcs_tensor *d_out,
                     float *d_kd, float *d_arm, float *d_pos, float *d_nrm, float *d_view_pos, float *d_light_pos, mcs_stream s)
{
    return ew<true>(__func__, s, Pbr{min_roughness, bsdf}, {kd, arm, pos, nrm, view_pos, light_pos, d_out},
                    {d_kd, d_arm, d_pos, d_nrm, d_view_pos, d_light_pos});
}
int mcs_prepare_shading_normal_fwd(const mcs_tensor *pos, const mcs_tensor *view_pos, const mcs_tensor *perturbed_nrm, const mcs_tensor *smooth_nrm,
                                   const mcs_tensor *smooth_tng, const mcs_tensor *geom_nrm, int32_t two_sided_shading, int32_t opengl,
                                   float *out, mcs_stream s)
{
    return ew<false>(__func__, s, Psn{two_sided_shading, opengl}, {pos, view_pos, perturbed_nrm, smooth_nrm, smooth_tng, geom_nrm}, {out});
}
int mcs_prepare_shading_normal_bwd(const mcs_tensor *pos, const mcs_tensor *view_pos, const mcs_tensor *perturbed_nrm, const mcs_tensor *smooth_nrm,
                                   const mcs_tensor *smooth_tng, const mcs_tensor *geom_nrm, int32_t two_sided_shading, int32_t opengl,
                                   const mcs_tensor *d_out,
                                   float *d_pos, float *d_view_pos, float *d_perturbed_nrm, float *d_smooth_nrm, float *d_smooth_tng, float *d_geom_nrm,
                                   mcs_stream s)
{
    return ew<true>(__func__, s, Psn{two_sided_shading, opengl}, {pos, view_pos, perturbed_nrm, smooth_nrm, smooth_tng, geom_nrm, d_out},
                    {d_pos, d_view_pos, d_perturbed_nrm, d_smooth_nrm, d_smooth_tng, d_geom_nrm});
}

int mcs_shade_combine_fwd(const mcs_tensor *a4, const mcs_tensor *b4, const mcs_tensor *kd, const mcs_tensor *ks, int32_t pbr, float *out, mcs_stream s)
{
    const mcs_tensor *all[] = {a4, b4, kd, ks};
    if (!spans_grid(__func__, a4, "a4", all) || (pbr && !spans_grid(__func__, b4, "b4", all))) return 1;
    return ew<false>(__func__, s, Combine{pbr}, {a4, b4, kd, ks}, {out});
}
int mcs_shade_combine_bwd(const mcs_tensor *a4, const mcs_tensor *b4, const mcs_tensor *kd, const mcs_tensor *ks, int32_t pbr, const mcs_tensor *d_out,
                          float *d_a4, float *d_b4, float *d_kd, float *d_ks, mcs_stream s)
{
    const mcs_tensor *all[] = {a4, b4, kd, ks, d_out};
    if (!spans_grid(__func__, a4, "a4", all) || (pbr && !spans_grid(__func__, b4, "b4", all))) return 1;
    return ew<true>(__func__, s, Combine{pbr}, {a4, b4, kd, ks, d_out}, {d_a4, d_b4, d_kd, d_ks});
}

}  // extern "C"
