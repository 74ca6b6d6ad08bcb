// hashgrid.cu -- multiresolution hash-grid encoding (Müller et al. 2022, "Instant Neural Graphics Primitives"), the encoding behind the
// reference's MLPTexture3D (render/mlptexture.py:57-73, tiny-cuda-nn `HashGrid`): 3 input dimensions, 2 features per level, linear
// interpolation.  Semantics (the contract; the CPU oracle oracle/hashgrid.c restates it):
//
// Level table, built once on the host in double precision (nvdiffrecmc_b200/tinycudann), passed by value:
//   scale_l = fl32(base_resolution * per_level_scale^l - 1), res_l = ceil(scale_l) + 1,
//   size_l = min(next_multiple_of_8(res_l^3), 2^log2_hashmap_size) (2^log2_hashmap_size if res_l^3 >= 2^31), offset_l = sum of the sizes
//   before l; the level is dense iff res_l^3 <= size_l, hashed otherwise.  params: 2 * offset_L fp32, entry e of level l holds its two
//   features at 2 * (offset_l + e) + f.
// Per point x and level l:
//   p_d = fmaf(scale_l, x_d, 0.5f), g_d = (uint32) cvt.rmi.s32.f32(p_d) (floor, saturating, NaN -> 0), t_d = p_d - floorf(p_d);
//   corner c in 0..7 (bit 0 = x) sits at g + (c&1, c>>1&1, c>>2&1); all index arithmetic is uint32 with wrap-around:
//   dense:  idx = (cx + cy * res + cz * res^2) mod size_l   (at x_d = 1 the corner can reach res and alias into the next row: kept)
//   hashed: idx = (cx ^ cy * 2654435761 ^ cz * 805459861) mod size_l
//   w_c = (wx * wy) * wz with w_d = t_d if bit d of c is set, else 1 - t_d;
//   y[2l + f] = sum over c ascending, from 0, of w_c * v_{c,f}.
// Adjoints:
//   d params[offset_l + idx_c, f] += w_c * dy[2l + f]   (float atomics: the only order-dependent result);
//   d x_d = sum over l ascending, from 0, of scale_l * a_{l,d}, a_{l,d} = sum over c ascending, from 0, of dw_{c,d} * s_c with
//   s_c = dy[2l] * v_{c,0} + dy[2l+1] * v_{c,1} and dw_{c,d} = +-(product of the other two weights, lower dimension first), + if bit d of
//   c is set.  Deterministic (no atomics).
//   A level whose two upstream gradients are exactly zero is skipped by both adjoints: no atomics, no d x term (the accumulators start
//   at +0 and never hold -0, so skipping adds nothing that could change a bit).
// Every product and sum above is one IEEE round-to-nearest operation, never contracted (__fmul_rn / __fadd_rn); the fma of p_d is the
// only fused operation.  Every index is reduced modulo the level size, so every access stays in bounds for every input; for NaN / Inf
// inputs the values are unspecified.
#include "hashgrid.cuh"

namespace {

struct HgArgs {
    const float *x;            // [n,3]
    int64_t n;
    const float2 *params;      // [entries] pairs
    mcs_hashgrid_levels lv;
    float2 *out;               // [n, n_levels] pairs
    const float2 *dy;          // [n, n_levels] pairs
    float2 *dparams;
    float *dx;                 // [n,3]
};

enum { HG_FWD = 0, HG_BWD_PARAMS = 1, HG_BWD_DX = 2 };

// One thread per point.  The forward is level-major (blockIdx.y = level: the resident CTAs share one level's table of <= 4 MB); the
// backward passes are point-major (one thread loops over the levels in ascending order, which d x needs for its deterministic sum).
// Measured at 2 x 8 x 800^2 G-buffer points on an H100 80GB HBM3 at 400 W (DESIGN.md section 4): forward level-major 8.76-8.78 ms,
// point-major 8.79-8.81 ms; d params point-major 8.58-8.61 ms, level-major 13.40-13.41 ms; d params + d x as two point-major passes
// 13.00-13.18 ms, fused into one point-major pass 13.46-13.68 ms.
template <int MODE>
__global__ void __launch_bounds__(256) k_hashgrid(const HgArgs a)
{
    constexpr bool kPointMajor = MODE != HG_FWD;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < a.n;
    const int L = a.lv.n_levels;
    float x[3] = {0.0f, 0.0f, 0.0f};
    if (in) { x[0] = __ldg(a.x + 3 * i); x[1] = __ldg(a.x + 3 * i + 1); x[2] = __ldg(a.x + 3 * i + 2); }
    float dx[3] = {0.0f, 0.0f, 0.0f};
    const int l0 = kPointMajor ? 0 : (int)blockIdx.y, l1 = kPointMajor ? L : l0 + 1;
    for (int l = l0; l < l1; ++l) {
        const uint32_t off = a.lv.offset[l], size = a.lv.offset[l + 1] - off, res = a.lv.res[l];
        const bool dense = (a.lv.dense_mask >> l) & 1u;
        const float s = a.lv.scale[l];
        const Cell cl = hg_cell(s, x);
        float2 dy = make_float2(0.0f, 0.0f);
        if (MODE != HG_FWD && in) dy = __ldg(a.dy + i * L + l);
        const bool live = in && (MODE == HG_FWD || dy.x != 0.0f || dy.y != 0.0f);
        if (MODE == HG_FWD) {
            if (!in) continue;
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
            a.out[i * L + l] = make_float2(y0, y1);
            continue;
        }
        if (MODE & HG_BWD_PARAMS) {
            // the coarse dense levels take many points per entry (level 0 of the reference config: 4 096 entries); the hashed ones
            // rarely see two lanes of a warp on one entry, and grouping them costs more than it saves
            const bool agg = dense;
            if (agg || live) {
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    float w1[3];
                    hg_weights(cl, c, w1);
                    const float w = __fmul_rn(__fmul_rn(w1[0], w1[1]), w1[2]);
                    const uint32_t idx = hg_index(cl, c, dense, res, size);
                    hg_scatter(a.dparams + off, idx, make_float2(__fmul_rn(w, dy.x), __fmul_rn(w, dy.y)), live, agg);
                }
            }
        }
        if ((MODE & HG_BWD_DX) && live) {
            float ad[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                float w1[3];
                hg_weights(cl, c, w1);
                const float2 v = __ldg(a.params + off + hg_index(cl, c, dense, res, size));
                const float sc = __fadd_rn(__fmul_rn(dy.x, v.x), __fmul_rn(dy.y, v.y));
                const float dw[3] = {__fmul_rn(w1[1], w1[2]), __fmul_rn(w1[0], w1[2]), __fmul_rn(w1[0], w1[1])};
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    const float t = __fmul_rn(((c >> d) & 1) ? dw[d] : -dw[d], sc);
                    ad[d] = __fadd_rn(ad[d], t);
                }
            }
#pragma unroll
            for (int d = 0; d < 3; ++d) dx[d] = __fadd_rn(dx[d], __fmul_rn(s, ad[d]));
        }
    }
    if ((MODE & HG_BWD_DX) && in) { a.dx[3 * i] = dx[0]; a.dx[3 * i + 1] = dx[1]; a.dx[3 * i + 2] = dx[2]; }
}

template <int MODE>
int hg_launch(const HgArgs &a, cudaStream_t s)
{
    const unsigned blocks = (unsigned)((a.n + 255) / 256);
    const dim3 grid(blocks, MODE == HG_FWD ? a.lv.n_levels : 1);
    k_hashgrid<MODE><<<grid, 256, 0, s>>>(a);
    MCS_LAUNCH_CHECK();
    return 0;
}

int hg_validate(const char *fn, const float *x, int64_t n, const float *params, const mcs_hashgrid_levels *lv)
{
    MCS_REQUIRE(x && params && lv, "%s: null pointer", fn);
    MCS_REQUIRE(n >= 0, "%s: n must be >= 0 (got %lld)", fn, (long long)n);
    MCS_REQUIRE(n <= (int64_t)(UINT32_MAX / 2) * 256, "%s: n too large", fn);
    MCS_REQUIRE(lv->n_levels >= 1 && lv->n_levels <= 16, "%s: n_levels must be in 1..16 (got %d)", fn, lv->n_levels);
    MCS_REQUIRE(((uintptr_t)params & 7) == 0, "%s: params must be 8-byte aligned", fn);
    for (int l = 0; l <= lv->n_levels; ++l) {
        MCS_REQUIRE(lv->offset[l] % 8 == 0, "%s: offset[%d] = %u is not a multiple of 8", fn, l, lv->offset[l]);
        if (l > 0) {
            MCS_REQUIRE(lv->offset[l] >= lv->offset[l - 1], "%s: offsets not increasing at level %d", fn, l - 1);
            MCS_REQUIRE(lv->offset[l] > lv->offset[l - 1], "%s: level %d has size 0", fn, l - 1);
        }
    }
    return 0;
}

}  // namespace

extern "C" {

int mcs_hashgrid_fwd(const float *x, int64_t n, const float *params, const mcs_hashgrid_levels *lv, float *out, mcs_stream stream)
{
    if (int e = hg_validate("mcs_hashgrid_fwd", x, n, params, lv)) return e;
    MCS_REQUIRE(out != nullptr, "mcs_hashgrid_fwd: null pointer");
    MCS_REQUIRE(((uintptr_t)out & 7) == 0, "mcs_hashgrid_fwd: out must be 8-byte aligned");
    if (n == 0) return 0;
    HgArgs a{};
    a.x = x; a.n = n; a.params = (const float2 *)params; a.lv = *lv; a.out = (float2 *)out;
    return hg_launch<HG_FWD>(a, (cudaStream_t)stream);
}

int mcs_hashgrid_bwd(const float *x, int64_t n, const float *params, const mcs_hashgrid_levels *lv, const float *d_out, float *d_params,
                     float *d_x, mcs_stream stream)
{
    if (int e = hg_validate("mcs_hashgrid_bwd", x, n, params, lv)) return e;
    MCS_REQUIRE(d_out != nullptr, "mcs_hashgrid_bwd: null pointer");
    MCS_REQUIRE(d_params || d_x, "mcs_hashgrid_bwd: null pointer (d_params and d_x both null)");
    MCS_REQUIRE(((uintptr_t)d_out & 7) == 0 && ((uintptr_t)d_params & 7) == 0, "mcs_hashgrid_bwd: d_out and d_params must be 8-byte aligned");
    if (n == 0) return 0;
    HgArgs a{};
    a.x = x; a.n = n; a.params = (const float2 *)params; a.lv = *lv; a.dy = (const float2 *)d_out; a.dparams = (float2 *)d_params; a.dx = d_x;
    const cudaStream_t s = (cudaStream_t)stream;
    if (d_params)
        if (int e = hg_launch<HG_BWD_PARAMS>(a, s)) return e;
    if (d_x)
        if (int e = hg_launch<HG_BWD_DX>(a, s)) return e;
    return 0;
}

}  // extern "C"
