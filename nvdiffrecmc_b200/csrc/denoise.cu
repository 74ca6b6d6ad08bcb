// denoise.cu -- cross-bilateral (SVGF-style) denoiser, forward and transposed backward, for sm_90a.
// Replaces bilateral_denoiser_fwd_kernel / _bwd_kernel, render/optixutils/c_src/denoising.cu:14-130
// (8x8 blocks, every tap re-fetched from global memory with 2 expf + powf(.,128) + sqrtf per tap).
//
// H100 design (compute-bound: (2r+1)^2 = 529 taps/px at sigma = 2, only 48 B/px of compulsory HBM
// traffic, SURVEY.md section 8d):
//   * one CTA = 32x16 output pixels, the (32+2r)x(16+2r) halo tile of guides (normal, depth,
//     depth-gradient) and signals staged ONCE in shared memory: by the TMA unit as AoS tiles when the operands are contiguous
//     (bilateral_tma_kernel below: the path render.shade()'s fused tail and bench.py take), else by plain loads as SoA planes
//     (bilateral_kernel: strided channel slices; conflict-free: a warp reads 32 consecutive floats of a plane row);
//   * each thread produces two vertically adjacent outputs so every tap value read from shared
//     memory is used twice (halves LDS traffic, the co-limiter next to the FP32/MUFU pipes);
//   * the spatial gaussian exponent is one FMA on a running tap offset; gaussian and depth term are merged into ONE
//     ex2.approx (exp(a)*exp(b) = exp2((a+b)*log2 e)); 1/max(dz*dist, eps) = min(inv_dz * rsqrt(dist^2), 1/eps) with the
//     guarded 1/dz staged per pixel; pow(x,128) is 7 squarings -- 2 MUFU and no table look-up per tap;
//   * out-of-image taps are stored as zero normals => clamp(dot, 1e-4, 1)^128 underflows to exactly
//     0, which reproduces the reference's `continue` without a branch;
//   * the diffuse and specular signals, which render.py:120-121 filters with identical guides, can
//     share one pass (NSIG = 2): weights are computed once.
#include "common.cuh"
#include <cfloat>          // FLT_MAX
#include <cuda.h>          // CUtensorMap + the cuTensorMapEncodeTiled prototype (resolved at run time through cudaGetDriverEntryPoint: no libcuda link)

namespace {

constexpr int TILE_W = 32;
constexpr int TILE_H = 16;
constexpr float FLT_EPS_ = 0.0001f;      // denoising.cu:12
constexpr float LOG2E = 1.4426950408889634f;

// what the filter body needs besides the staged tile; both kernels' parameter blocks start with it
struct FilterParams {
    float *out[2];         // fwd: [B,H,W,4] ; bwd: [B,H,W,3]
    int B, H, W;
    int r;
    float neg_inv_2var_log2e;   // -log2(e) / (2 sigma^2)
};

struct BilateralParams {
    FilterParams f;
    TView nrm, zdz;
    TView sig[2];          // fwd: col ; bwd: out_grad (first 3 channels used)
};

// MUFU approximations without the range-handling wrappers of exp2f / __fdividef (their operands are bounded here: exponents
// <= 0, where a flushed denormal weight is indistinguishable from the reference's 1e-38; reciprocal arguments >= 1e-4)
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rsqrt_approx(float x) { float y; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// 1 / max(dz * dist, 1e-4) = min(inv_dz * rsqrt(dist^2), 1e4) with inv_dz = dz > 0 ? 1/dz : +inf  (dist = 0 -> inf -> 1e4 as well)
__device__ __forceinline__ float guarded_inv(float dz) { return dz > 0.0f ? 1.0f / dz : INFINITY; }

// denoising.cu:26,86 filter_rad: the literal 2.5 is a double, so sigma * 2.5 is rounded in double, not fp32.  The two differ whenever the
// fp32 product rounds down onto an integer: sigma = 3.2f is 3.2000000477, 8.0000001192 in double (r = 19) but exactly 8.0f in fp32 (r = 17).
static int filter_radius(float sigma) { return 2 * (int)ceil((double)sigma * 2.5) + 1; }

__device__ __forceinline__ float pow128(float x)
{
    x *= x; x *= x; x *= x; x *= x; x *= x; x *= x; x *= x;
    return x;
}

// The filter that follows staging, shared by both kernels so that their results are bit-identical by construction: centre loads, tap
// loop and epilogue.  A Tile reads the staged halo tile: tile pixel i = row * pitch + column, and the tap window of the output in column
// lx starts at column lx + col0.
//   normal(i)                     -> the normal (zero outside the image);
//   centre_depth(i, z, inv_dz)    -> depth and guarded 1/dz;
//   tap_depth(i, z, inv_dz)       -> depth, and the guarded 1/dz where BWD reads it (the forward pass weighs with the centre's);
//   signal(s, i, v)               -> the three values of signal s.
template <int NSIG, bool BWD, class Tile>
__device__ __forceinline__ void filter_tile(const Tile &t, const FilterParams &p)
{
    const int r = p.r;
    const int b = blockIdx.z;
    // two vertically adjacent outputs per thread: rows 2*ty and 2*ty+1 of the tile
    const int lx = threadIdx.x, lyA = 2 * threadIdx.y;
    f3 cn[2]; float cz[2], cdz[2];
#pragma unroll
    for (int o = 0; o < 2; ++o) {
        const int ci = (lyA + o + r) * t.pitch + r + lx + t.col0;         // r rows and r columns into the tap window
        cn[o] = t.normal(ci); t.centre_depth(ci, cz[o], cdz[o]);      // cdz = guarded 1/dz of the centre
    }
    float acc[2][NSIG][3]; float accw[2] = {0.0f, 0.0f};
#pragma unroll
    for (int o = 0; o < 2; ++o)
#pragma unroll
        for (int s = 0; s < NSIG; ++s) acc[o][s][0] = acc[o][s][1] = acc[o][s][2] = 0.0f;

    const float k2 = p.neg_inv_2var_log2e;
    for (int rr = 0; rr <= 2 * r + 1; ++rr) {
        // tap row rr of the tile serves output A at vertical offset rr - r and output B at rr - r - 1; a row outside an output's
        // window gets exponent -inf (weight exactly 0)
        const float fyA = (float)(rr - r), fyB = (float)(rr - r - 1);
        const float fy2[2] = {fyA * fyA, fyB * fyB};
        const float gy[2] = {rr <= 2 * r ? fy2[0] * k2 : -INFINITY, rr >= 1 ? fy2[1] * k2 : -INFINITY};
        const int rowoff = (lyA + rr) * t.pitch + lx + t.col0;
        float fx = (float)(-r);
        for (int cx = 0; cx <= 2 * r; ++cx, fx += 1.0f) {
            const int i = rowoff + cx;
            const float fx2 = fx * fx;
            const f3 tn = t.normal(i);
            float tz, tinv;
            t.tap_depth(i, tz, tinv);
            float sg[NSIG][3];
#pragma unroll
            for (int s = 0; s < NSIG; ++s) t.signal(s, i, sg[s]);
#pragma unroll
            for (int o = 0; o < 2; ++o) {
                const float wn = pow128(fminf(fmaxf(dot(tn, cn[o]), FLT_EPS_), 1.0f));
                // fwd: centre's dz (denoising.cu:59); bwd: tap's dz (denoising.cu:118)
                const float inv_den = fminf((BWD ? tinv : cdz[o]) * rsqrt_approx(fx2 + fy2[o]), 1.0f / FLT_EPS_);
                const float e = fmaf(fx2, k2, gy[o]) - LOG2E * (fabsf(tz - cz[o]) * inv_den);
                const float w = wn * ex2_approx(e);
#pragma unroll
                for (int s = 0; s < NSIG; ++s) {
                    acc[o][s][0] = fmaf(sg[s][0], w, acc[o][s][0]);
                    acc[o][s][1] = fmaf(sg[s][1], w, acc[o][s][1]);
                    acc[o][s][2] = fmaf(sg[s][2], w, acc[o][s][2]);
                }
                accw[o] += w;
            }
        }
    }

    const int gx = blockIdx.x * TILE_W + lx;
#pragma unroll
    for (int o = 0; o < 2; ++o) {
        const int gy = blockIdx.y * TILE_H + lyA + o;
        if (gx < p.W && gy < p.H) {
            const int64_t px = ((int64_t)b * p.H + gy) * p.W + gx;
#pragma unroll
            for (int s = 0; s < NSIG; ++s) {
                if (!BWD) reinterpret_cast<float4 *>(p.out[s])[px] = make_float4(acc[o][s][0], acc[o][s][1], acc[o][s][2], fmaxf(accw[o], 0.0001f));
                else { float *d = p.out[s] + px * 3; d[0] = acc[o][s][0]; d[1] = acc[o][s][1]; d[2] = acc[o][s][2]; }
            }
        }
    }
}

// SoA planes staged by bilateral_kernel (pitch = tw, halo r on both sides): a warp reads 32 consecutive floats of a plane row, conflict-free
template <bool BWD>
struct SoaTile {
    static constexpr int col0 = 0;
    const float *nx, *ny, *nz, *z, *inv_dz;
    const float *sig;          // NSIG * 3 planes
    int plane, pitch;
    __device__ __forceinline__ f3 normal(int i) const { return F3(nx[i], ny[i], nz[i]); }
    __device__ __forceinline__ void centre_depth(int i, float &cz, float &cinv) const { cz = z[i]; cinv = inv_dz[i]; }
    __device__ __forceinline__ void tap_depth(int i, float &tz, float &tinv) const { tz = z[i]; tinv = BWD ? inv_dz[i] : 0.0f; }
    __device__ __forceinline__ void signal(int s, int i, float (&v)[3]) const
    {
        v[0] = sig[(3 * s + 0) * plane + i]; v[1] = sig[(3 * s + 1) * plane + i]; v[2] = sig[(3 * s + 2) * plane + i];
    }
};

template <int NSIG, bool BWD>
__global__ void __launch_bounds__(256) bilateral_kernel(BilateralParams p)
{
    extern __shared__ float smem[];
    const int r = p.f.r;
    const int tw = TILE_W + 2 * r, th = TILE_H + 2 * r;
    const int plane = tw * th;
    float *s_nx = smem, *s_ny = s_nx + plane, *s_nz = s_ny + plane, *s_z = s_nz + plane, *s_dz = s_z + plane;
    float *s_sig = s_dz + plane;                       // NSIG * 3 planes

    const int tid = threadIdx.y * blockDim.x + threadIdx.x;
    const int b = blockIdx.z;
    const int x0 = blockIdx.x * TILE_W - r, y0 = blockIdx.y * TILE_H - r;

    for (int i = tid; i < plane; i += 256) {
        int ty = i / tw, tx = i - ty * tw;
        int gy = y0 + ty, gx = x0 + tx;
        bool in = gy >= 0 && gx >= 0 && gy < p.f.H && gx < p.f.W;
        f3 n = F3(0.0f); float z = 0.0f, dz = 0.0f;
        if (in) {
            n = p.nrm.ld3(b, gy, gx);
            const float *q = p.zdz.p + p.zdz.off(b, gy, gx);
            z = __ldg(q); dz = __ldg(q + p.zdz.s3);
        }
        s_nx[i] = n.x; s_ny[i] = n.y; s_nz[i] = n.z; s_z[i] = z; s_dz[i] = guarded_inv(dz);     // plane holds 1/dz (guarded)
#pragma unroll
        for (int s = 0; s < NSIG; ++s) {
            f3 c = F3(0.0f);
            if (in) c = p.sig[s].ld3(b, gy, gx);
            s_sig[(3 * s + 0) * plane + i] = c.x; s_sig[(3 * s + 1) * plane + i] = c.y; s_sig[(3 * s + 2) * plane + i] = c.z;
        }
    }
    __syncthreads();
    filter_tile<NSIG, BWD>(SoaTile<BWD>{s_nx, s_ny, s_nz, s_z, s_dz, s_sig, plane, tw}, p.f);
}

// ---------------------------------------------------------------------------------------------
// Forward and transposed (backward) filter with the halo tile staged by the TMA unit (north_star: "the bilateral denoiser is a TMA-staged tiled kernel").
// Applies when the signals and the normals are contiguous [B,H,W,3] fp32 and zdz contiguous [B,H,W,2] with 16-byte aligned bases and
// W % 4 == 0 -- the layout render.shade()'s fused tail (ou.denoise_and_combine) and bench.py hand over; strided channel slices of an
// 8-channel tensor (the reference's BilateralDenoiser.forward) have 12-byte pixel pitches that a tensor map cannot describe and
// take bilateral_kernel.  Each operand is a 3-D tensor (W * C floats, H, B); ONE thread issues one `cp.async.bulk.tensor.3d` (SASS
// UTMALDG) per operand for the box (TWP * C, TILE_H + 2r, 1) at (x0 * C, y0, b) with x0 = tile origin - (r rounded up to 4 pixels) so that
// the box starts on a 16-byte boundary, completion counted in bytes on an mbarrier.
// Out-of-image coordinates -- negative ones included -- are ZERO-FILLED by the copy engine: a zero normal makes the tap weight
// underflow to exactly 0, which is the reference's `continue` (denoising.cu:43), so the staging loop's bounds checks, index
// arithmetic and strided loads disappear.  Tiles stay AoS in shared memory: lane x reads word 3 x + c (stride 3: conflict-free);
// (depth, depth gradient) pairs are read with one 64-bit load after dz has been replaced by its guarded reciprocal in place.
// The backward pass reads its [B,H,W,4] upstream gradients with one 128-bit shared load per tap and signal.
// The tap loop is filter_tile, as in bilateral_kernel<NSIG, BWD>: results are bit-identical.
// ---------------------------------------------------------------------------------------------
struct BilateralTmaParams {
    FilterParams f;
    int twp;
    int rl;                  // left halo of the staged tile = r rounded up to a multiple of 4 pixels: the box must START on a 16-byte boundary
                             // in global memory (a start at -r pixels x 12 bytes raises "illegal instruction")
};

// AoS tiles staged by bilateral_tma_kernel (pitch = twp, left halo rl, so col0 = rl - r)
template <bool BWD>
struct TmaTile {
    const float *n, *zd, *z;   // normals [.,3]; (z, dz) pairs, dz replaced by its guarded reciprocal in the backward pass; forward: z plane
    const float *sig;          // NSIG sections of ns floats, [.,3] forward, [.,4] backward
    int ns, pitch, col0;
    __device__ __forceinline__ f3 normal(int i) const { return F3(n[3 * i], n[3 * i + 1], n[3 * i + 2]); }
    __device__ __forceinline__ void centre_depth(int i, float &cz, float &cinv) const { cz = zd[2 * i]; cinv = BWD ? zd[2 * i + 1] : guarded_inv(zd[2 * i + 1]); }
    __device__ __forceinline__ void tap_depth(int i, float &tz, float &tinv) const
    {
        if (BWD) { const float2 zz = reinterpret_cast<const float2 *>(zd)[i]; tz = zz.x; tinv = zz.y; }
        else { tz = z[i]; tinv = 0.0f; }
    }
    __device__ __forceinline__ void signal(int s, int i, float (&v)[3]) const
    {
        if (BWD) {      // one 128-bit shared load per signal (16-byte pixels: conflict-free)
            const float4 g4 = reinterpret_cast<const float4 *>(sig + s * ns)[i];
            v[0] = g4.x; v[1] = g4.y; v[2] = g4.z;
        } else { v[0] = sig[s * ns + 3 * i]; v[1] = sig[s * ns + 3 * i + 1]; v[2] = sig[s * ns + 3 * i + 2]; }
    }
};

__device__ __forceinline__ uint32_t dn_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, int c0, int c1, int c2, uint64_t *bar)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dn_smem_u32(dst)),
                 "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(dn_smem_u32(bar))
                 : "memory");
}

template <int NSIG, bool BWD>
__global__ void __launch_bounds__(256) bilateral_tma_kernel(const __grid_constant__ CUtensorMap m_nrm, const __grid_constant__ CUtensorMap m_zdz,
                                                                const __grid_constant__ CUtensorMap m_sigA, const __grid_constant__ CUtensorMap m_sigB,
                                                                BilateralTmaParams p)
{
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t bar;
    const int r = p.f.r, twp = p.twp, th = TILE_H + 2 * r;
    constexpr int CS = BWD ? 4 : 3;                 // forward: colour [.,3]; backward: out_grad [.,4] (weight channel unused, denoising.cu:122)
    const int n3 = (twp * 3 * th + 31) & ~31, n2 = (twp * 2 * th + 31) & ~31;    // 128-byte aligned sections
    const int ns = (twp * CS * th + 31) & ~31;
    float *s_n = smem, *s_zd = s_n + n3, *s_sig = s_zd + n2, *s_z = s_sig + NSIG * ns;     // s_z: forward only (depth plane)
    const int tid = threadIdx.y * blockDim.x + threadIdx.x;
    const int b = blockIdx.z;
    const int x0 = blockIdx.x * TILE_W - p.rl, y0 = blockIdx.y * TILE_H - r;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(dn_smem_u32(&bar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint32_t bytes = (uint32_t)(sizeof(float) * (size_t)twp * th * (3 + 2 + CS * NSIG));
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(dn_smem_u32(&bar)), "r"(bytes) : "memory");
        tma_load_3d(s_n, &m_nrm, x0 * 3, y0, b, &bar);
        tma_load_3d(s_zd, &m_zdz, x0 * 2, y0, b, &bar);
        tma_load_3d(s_sig, &m_sigA, x0 * CS, y0, b, &bar);
        if (NSIG == 2) tma_load_3d(s_sig + ns, &m_sigB, x0 * CS, y0, b, &bar);
    }
    __syncthreads();
    asm volatile("{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], 0;\n@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}" ::"r"(dn_smem_u32(&bar)) : "memory");
    // (z, dz) -> (z, guarded 1/dz) in place; the tap loop reads the pair with one 64-bit shared load (8-byte pixels: conflict-free)
    // the forward pass only needs the tap's depth: a de-interleaved plane (one 32-bit load; measured 1.41 vs 1.50 ms against the pair load)
    for (int i = tid; i < twp * th; i += 256) {
        if (BWD) s_zd[2 * i + 1] = guarded_inv(s_zd[2 * i + 1]);
        else s_z[i] = s_zd[2 * i];
    }
    __syncthreads();
    filter_tile<NSIG, BWD>(TmaTile<BWD>{s_n, s_zd, s_z, s_sig, ns, twp, p.rl - r}, p.f);
}

typedef CUresult (*encode_tiled_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                    const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static encode_tiled_fn tma_encoder()
{
    static encode_tiled_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (encode_tiled_fn)ptr;
    }
    return fn;
}

// contiguous [B,H,W,C] fp32, 16-byte aligned base and row pitch
static bool tma_ok(const mcs_tensor *t, int C)
{
    return t->sizes[3] == C && t->strides[3] == 1 && t->strides[2] == C && t->strides[1] == C * t->sizes[2] && t->strides[0] == C * t->sizes[2] * t->sizes[1] &&
           ((uintptr_t)t->ptr % 16 == 0) && ((size_t)t->sizes[2] * C * sizeof(float)) % 16 == 0;
}

static bool tma_encode(CUtensorMap *m, const mcs_tensor *t, int C, int twp, int th)
{
    const cuuint64_t dims[3] = {(cuuint64_t)t->sizes[2] * C, (cuuint64_t)t->sizes[1], (cuuint64_t)t->sizes[0]};
    const cuuint64_t strides[2] = {(cuuint64_t)t->sizes[2] * C * sizeof(float), (cuuint64_t)t->sizes[2] * C * sizeof(float) * t->sizes[1]};
    const cuuint32_t box[3] = {(cuuint32_t)(twp * C), (cuuint32_t)th, 1u};
    const cuuint32_t estr[3] = {1u, 1u, 1u};
    return tma_encoder()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void *>(t->ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int check_guides(const mcs_tensor *nrm, const mcs_tensor *zdz, const mcs_tensor *sig, int sig_c, const char *sig_name)
{
    MCS_REQUIRE(view_ok(nrm) && view_ok(zdz) && view_ok(sig), "bilateral: null / empty tensor argument");
    MCS_REQUIRE(nrm->sizes[3] == 3, "bilateral: nrm must have 3 channels");
    MCS_REQUIRE(zdz->sizes[3] == 2, "bilateral: zdz must have 2 channels");
    MCS_REQUIRE(sig->sizes[3] == sig_c, "bilateral: %s must have %d channels", sig_name, sig_c);
    for (int d = 0; d < 3; ++d)
        MCS_REQUIRE(nrm->sizes[d] == sig->sizes[d] && zdz->sizes[d] == sig->sizes[d], "bilateral: shape mismatch in dim %d", d);
    return 0;
}

// Every entry point: validates the operands, then filters with bilateral_tma_kernel when the operands are contiguous and its tile fits the
// tensor-map box and shared memory, else with bilateral_kernel.  sigB and outB are not read when NSIG == 1.
template <int NSIG, bool BWD>
static int launch_bilateral(const mcs_tensor *nrm, const mcs_tensor *zdz, float sigma, const mcs_tensor *sigA, const mcs_tensor *sigB, float *outA, float *outB,
                            cudaStream_t stream)
{
    constexpr int CS = BWD ? 4 : 3;
    if (int e = check_guides(nrm, zdz, sigA, CS, NSIG == 1 ? (BWD ? "out_grad" : "col") : (BWD ? "out_gradA" : "colA"))) return e;
    if (NSIG == 2)
        if (int e = check_guides(nrm, zdz, sigB, CS, BWD ? "out_gradB" : "colB")) return e;
    MCS_REQUIRE(sigma > 0.0f, "bilateral: sigma must be > 0");
    FilterParams f{};
    f.out[0] = outA; f.out[1] = outB;
    f.B = nrm->sizes[0]; f.H = nrm->sizes[1]; f.W = nrm->sizes[2];
    f.r = filter_radius(sigma);
    // Below sigma ~ 4.6e-20 the quotient overflows to -inf, and the centre tap's 0 * k2 would be NaN where the reference's -0 / (2 sigma^2)
    // gives weight 1: -FLT_MAX keeps that 0 (every other tap's exponent is still <= -FLT_MAX, weight 0).  Only once 2 sigma^2, rounded as
    // the reference rounds it (denoising.cu:25,53), is 0 (sigma ~ 2.6e-23) is k2 -inf, and then the reference's centre tap is NaN too.
    const float var = sigma * sigma, two_var = 2.0f * var;
    f.neg_inv_2var_log2e = two_var > 0.0f ? fmaxf(-LOG2E / two_var, -FLT_MAX) : -INFINITY;
    const int th = TILE_H + 2 * f.r;
    const dim3 grid((f.W + TILE_W - 1) / TILE_W, (f.H + TILE_H - 1) / TILE_H, f.B), block(32, 8, 1);

    const int rl = (f.r + 3) & ~3, twp = (TILE_W + rl + f.r + 3) & ~3;
    const size_t n3 = ((size_t)twp * 3 * th + 31) & ~(size_t)31, n2 = ((size_t)twp * 2 * th + 31) & ~(size_t)31, n1 = ((size_t)twp * th + 31) & ~(size_t)31;
    const size_t ns = ((size_t)twp * CS * th + 31) & ~(size_t)31;
    const size_t smem_tma = sizeof(float) * (n3 + n2 + NSIG * ns + (BWD ? 0 : n1));
    CUtensorMap mn, mz, ma, mb;
    const bool tma = tma_encoder() != nullptr && tma_ok(nrm, 3) && tma_ok(zdz, 2) && tma_ok(sigA, CS) && (NSIG == 1 || tma_ok(sigB, CS)) &&
                     twp * CS <= 256 && th <= 256 &&        // tensor-map box extents are limited to 256 elements
                     smem_tma <= 227 * 1024 && tma_encode(&mn, nrm, 3, twp, th) && tma_encode(&mz, zdz, 2, twp, th) &&
                     tma_encode(&ma, sigA, CS, twp, th) && tma_encode(&mb, NSIG == 2 ? sigB : sigA, CS, twp, th);
    if (tma) {
        auto kern = bilateral_tma_kernel<NSIG, BWD>;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_tma) != cudaSuccess) { mcs_set_error("bilateral (TMA): cudaFuncSetAttribute failed"); return 2; }
        kern<<<grid, block, smem_tma, stream>>>(mn, mz, ma, mb, BilateralTmaParams{f, twp, rl});
        if (cudaGetLastError() != cudaSuccess) { mcs_set_error("bilateral (TMA): launch failed"); return 2; }
        return 0;
    }

    const int tw = TILE_W + 2 * f.r;
    const size_t smem = sizeof(float) * ((size_t)(5 + 3 * NSIG) * tw * th);
    MCS_REQUIRE(smem <= 227 * 1024, "bilateral: sigma %.3f needs a %zu-byte tile (> 227 KB shared memory)", sigma, smem);
    auto kern = bilateral_kernel<NSIG, BWD>;
    MCS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, block, smem, stream>>>(BilateralParams{f, make_view(nrm), make_view(zdz), {make_view(sigA), NSIG == 2 ? make_view(sigB) : TView{}}});
    MCS_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" {

int mcs_bilateral_fwd(const mcs_tensor *col, const mcs_tensor *nrm, const mcs_tensor *zdz, float sigma, float *out, mcs_stream stream)
{
    return launch_bilateral<1, false>(nrm, zdz, sigma, col, nullptr, out, nullptr, (cudaStream_t)stream);
}

int mcs_bilateral_bwd(const mcs_tensor *nrm, const mcs_tensor *zdz, float sigma, const mcs_tensor *out_grad, float *col_grad, mcs_stream stream)
{
    return launch_bilateral<1, true>(nrm, zdz, sigma, out_grad, nullptr, col_grad, nullptr, (cudaStream_t)stream);
}

int mcs_bilateral_fwd2(const mcs_tensor *colA, const mcs_tensor *colB, const mcs_tensor *nrm, const mcs_tensor *zdz, float sigma,
                       float *outA, float *outB, mcs_stream stream)
{
    return launch_bilateral<2, false>(nrm, zdz, sigma, colA, colB, outA, outB, (cudaStream_t)stream);
}

int mcs_bilateral_bwd2(const mcs_tensor *nrm, const mcs_tensor *zdz, float sigma, const mcs_tensor *out_gradA, const mcs_tensor *out_gradB,
                       float *col_gradA, float *col_gradB, mcs_stream stream)
{
    return launch_bilateral<2, true>(nrm, zdz, sigma, out_gradA, out_gradB, col_gradA, col_gradB, (cudaStream_t)stream);
}

}  // extern "C"
