/*
 * mcshade.h -- C ABI of libmcshade.so, the H100-native (sm_90a) replacement for the nvdiffrecmc
 * per-iteration hot path.  No torch / pybind types cross this boundary: plain device pointers,
 * sizes, element strides and a CUDA stream handle.  Every entry point returns 0 on success and a
 * non-zero code on failure (mcs_last_error() then holds a message); unlike the reference
 * (render/optixutils/c_src/common.h:37-61, errors formatted then dropped) nothing fails silently.
 * All work is enqueued on `stream` and NO entry point synchronises the host (the reference forces a
 * cudaStreamSynchronize after every env_shade launch, optixutils/c_src/torch_bindings.cpp:185,269).
 *
 * Each declaration cites the reference interface it replaces (paths relative to the reference
 * repository root).
 */
#ifndef MCSHADE_H
#define MCSHADE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MCS_ABI_VERSION 2

/* Strided NHWC view of fp32 (or int32) device memory.  sizes/strides are in ELEMENTS, dims are
 * (N, H, W, C); a size-1 dimension broadcasts (stride ignored), exactly like the reference's
 * accessors (optixutils/c_src/common.h:13-27 fetch3; renderutils/c_src/tensor.h:32 nhwcIndex). */
typedef struct mcs_tensor {
    const void *ptr;
    int32_t sizes[4];
    int32_t strides[4];
} mcs_tensor;

typedef struct mcs_ctx mcs_ctx;       /* opaque; replaces OptiXStateWrapper (optixutils/c_src/optix_wrapper.h:17-37) */
typedef void *mcs_stream;             /* cudaStream_t */

/* ---- library ------------------------------------------------------------------------------- */
int mcs_abi_version(void);
const char *mcs_last_error(void);     /* thread-local message of the last failing call */

/* ---- context: replaces OptiXStateWrapper(path, cuda_home) ctor/dtor,
 *      optixutils/c_src/optix_wrapper.cpp:306-348 (no NVRTC, no OptiX: nothing to compile at run time) */
int mcs_ctx_create(mcs_ctx **out);
int mcs_ctx_destroy(mcs_ctx *ctx);

/* ---- acceleration structure: replaces optix_build_bvh(state, verts, tris, rebuild),
 *      optixutils/c_src/torch_bindings.cpp:37-116 (optixAccelBuild).
 *      verts: V x 3 fp32 contiguous, tris: T x 3 int32 contiguous (device).  rebuild != 0: full LBVH
 *      build (Morton sort + Karras topology + refit); rebuild == 0: refit boxes on the existing
 *      topology (OPTIX_BUILD_OPERATION_UPDATE).  Runs on `stream` (the reference uses stream 0). */
int mcs_bvh_build(mcs_ctx *ctx, const float *verts, int32_t V, const int32_t *tris, int32_t T, uint32_t rebuild, mcs_stream stream);

/* Test / inspection hook: copies the binary LBVH (sorted Morton keys, sorted->original triangle
 * ids, Karras children, padded node boxes) into caller-provided DEVICE buffers of sizes
 * T, T, T-1, T-1, (2T-1)*3, (2T-1)*3.  Node ids: internal 0..T-2, leaf j = T-1+j. */
int mcs_bvh_export(mcs_ctx *ctx, uint32_t *morton, int32_t *prim, int32_t *left, int32_t *right, float *lo, float *hi, mcs_stream stream);

/* Test / inspection hook: copies the shadow-ray view that env_shade walks into caller-provided DEVICE
 * buffers: the 4-wide quantised nodes (max(T-1,1) x 4 x uint4), the triangle records its leaf runs
 * index (T x 3 float4: (v0, original id), (e1, -), (e2, -)) and the grid (origin, cell, 1 / cell). */
int mcs_bvh_export_shadow(mcs_ctx *ctx, uint32_t *nodesq4, float *tris, float *qgrid, mcs_stream stream);

/* Any-hit visibility of n rays (origin, direction; t in (0, 1e16)), the "integer visibility mask":
 * vis[i] = 1 if nothing is hit.  Same predicate as the shadow rays inside env_shade; replaces
 * shadow_test()/optixTrace, optixutils/c_src/envsampling/kernel.cu:101-118. */
int mcs_trace_visibility(mcs_ctx *ctx, const float *ro, const float *rd, int64_t n, uint8_t *vis, mcs_stream stream);

/* Closest hit (primary visibility for the synthetic G-buffer producer, SURVEY.md section 8 row f2):
 * tri_id[i] = original triangle id or -1; tuv[i] = (t, u, v). */
int mcs_trace_closest(mcs_ctx *ctx, const float *ro, const float *rd, int64_t n, int32_t *tri_id, float *tuv, mcs_stream stream);

/* Closest hit beyond a per-ray bound (the ray-level form of depth peeling, see mcs_rasterize_peel): only hits with
 * t > sep(t_after[i]) count, sep(t) = fl32(t * (1 + 2^-16)); t_after[i] = +inf gives a miss.  Outputs as mcs_trace_closest. */
int mcs_trace_closest_after(mcs_ctx *ctx, const float *ro, const float *rd, const float *t_after, int64_t n, int32_t *tri_id, float *tuv,
                            mcs_stream stream);

/* ---- fused env-light importance sampling + shadow rays + BSDF:
 *      replaces env_shade_fwd / env_shade_bwd, optixutils/c_src/torch_bindings.cpp:123-188 / 190-272
 *      (optixLaunch of __raygen__rg, envsampling/kernel.cu:463-542).
 *      mask [B,H,W,1]; ro, gb_pos, gb_normal, gb_kd, gb_ks [B,H,W,3]; gb_view_pos broadcastable
 *      [B|1,H|1,W|1,3]; light [1,Hl,Wl,3]; pdf [1,Hl,Wl,1]; rows [1,Hl,1,1]; cols [1,Hl,Wl,1];
 *      perms int32 [1,P,1,N*N] (all as mcs_tensor views, arbitrary strides).
 *      bsdf: 0 'pbr', 1 'diffuse', 2 'white' (optixutils/ops.py:136).
 *      batch_offset is added to the batch index inside the per-pixel RNG hash so a rank that holds
 *      views [o, o+B) of a larger batch reproduces the single-GPU random stream (kernel.cu:504).
 *      Outputs are contiguous [B,H,W,3] fp32 and are fully written (masked pixels = 0).
 *      hit_record (optional, may be NULL): uint32 [B,H,W,ceil(2*n_samples_x^2/32)], receives one bit per sample slot
 *      w (w < N^2: light sample of stratum w; else BSDF sample of stratum w-N^2): 1 = shadow ray occluded.  Passing the
 *      same buffer to mcs_env_shade_bwd (same seed, same inputs) lets the backward pass REPLAY visibility instead of
 *      re-tracing every ray as the reference does (torch_bindings.cpp:266-267 launches the same program with backward=1).
 *      rec_count / rec_rays (optional, together): the full RAY RECORD -- rec_count uint32 [B,H,W] = number of rays that were
 *      evaluated for the pixel (visible, or occluded with shadow_scale < 1), rec_rays fp32 [B,H,W,5,rec_slots] =
 *      (dx, dy, dz, MIS weight, env texel | occluded << 31) in evaluation order, rec_slots >= 2*n_samples_x^2.  With it the
 *      backward pass needs neither sampling nor traversal: see mcs_env_shade_bwd_replay.
 *      seed_offset_dev (optional, may be NULL): DEVICE pointer to one uint32 that the kernel adds to rnd_seed when it starts.  The
 *      reference passes the seed by value from a host counter (render/render.py:19,112-116); a host value is frozen into a captured
 *      CUDA graph, a device value is not -- the training step can be captured once and replayed with an advancing seed. */
int mcs_env_shade_fwd(mcs_ctx *ctx,
                      const mcs_tensor *mask, const mcs_tensor *ro, const mcs_tensor *gb_pos, const mcs_tensor *gb_normal,
                      const mcs_tensor *gb_view_pos, const mcs_tensor *gb_kd, const mcs_tensor *gb_ks,
                      const mcs_tensor *light, const mcs_tensor *pdf, const mcs_tensor *rows, const mcs_tensor *cols,
                      const mcs_tensor *perms,
                      uint32_t bsdf, uint32_t n_samples_x, uint32_t rnd_seed, const uint32_t *seed_offset_dev, float shadow_scale, int32_t batch_offset,
                      float *diff, float *spec, uint32_t *hit_record, uint32_t *rec_count, float *rec_rays, int32_t rec_slots, mcs_stream stream);

/* Gradient outputs: gb_pos_grad, gb_normal_grad, gb_kd_grad, gb_ks_grad contiguous [B,H,W,3]
 * (fully written), light_grad contiguous [Hl,Wl,3] (zeroed by the call, then accumulated). */
int mcs_env_shade_bwd(mcs_ctx *ctx,
                      const mcs_tensor *mask, const mcs_tensor *ro, const mcs_tensor *gb_pos, const mcs_tensor *gb_normal,
                      const mcs_tensor *gb_view_pos, const mcs_tensor *gb_kd, const mcs_tensor *gb_ks,
                      const mcs_tensor *light, const mcs_tensor *pdf, const mcs_tensor *rows, const mcs_tensor *cols,
                      const mcs_tensor *perms,
                      uint32_t bsdf, uint32_t n_samples_x, uint32_t rnd_seed, const uint32_t *seed_offset_dev, float shadow_scale, int32_t batch_offset,
                      const mcs_tensor *diff_grad, const mcs_tensor *spec_grad,
                      float *gb_pos_grad, float *gb_normal_grad, float *gb_kd_grad, float *gb_ks_grad, float *light_grad,
                      const uint32_t *hit_record /* NULL = re-trace */, mcs_stream stream);

/* Backward from the ray record written by mcs_env_shade_fwd (same G-buffer, light and shadow_scale): one warp per pixel walks
 * the recorded rays and runs only the adjoint BSDF + env-map gradient scatter.  Outputs as mcs_env_shade_bwd. */
int mcs_env_shade_bwd_replay(const mcs_tensor *gb_pos, const mcs_tensor *gb_normal, const mcs_tensor *gb_view_pos, const mcs_tensor *gb_kd,
                             const mcs_tensor *gb_ks, const mcs_tensor *light, uint32_t bsdf, uint32_t n_samples_x, float shadow_scale,
                             const mcs_tensor *diff_grad, const mcs_tensor *spec_grad, const uint32_t *rec_count, const float *rec_rays, int32_t rec_slots,
                             float *gb_pos_grad, float *gb_normal_grad, float *gb_kd_grad, float *gb_ks_grad, float *light_grad, mcs_stream stream);

/* Debug/parity hook: forward pass that also records, per pixel and per ray slot
 * (slot = 2*i for the light sample of stratum i, 2*i+1 for the BSDF sample), the env texel read
 * ((y<<16)|x) and the shadow-ray result (1 visible, 0 occluded; 255/-1 for masked pixels).
 * rec_texel int32 [B,H,W,2N^2], rec_vis uint8 [B,H,W,2N^2].  Rays whose contribution is provably
 * zero are not traced by the product; their rec_vis is 2 ("skipped"). */
int mcs_env_shade_records(mcs_ctx *ctx,
                          const mcs_tensor *mask, const mcs_tensor *ro, const mcs_tensor *gb_pos, const mcs_tensor *gb_normal,
                          const mcs_tensor *gb_view_pos, const mcs_tensor *gb_kd, const mcs_tensor *gb_ks,
                          const mcs_tensor *light, const mcs_tensor *pdf, const mcs_tensor *rows, const mcs_tensor *cols,
                          const mcs_tensor *perms,
                          uint32_t bsdf, uint32_t n_samples_x, uint32_t rnd_seed, const uint32_t *seed_offset_dev, float shadow_scale, int32_t batch_offset,
                          float *diff, float *spec, int32_t *rec_texel, uint8_t *rec_vis, mcs_stream stream);

/* ---- bilateral denoiser: replaces bilateral_denoiser_fwd / _bwd,
 *      optixutils/c_src/torch_bindings.cpp:274-319 (denoising.cu:14-130).
 *      col, nrm [B,H,W,3], zdz [B,H,W,2] strided views; out contiguous [B,H,W,4]
 *      = (sum w*col, max(sum w, 1e-4)); col_grad contiguous [B,H,W,3]; out_grad [B,H,W,4] view. */
int mcs_bilateral_fwd(const mcs_tensor *col, const mcs_tensor *nrm, const mcs_tensor *zdz, float sigma, float *out, mcs_stream stream);
int mcs_bilateral_bwd(const mcs_tensor *nrm, const mcs_tensor *zdz, float sigma, const mcs_tensor *out_grad, float *col_grad, mcs_stream stream);
/* Fused fast path for the two calls render/render.py:120-121 makes with identical guides
 * (diffuse + specular): weights are computed once.  outA/outB as above. */
int mcs_bilateral_fwd2(const mcs_tensor *colA, const mcs_tensor *colB, const mcs_tensor *nrm, const mcs_tensor *zdz, float sigma,
                       float *outA, float *outB, mcs_stream stream);
int mcs_bilateral_bwd2(const mcs_tensor *nrm, const mcs_tensor *zdz, float sigma, const mcs_tensor *out_gradA, const mcs_tensor *out_gradB,
                       float *col_gradA, float *col_gradB, mcs_stream stream);

/* ---- renderutils elementwise ops: replace the *_fwd / *_bwd functions of renderutils_plugin,
 *      renderutils/c_src/torch_bindings.cpp:866-888.  Inputs are broadcastable NHWC views; the launch
 *      grid (N,H,W) is the max over inputs (update_grid, torch_bindings.cpp:87-101); outputs and
 *      gradients are contiguous full-grid fp32 (gradients of broadcast inputs are NOT reduced, as in
 *      the reference, tensor.h:61,75 -- the autograd wrapper sums them). */
int mcs_lambert_fwd(const mcs_tensor *nrm, const mcs_tensor *wi, float *out, mcs_stream s);                                   /* torch_bindings.cpp:255 */
int mcs_lambert_bwd(const mcs_tensor *nrm, const mcs_tensor *wi, const mcs_tensor *d_out, float *d_nrm, float *d_wi, mcs_stream s);
int mcs_frostbite_fwd(const mcs_tensor *nrm, const mcs_tensor *wi, const mcs_tensor *wo, const mcs_tensor *lin_rough, float *out, mcs_stream s);
int mcs_frostbite_bwd(const mcs_tensor *nrm, const mcs_tensor *wi, const mcs_tensor *wo, const mcs_tensor *lin_rough, const mcs_tensor *d_out,
                      float *d_nrm, float *d_wi, float *d_wo, float *d_lin_rough, mcs_stream s);
int mcs_fresnel_shlick_fwd(const mcs_tensor *f0, const mcs_tensor *f90, const mcs_tensor *cos_theta, float *out, mcs_stream s);
int mcs_fresnel_shlick_bwd(const mcs_tensor *f0, const mcs_tensor *f90, const mcs_tensor *cos_theta, const mcs_tensor *d_out,
                           float *d_f0, float *d_f90, float *d_cos, mcs_stream s);
int mcs_ndf_ggx_fwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_theta, float *out, mcs_stream s);
int mcs_ndf_ggx_bwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_theta, const mcs_tensor *d_out, float *d_alpha_sqr, float *d_cos, mcs_stream s);
int mcs_lambda_ggx_fwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_theta, float *out, mcs_stream s);
int mcs_lambda_ggx_bwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_theta, const mcs_tensor *d_out, float *d_alpha_sqr, float *d_cos, mcs_stream s);
int mcs_masking_smith_fwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_i, const mcs_tensor *cos_o, float *out, mcs_stream s);
int mcs_masking_smith_bwd(const mcs_tensor *alpha_sqr, const mcs_tensor *cos_i, const mcs_tensor *cos_o, const mcs_tensor *d_out,
                          float *d_alpha_sqr, float *d_cos_i, float *d_cos_o, mcs_stream s);
int mcs_pbr_specular_fwd(const mcs_tensor *col, const mcs_tensor *nrm, const mcs_tensor *wo, const mcs_tensor *wi, const mcs_tensor *alpha,
                         float min_roughness, float *out, mcs_stream s);
int mcs_pbr_specular_bwd(const mcs_tensor *col, const mcs_tensor *nrm, const mcs_tensor *wo, const mcs_tensor *wi, const mcs_tensor *alpha,
                         float min_roughness, const mcs_tensor *d_out,
                         float *d_col, float *d_nrm, float *d_wo, float *d_wi, float *d_alpha, mcs_stream s);
/* pbr_bsdf_fwd / pbr_bsdf_bwd, renderutils/c_src/torch_bindings.cpp:653-722; bsdf: 0 lambert, 1 frostbite */
int mcs_pbr_bsdf_fwd(const mcs_tensor *kd, const mcs_tensor *arm, const mcs_tensor *pos, const mcs_tensor *nrm, const mcs_tensor *view_pos,
                     const mcs_tensor *light_pos, float min_roughness, int32_t bsdf, float *out, mcs_stream s);
int mcs_pbr_bsdf_bwd(const mcs_tensor *kd, const mcs_tensor *arm, const mcs_tensor *pos, const mcs_tensor *nrm, const mcs_tensor *view_pos,
                     const mcs_tensor *light_pos, float min_roughness, int32_t bsdf, const mcs_tensor *d_out,
                     float *d_kd, float *d_arm, float *d_pos, float *d_nrm, float *d_view_pos, float *d_light_pos, mcs_stream s);
/* prepare_shading_normal_fwd / _bwd, renderutils/c_src/torch_bindings.cpp:170-250 (normal.cu:95-178) */
int mcs_prepare_shading_normal_fwd(const mcs_tensor *pos, const mcs_tensor *view_pos, const mcs_tensor *perturbed_nrm, const mcs_tensor *smooth_nrm,
                                   const mcs_tensor *smooth_tng, const mcs_tensor *geom_nrm, int32_t two_sided_shading, int32_t opengl,
                                   float *out, mcs_stream s);
int mcs_prepare_shading_normal_bwd(const mcs_tensor *pos, const mcs_tensor *view_pos, const mcs_tensor *perturbed_nrm, const mcs_tensor *smooth_nrm,
                                   const mcs_tensor *smooth_tng, const mcs_tensor *geom_nrm, int32_t two_sided_shading, int32_t opengl,
                                   const mcs_tensor *d_out,
                                   float *d_pos, float *d_view_pos, float *d_perturbed_nrm, float *d_smooth_nrm, float *d_smooth_tng, float *d_geom_nrm,
                                   mcs_stream s);

/* ---- image loss (SURVEY section 8 row f3): replaces image_loss_fwd / image_loss_bwd, renderutils/c_src/torch_bindings.cpp:739-800
 *      (loss.cu:105-227).  loss: 0 l1, 1 mse, 2 relmse, 3 smape, 4 n2n (FIX: the reference's strToLoss maps "n2n" to l1);
 *      tonemapper: 0 none, 1 log_srgb.  Forward writes mcs_image_loss_num_partials(N,H,W) deterministic per-CTA partial sums of
 *      mean_c(loss) -- the caller sums them and divides by N*H*W exactly like renderutils/ops.py:494.  Backward takes the upstream
 *      gradient of those partials ([P,1,1,1] view, or one broadcast value) and writes contiguous [N,H,W,3] gradients. */
int mcs_image_loss_num_partials(int32_t N, int32_t H, int32_t W);
int mcs_image_loss_fwd(const mcs_tensor *img, const mcs_tensor *target, int32_t loss, int32_t tonemapper, float *partials, mcs_stream s);
int mcs_image_loss_bwd(const mcs_tensor *img, const mcs_tensor *target, int32_t loss, int32_t tonemapper, const mcs_tensor *d_partials,
                       float *d_img, float *d_target, mcs_stream s);

/* ---- batched 4x4 transform (row f3): replaces xfm_fwd / xfm_bwd, renderutils/c_src/torch_bindings.cpp:803-864 (mesh.cu:19-90).
 *      points as a (1|B, V, 3, 1) view, matrix as (B, 4, 4, 1); out contiguous [B,V,4] (is_points) or [B,V,3] (vectors);
 *      d_out (B, V, 4|3, 1) view; d_points contiguous [B,V,3] (a broadcast input's gradient is reduced by the caller). */
int mcs_xfm_fwd(const mcs_tensor *points, const mcs_tensor *matrix, int32_t is_points, float *out, mcs_stream s);
int mcs_xfm_bwd(const mcs_tensor *points, const mcs_tensor *matrix, const mcs_tensor *d_out, int32_t is_points, float *d_points, mcs_stream s);

/* ---- tail of render.shade() (row f3): normalise the denoiser outputs and recombine the demodulated signals, render/render.py:119-131.
 *      a4 / b4: [B,H,W,4] raw bilateral outputs (rgb weighted sum, weight) of the diffuse / specular signal; kd, ks [B,H,W,3];
 *      pbr != 0: out = a.rgb/a.w * kd * (1 - ks.z) + b.rgb/b.w ;  pbr == 0 ('diffuse' / 'white'): out = a.rgb/a.w * kd (b4, ks ignored but
 *      must be valid views).  Backward writes contiguous gradients for a4, kd (and b4, ks when pbr).  Every output has a4's [B,H,W], so
 *      a4 (and b4 when pbr) must span the broadcast grid of all operands (d_out included); kd / ks / d_out may broadcast.  An a4 / b4
 *      smaller than that grid is an error, reported before any launch. */
int mcs_shade_combine_fwd(const mcs_tensor *a4, const mcs_tensor *b4, const mcs_tensor *kd, const mcs_tensor *ks, int32_t pbr, float *out, mcs_stream s);
int mcs_shade_combine_bwd(const mcs_tensor *a4, const mcs_tensor *b4, const mcs_tensor *kd, const mcs_tensor *ks, int32_t pbr, const mcs_tensor *d_out,
                          float *d_a4, float *d_b4, float *d_kd, float *d_ks, mcs_stream s);

/* ---- primary visibility + attribute interpolation (SURVEY section 8 row f2): stands in for dr.rasterize / dr.interpolate of nvdiffrast at
 *      the call sites render/render.py:208-234 (closest hit on the context's LBVH instead of rasterisation).
 *      mtx: [B,4,4] row-major fp32 device array, clip = mtx * (p, 1) (inverted on the device, no host round trip).  rast: [B,H,W,4] contiguous, nvdiffrast
 *      convention (u, v, z/w, triangle_id + 1) with u / v the barycentric weights of vertex 0 / 1; all zero = background.
 *      interpolate: attr [V,C] (attr_batch_stride 0) or [B,V,C] (stride V*C), tris int32 [T,3], out / d_out [B,H,W,C];
 *      d_attr (same layout as attr) must be zeroed by the caller and receives float atomics. */
int mcs_rasterize(mcs_ctx *ctx, const float *mtx, int32_t B, int32_t H, int32_t W, float *rast, mcs_stream stream);
/* Depth peeling, the stand-in for dr.DepthPeeler (render/render.py:308-311): one layer per call.  t_state: [B,H,W] fp32 device array,
 * in/out, zero-filled by the caller before layer 0; it holds each pixel's last hit t along the un-projected near-far segment, or +inf
 * once the pixel is exhausted.  Layer k+1 is the closest hit with t > sep(t_prev), sep(t) = fl32(t * (1 + 2^-16)): surfaces closer
 * than that along the ray merge into one layer, so a ray through a shared edge does not return the same surface twice.  Layer 0 equals
 * mcs_rasterize bit for bit; an exhausted pixel is all zeros.  rast as mcs_rasterize.  No host sync (a peel loop can be captured in a
 * CUDA graph); the BVH must not be rebuilt or refitted between the layers of one peel. */
int mcs_rasterize_peel(mcs_ctx *ctx, const float *mtx, int32_t B, int32_t H, int32_t W, float *t_state, float *rast, mcs_stream stream);
int mcs_interpolate_fwd(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                        int32_t B, int32_t H, int32_t W, float *out, mcs_stream stream);
int mcs_interpolate_bwd(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                        int32_t B, int32_t H, int32_t W, const float *d_out, float *d_attr, mcs_stream stream);

/* ---- geometry gradients through the G-buffer: the silhouette term of geometry/dlmesh.py:75 (alpha of render_mesh's composite_buffer,
 *      render/render.py:290, where dr.antialias runs on every buffer) needs d rast / d pos.  pos: clip-space vertices [V,4]
 *      (pos_batch_stride 0) or [B,V,4] (stride V*4), fp32 contiguous; it must equal mtx * (verts, 1) for the vertices the BVH was built from.
 *      d_pos (same layout as pos) must be zeroed by the caller and receives float atomics; z and the id channel carry no gradient.
 *   rasterize_bwd: d_rast [B,H,W,4] -> d_pos through the perspective-correct barycentrics of pos (derivation in csrc/raster.cu).
 *   interpolate_bwd_rast: as mcs_interpolate_bwd, plus d_rast [B,H,W,4] = (sum_c g (A0 - A2), sum_c g (A1 - A2), 0, 0) written for every
 *      pixel; d_attr may be null (no attribute gradient).
 *   aa_topology: adj int32 [T,3], adj[t,k] = the triangle across edge (tri[t,k], tri[t,(k+1)%3]), -1 boundary, -2 three or more triangles;
 *      workspace: mcs_aa_topology_workspace_bytes(T) bytes, 8-byte aligned, device memory, contents ignored on entry.
 *   antialias: pixel-pair analytic antialiasing of color [B,H,W,C] (C >= 1, contiguous) given rast, pos, tris and adj; out [B,H,W,C].
 *      The backward writes d_color [B,H,W,C] (overwritten, may be null) and adds into d_pos (may be null; not both null).
 *      Semantics in csrc/raster.cu. */
int mcs_rasterize_bwd(const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const float *rast, int32_t B, int32_t H,
                      int32_t W, const float *d_rast, float *d_pos, mcs_stream stream);
int mcs_interpolate_bwd_rast(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                             int32_t B, int32_t H, int32_t W, const float *d_out, float *d_attr, float *d_rast, mcs_stream stream);

/* ---- screen-space derivatives (render/render.py:225-234: dr.interpolate(..., rast_db=, diff_attrs='all') builds gb_texc_deriv and the
 *      denoiser's depth guide gb_depth); semantics in csrc/raster.cu.  pos / tris / rast as mcs_rasterize_bwd.
 *   rast_db: rast_db [B,H,W,4] = (du/dX, du/dY, dv/dX, dv/dY) in pixels (nvdiffrast's layout) for the triangle id stored in rast, from pos
 *      alone; 0 for background, ids >= T and degenerate (S == 0) pixels.  Bit-reproducible (explicitly rounded).
 *   rasterize_bwd_db: d_rast (may be null) and d_rast_db [B,H,W,4] -> d_pos (caller-zeroed, float atomics).
 *   interpolate_da: out_da [B,H,W,2*n_diff], channels 2k / 2k+1 = (dA/dX, dA/dY) of the k-th selected attribute; diff_idx is a HOST array of
 *      n_diff (1..32) indices in [0, C), repeats allowed, or NULL for all C attributes in order (then n_diff must equal C).  The backward
 *      adds into d_attr (caller-zeroed, float atomics; may be null) and overwrites d_rast_db [B,H,W,4] (may be null; not both null). */
int mcs_rast_db(const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const float *rast, int32_t B, int32_t H,
                int32_t W, float *rast_db, mcs_stream stream);
int mcs_rasterize_bwd_db(const float *pos, int64_t pos_batch_stride, int32_t V, const int32_t *tris, int32_t T, const float *rast, int32_t B,
                         int32_t H, int32_t W, const float *d_rast, const float *d_rast_db, float *d_pos, mcs_stream stream);
int mcs_interpolate_da_fwd(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                           const float *rast_db, int32_t B, int32_t H, int32_t W, int32_t n_diff, const int32_t *diff_idx, float *out_da,
                           mcs_stream stream);
int mcs_interpolate_da_bwd(const float *attr, int64_t attr_batch_stride, int32_t V, int32_t C, const int32_t *tris, int32_t T, const float *rast,
                           const float *rast_db, int32_t B, int32_t H, int32_t W, int32_t n_diff, const int32_t *diff_idx, const float *d_out_da,
                           float *d_attr, float *d_rast_db, mcs_stream stream);

int64_t mcs_aa_topology_workspace_bytes(int32_t T);
int mcs_aa_topology(const int32_t *tris, int32_t T, void *workspace, int32_t *adj, mcs_stream stream);
int mcs_antialias_fwd(const float *color, int32_t C, const float *rast, int32_t B, int32_t H, int32_t W, const float *pos, int64_t pos_batch_stride,
                      int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, float *out, mcs_stream stream);
int mcs_antialias_bwd(const float *color, int32_t C, const float *rast, int32_t B, int32_t H, int32_t W, const float *pos, int64_t pos_batch_stride,
                      int32_t V, const int32_t *tris, int32_t T, const int32_t *adj, const float *d_out, float *d_color, float *d_pos, mcs_stream stream);

/* Nearest-texel fetch out[i,:] = tex[idx[i],:] (tex [T,C] contiguous, idx int64 [n]; out-of-range indices give zeros) and its scatter-add
 * backward into a caller-zeroed d_tex [T,C] (float atomics) -- the material look-up of the synthetic G-buffer producer. */
int mcs_texel_fetch_fwd(const float *tex, int64_t T, int32_t C, const int64_t *idx, int64_t n, float *out, mcs_stream stream);
int mcs_texel_fetch_bwd(int64_t T, int32_t C, const int64_t *idx, int64_t n, const float *d_out, float *d_tex, mcs_stream stream);

/* ---- env-light pdf / CDF tables (SURVEY section 8 row a17): replaces the torch-op chain of EnvironmentLight.update_pdf,
 *      render/light.py:46-59.  base: (1, Hl, Wl, 3) view.  Outputs (caller-allocated, contiguous): pdf [Hl,Wl] normalised to sum 1,
 *      rows [Hl] (what the call site passes as lgt.rows[:,0], render/render.py:114), cols [Hl,Wl]; row_totals: Hl doubles of scratch
 *      (holds the un-normalised row sums on return).  Sums are carried in fp64 and rounded once. */
int mcs_update_pdf(const mcs_tensor *base, float *pdf, float *rows, float *cols, double *row_totals, mcs_stream s);

/* ---- multiresolution hash-grid encoding: stands in for tiny-cuda-nn's `HashGrid` Encoding behind MLPTexture3D (render/mlptexture.py:57-73),
 *      3 input dimensions, 2 features per level, linear interpolation; semantics in csrc/hashgrid.cu.
 *      The level table is built on the host (nvdiffrecmc_b200/tinycudann) and passed by value: offset[l] is the first entry of level l
 *      (offset[n_levels] = total entries; non-decreasing multiples of 8, every level non-empty), res / scale its resolution and scale,
 *      bit l of dense_mask set for a dense level.  x [n,3], out / d_out [n, 2*n_levels], params / d_params [2 * offset[n_levels]], d_x [n,3]:
 *      fp32, contiguous; params, out, d_out, d_params 8-byte aligned.  The backward adds into d_params (caller-zeroed, float atomics; may be
 *      null) and overwrites d_x (deterministic; may be null; not both null).  n = 0 is a no-op.  No host sync, no allocation. */
typedef struct mcs_hashgrid_levels {
    int32_t n_levels;
    uint32_t offset[17];
    uint32_t res[16];
    float scale[16];
    uint32_t dense_mask;
} mcs_hashgrid_levels;
int mcs_hashgrid_fwd(const float *x, int64_t n, const float *params, const mcs_hashgrid_levels *lv, float *out, mcs_stream stream);
int mcs_hashgrid_bwd(const float *x, int64_t n, const float *params, const mcs_hashgrid_levels *lv, const float *d_out, float *d_params,
                     float *d_x, mcs_stream stream);

/* ---- MLP texture: MLPTexture3D.sample (render/mlptexture.py:86-96) fused, one forward kernel and one backward kernel (plus a d W sum over
 *      chunks); semantics in csrc/mlptexture.cu.  t [n,3] points, aabb [2,3], min_max [2,channels] (row 0 = lo, row 1 = hi), device fp32,
 *      contiguous.  params / lv: the hash-grid encoding as mcs_hashgrid_*, with lv->n_levels == 16.  weights: a HOST array of hidden + 1
 *      device pointers, torch Linear.weight layout [out, in] row-major: weights[l] is [32,32] for l < hidden, weights[hidden] [channels,32];
 *      hidden in 1..4, channels in 1..8.  out [n,channels] is overwritten.  enc [n,32]: the encoding, written by the forward when non-null
 *      (needed by the backward) and read by the backward; 16-byte aligned.
 *      The backward adds into d_params (caller-zeroed, float atomics, 8-byte aligned; may be null), overwrites d_t [n,3] (may be null) and
 *      overwrites d_weights[l] (d_weights is a HOST array of hidden + 1 device pointers; it or any entry may be null) -- the true gradients,
 *      at least one requested.  d W is deterministic: chunk partials over MCS_MLPTEX_CHUNK consecutive points are written to `workspace`
 *      (mcs_mlptex_workspace_bytes(n, hidden, channels) bytes of device memory, 16-byte aligned, contents ignored on entry; needed only for
 *      d W) and summed in chunk order.  n = 0 is a no-op (d W zeroed).  No host sync, no allocation. */
#define MCS_MLPTEX_CHUNK 1024
int64_t mcs_mlptex_workspace_bytes(int64_t n, int32_t hidden, int32_t channels);
int mcs_mlptex_fwd(const float *t, int64_t n, const float *aabb, const float *min_max, const float *params, const mcs_hashgrid_levels *lv,
                   int32_t hidden, int32_t channels, const float *const *weights, float *out, float *enc, mcs_stream stream);
int mcs_mlptex_bwd(const float *t, int64_t n, const float *aabb, const float *min_max, const float *params, const mcs_hashgrid_levels *lv,
                   int32_t hidden, int32_t channels, const float *const *weights, const float *enc, const float *d_out, float *d_params,
                   float *d_t, float *const *d_weights, void *workspace, mcs_stream stream);

/* ---- filtered, mip-mapped texture sampling: stands in for nvdiffrast's `dr.texture` in Texture2D.sample and its mip chain's backward
 *      (render/texture.py:27-30,57-68), the regulariser taps (render/render.py:54,75-95) and the probe look-ups (render/light.py:64,76);
 *      semantics in csrc/texture.cu.  The level table is passed by value: level k is ptr[k], [Bt, h[k], w[k], C] fp32 contiguous, with
 *      h[k] = max(1, h[0] >> k), w[k] = max(1, w[0] >> k); batch_stride[k] = 0 shares the level over the minibatch, else h*w*C (every
 *      level alike).  uv [B,H,W,2], uv_da [B,H,W,4] (du/dX, du/dY, dv/dX, dv/dY; required by linear-mipmap-linear, else ignored), out and
 *      d_out [B,H,W,C], contiguous fp32; uv 8-byte and uv_da 16-byte aligned.  MCS_TEX_LINEAR reads level 0 only.
 *      The backward adds into d_tex[k] (a HOST array of n_levels device pointers, caller-zeroed, float atomics; the array or any entry may be
 *      null) and overwrites d_uv [B,H,W,2] and d_uv_da [B,H,W,4] (deterministic; each may be null; d_uv_da is only written with
 *      MCS_TEX_LINEAR_MIPMAP_LINEAR; at least one gradient).  One launch per call, no host sync, no allocation. */
enum { MCS_TEX_LINEAR = 0, MCS_TEX_LINEAR_MIPMAP_LINEAR = 1 };
enum { MCS_TEX_WRAP = 0, MCS_TEX_CLAMP = 1 };
typedef struct mcs_texture_levels {
    int32_t n_levels;          /* 1..16 */
    int32_t C;                 /* channels, >= 1 */
    const float *ptr[16];
    int32_t h[16];
    int32_t w[16];
    int64_t batch_stride[16];  /* elements */
} mcs_texture_levels;
int mcs_texture_fwd(const mcs_texture_levels *tex, const float *uv, const float *uv_da, int32_t B, int32_t H, int32_t W, int32_t filter_mode,
                    int32_t boundary_mode, float *out, mcs_stream stream);
int mcs_texture_bwd(const mcs_texture_levels *tex, const float *uv, const float *uv_da, int32_t B, int32_t H, int32_t W, int32_t filter_mode,
                    int32_t boundary_mode, const float *d_out, float *const *d_tex, float *d_uv, float *d_uv_da, mcs_stream stream);

/* ---- DMTet geometry: marching_tets and sdf_reg_loss (geometry/dmtet.py:91-153); semantics in csrc/dmtet.cu.  All arrays are device
 *      memory.  Static tables of one tet grid (V vertices, T tets, E unique edges), built once by the caller:
 *        edges [E,2] int32, 8-byte aligned: the unique vertex pairs of the tets' six base edges, each as (min, max), sorted
 *          lexicographically;
 *        tets [T,4] int32, 16-byte aligned; tet_edges [T,6] int32: the row of `edges` of the tet's base edges (0,1) (0,2) (0,3) (1,2)
 *          (1,3) (2,3);
 *        v2e_offsets [V+1] / v2e_edges int32: for vertex v, v2e_edges[v2e_offsets[v] .. v2e_offsets[v+1]) lists the rows of `edges` with
 *          v as an end, in ascending order (a row whose two ends are v is listed twice).
 *      sdf [V] and pos [V,3] are fp32 with the given element strides.
 *      mcs_dmtet_count writes vid [E] (the output vertex of each edge, -1 where it does not cross), tet_prefix [T,2] (exclusive prefixes
 *      of the 1- and 2-triangle tets, 8-byte aligned) and counts [3] = (vertices M, 1-triangle tets n1, 2-triangle tets n2); workspace:
 *      mcs_dmtet_workspace_bytes(E, T) bytes, 8-byte aligned, contents ignored on entry.  mcs_dmtet_emit then writes verts [M,3] fp32,
 *      faces [n1 + 2 n2, 3] int64 and uv_idx [n1 + 2 n2, 3] int64; the caller sizes them from counts read back after the count phase.
 *      mcs_dmtet_bwd overwrites d_pos [V,3] and d_sdf [V] (contiguous) from d_verts [M,3] (contiguous) by a per-vertex gather, no atomics.
 *      mcs_sdf_reg_fwd: loss (one float) = the reference's sdf_reg_loss over the edge list edges [E,2] (any vertex pairs), m (one float) =
 *      the number of masked edges; partials: mcs_sdf_reg_num_partials(E) x 3 doubles of scratch.  mcs_sdf_reg_bwd overwrites d_sdf [V] from
 *      the upstream gradient d_loss (one float on the device), with v2e_* the CSR of that edge list.  No entry synchronises the host. */
#define MCS_DMTET_TILE 2048
int64_t mcs_dmtet_workspace_bytes(int32_t E, int32_t T);
int mcs_dmtet_count(const float *sdf, int64_t sdf_stride, const int32_t *edges, int32_t E, const int32_t *tets, int32_t T, int32_t *vid,
                    int32_t *tet_prefix, int32_t *counts, void *workspace, mcs_stream stream);
int mcs_dmtet_emit(const float *pos, int64_t pos_stride0, int64_t pos_stride1, const float *sdf, int64_t sdf_stride, const int32_t *edges, int32_t E,
                   const int32_t *tets, const int32_t *tet_edges, int32_t T, const int32_t *vid, const int32_t *tet_prefix, const int32_t *counts,
                   float *verts, int64_t *faces, int64_t *uv_idx, mcs_stream stream);
int mcs_dmtet_bwd(const float *pos, int64_t pos_stride0, int64_t pos_stride1, const float *sdf, int64_t sdf_stride, int32_t V, const int32_t *edges,
                  int32_t E, const int32_t *vid, const int32_t *v2e_offsets, const int32_t *v2e_edges, const float *d_verts, float *d_pos, float *d_sdf,
                  mcs_stream stream);
int32_t mcs_sdf_reg_num_partials(int32_t E);
int mcs_sdf_reg_fwd(const float *sdf, int64_t sdf_stride, const int32_t *edges, int32_t E, double *partials, float *loss, float *m, mcs_stream stream);
int mcs_sdf_reg_bwd(const float *sdf, int64_t sdf_stride, int32_t V, const int32_t *edges, const int32_t *v2e_offsets, const int32_t *v2e_edges,
                    const float *m, const float *d_loss, float *d_sdf, mcs_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* MCSHADE_H */
