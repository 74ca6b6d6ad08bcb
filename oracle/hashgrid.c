/* hashgrid.c -- CPU oracle of the multiresolution hash-grid encoding (TEST INFRASTRUCTURE, not product code).
 *
 * A plain-C restatement of the contract in nvdiffrecmc_b200/csrc/hashgrid.cu, written independently of the kernels:
 *   level table (double precision), forward, d x (levels ascending, corners ascending) and d params (a sequential scatter in point,
 *   level, corner order).
 * Two builds of this file (oracle/hashgrid.py): fp32 (`real` = float, compared bit for bit with the CUDA forward and d x) and fp64
 * (-DORACLE_F64, checked by finite differences and the adjoint identity).  Compile with -ffp-contract=off: every product and sum is one
 * IEEE round-to-nearest operation, the fma of p_d is the only fused one.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#ifdef ORACLE_F64
typedef double real;
#define R_FMA fma
#define R_FLOOR floor
#else
typedef float real;
#define R_FMA fmaf
#define R_FLOOR floorf
#endif

int hg_sizeof_real(void) { return (int)sizeof(real); }

/* Level table: returns 0, or 1 for an unsupported argument.  offset has n_levels + 1 entries. */
int hg_levels(int n_levels, int log2_hashmap_size, double base_resolution, double per_level_scale, uint64_t *offset, uint32_t *res,
              float *scale, uint32_t *dense_mask)
{
    if (n_levels < 1 || n_levels > 16 || log2_hashmap_size < 0 || log2_hashmap_size > 31) return 1;
    const uint64_t cap = (uint64_t)1 << log2_hashmap_size;
    offset[0] = 0;
    *dense_mask = 0;
    for (int l = 0; l < n_levels; ++l) {
        const float s = (float)(base_resolution * pow(per_level_scale, (double)l) - 1.0);
        const uint64_t r = (uint64_t)(int64_t)ceil((double)s) + 1;
        const uint64_t r3 = r * r * r;
        uint64_t size;
        if (r3 >= ((uint64_t)1 << 31)) {
            size = cap;
        } else {
            const uint64_t padded = (r3 + 7) / 8 * 8;
            size = padded < cap ? padded : cap;
        }
        if (r3 <= size) *dense_mask |= 1u << l;
        offset[l + 1] = offset[l] + size;
        res[l] = (uint32_t)r;
        scale[l] = s;
    }
    return 0;
}

/* cvt.rmi.s32.f32 of an already floored value: saturating, NaN -> 0 */
static int32_t cvt_rmi_s32(real g)
{
    if (g != g) return 0;
    if (g >= (real)2147483648.0) return INT32_MAX;
    if (g <= (real)-2147483648.0) return INT32_MIN;
    return (int32_t)g;
}

typedef struct {
    uint32_t g[3];
    real t[3];
} cell_t;

static cell_t cell(real s, const real *x)
{
    cell_t c;
    for (int d = 0; d < 3; ++d) {
        const real p = R_FMA(s, x[d], (real)0.5);
        const real f = R_FLOOR(p);
        c.g[d] = (uint32_t)cvt_rmi_s32(f);
        c.t[d] = p - f;
    }
    return c;
}

static uint32_t corner_index(const cell_t *cl, int c, int dense, uint32_t res, uint32_t size)
{
    const uint32_t cx = cl->g[0] + (uint32_t)(c & 1), cy = cl->g[1] + (uint32_t)((c >> 1) & 1), cz = cl->g[2] + (uint32_t)((c >> 2) & 1);
    uint32_t h;
    if (dense) {
        const uint32_t res2 = res * res;
        h = cx + cy * res + cz * res2;
    } else {
        h = cx ^ (cy * 2654435761u) ^ (cz * 805459861u);
    }
    return h % size;
}

static void corner_weights(const cell_t *cl, int c, real w1[3])
{
    for (int d = 0; d < 3; ++d) w1[d] = ((c >> d) & 1) ? cl->t[d] : (real)1 - cl->t[d];
}

/* x [n,3]; params [2 * offset[L]]; out [n, 2L] */
void hg_fwd(const real *x, int64_t n, const real *params, int L, const uint64_t *offset, const uint32_t *res, const float *scale,
            uint32_t dense_mask, real *out)
{
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        for (int l = 0; l < L; ++l) {
            const uint32_t size = (uint32_t)(offset[l + 1] - offset[l]);
            const cell_t cl = cell((real)scale[l], x + 3 * i);
            real y0 = 0, y1 = 0;
            for (int c = 0; c < 8; ++c) {
                real w1[3];
                corner_weights(&cl, c, w1);
                const real w = (w1[0] * w1[1]) * w1[2];
                const real *v = params + 2 * (offset[l] + corner_index(&cl, c, (dense_mask >> l) & 1u, res[l], size));
                y0 = y0 + w * v[0];
                y1 = y1 + w * v[1];
            }
            out[i * 2 * L + 2 * l] = y0;
            out[i * 2 * L + 2 * l + 1] = y1;
        }
    }
}

/* d_out [n, 2L]; d_params (may be null) accumulates; d_x (may be null) is overwritten. */
void hg_bwd(const real *x, int64_t n, const real *params, int L, const uint64_t *offset, const uint32_t *res, const float *scale,
            uint32_t dense_mask, const real *d_out, real *d_params, real *d_x)
{
    if (d_x) {
#pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < n; ++i) {
            real dx[3] = {0, 0, 0};
            for (int l = 0; l < L; ++l) {
                const real g0 = d_out[i * 2 * L + 2 * l], g1 = d_out[i * 2 * L + 2 * l + 1];
                if (g0 == 0 && g1 == 0) continue;
                const uint32_t size = (uint32_t)(offset[l + 1] - offset[l]);
                const cell_t cl = cell((real)scale[l], x + 3 * i);
                real a[3] = {0, 0, 0};
                for (int c = 0; c < 8; ++c) {
                    real w1[3];
                    corner_weights(&cl, c, w1);
                    const real *v = params + 2 * (offset[l] + corner_index(&cl, c, (dense_mask >> l) & 1u, res[l], size));
                    const real s = g0 * v[0] + g1 * v[1];
                    const real other[3] = {w1[1] * w1[2], w1[0] * w1[2], w1[0] * w1[1]};
                    for (int d = 0; d < 3; ++d) a[d] = a[d] + (((c >> d) & 1) ? other[d] : -other[d]) * s;
                }
                for (int d = 0; d < 3; ++d) dx[d] = dx[d] + (real)scale[l] * a[d];
            }
            for (int d = 0; d < 3; ++d) d_x[3 * i + d] = dx[d];
        }
    }
    if (d_params) {
        for (int64_t i = 0; i < n; ++i) {
            for (int l = 0; l < L; ++l) {
                const real g0 = d_out[i * 2 * L + 2 * l], g1 = d_out[i * 2 * L + 2 * l + 1];
                if (g0 == 0 && g1 == 0) continue;
                const uint32_t size = (uint32_t)(offset[l + 1] - offset[l]);
                const cell_t cl = cell((real)scale[l], x + 3 * i);
                for (int c = 0; c < 8; ++c) {
                    real w1[3];
                    corner_weights(&cl, c, w1);
                    const real w = (w1[0] * w1[1]) * w1[2];
                    real *dp = d_params + 2 * (offset[l] + corner_index(&cl, c, (dense_mask >> l) & 1u, res[l], size));
                    dp[0] = dp[0] + w * g0;
                    dp[1] = dp[1] + w * g1;
                }
            }
        }
    }
}
