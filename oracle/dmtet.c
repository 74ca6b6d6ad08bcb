/* dmtet.c -- CPU oracle of DMTet's marching tetrahedra and SDF regulariser (TEST INFRASTRUCTURE, not product code).
 *
 * A plain-C restatement of the contract in nvdiffrecmc_b200/csrc/dmtet.cu, written independently of the kernels: the static tables by a
 * sort of (edge key, slot) pairs and a counting sort, the extraction by sequential loops (vertices in edge order; the 1-triangle tets,
 * then the 2-triangle tets, in tet order) instead of scans, and the backward passes as sequential scatters in ascending edge order, which
 * add into each vertex in the order the kernels' per-vertex gathers do.
 * Two builds of this file (oracle/dmtet.py): fp32 (`real` = float, compared bit for bit with the CUDA vertices, faces, uv_idx, d pos and
 * d sdf) and fp64 (-DORACLE_F64, checked by finite differences).  Compile with -ffp-contract=off: every product, quotient and sum is one
 * IEEE round-to-nearest operation; the UV lattice's fmaf is the only fused one, as torch.linspace rounds once there.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#ifdef ORACLE_F64
typedef double real;
#else
typedef float real;
#endif

int dmt_sizeof_real(void) { return (int)sizeof(real); }

static const int BASE[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
static const int TRI[16][6] = {
    {-1, -1, -1, -1, -1, -1}, {1, 0, 2, -1, -1, -1}, {4, 0, 3, -1, -1, -1}, {1, 4, 2, 1, 3, 4},
    {3, 1, 5, -1, -1, -1},    {2, 3, 0, 2, 5, 3},    {1, 4, 0, 1, 5, 4},    {4, 2, 5, -1, -1, -1},
    {4, 5, 2, -1, -1, -1},    {4, 1, 0, 4, 5, 1},    {3, 2, 0, 3, 5, 2},    {1, 3, 5, -1, -1, -1},
    {4, 1, 2, 4, 3, 1},       {3, 0, 4, -1, -1, -1}, {2, 0, 1, -1, -1, -1}, {-1, -1, -1, -1, -1, -1}};
static const int NTRI[16] = {0, 1, 1, 2, 1, 2, 2, 1, 1, 2, 2, 1, 2, 1, 1, 0};

typedef struct { int64_t key, slot; } KeySlot;

static int cmp_key_slot(const void *pa, const void *pb)
{
    const KeySlot *a = (const KeySlot *)pa, *b = (const KeySlot *)pb;
    if (a->key != b->key) return a->key < b->key ? -1 : 1;
    return a->slot < b->slot ? -1 : (a->slot > b->slot);
}

/* The grid's unique edges (min, max), lexicographically sorted, into edges [<= 6T, 2]; each tet's six edge rows into tet_edges [T,6].
 * Returns E. */
int64_t dmt_edges(int64_t V, int64_t T, const int64_t *tet, int32_t *edges, int32_t *tet_edges)
{
    KeySlot *ks = (KeySlot *)malloc(sizeof(KeySlot) * (size_t)(6 * T));
    for (int64_t t = 0; t < T; ++t)
        for (int k = 0; k < 6; ++k) {
            int64_t a = tet[4 * t + BASE[k][0]], b = tet[4 * t + BASE[k][1]];
            if (a > b) { const int64_t s = a; a = b; b = s; }
            ks[6 * t + k].key = a * V + b;
            ks[6 * t + k].slot = 6 * t + k;
        }
    qsort(ks, (size_t)(6 * T), sizeof(KeySlot), cmp_key_slot);
    int64_t E = 0;
    for (int64_t i = 0; i < 6 * T; ++i) {
        if (i == 0 || ks[i].key != ks[i - 1].key) {
            edges[2 * E] = (int32_t)(ks[i].key / V);
            edges[2 * E + 1] = (int32_t)(ks[i].key % V);
            ++E;
        }
        tet_edges[ks[i].slot] = (int32_t)(E - 1);
    }
    free(ks);
    return E;
}

/* Vertex -> edge CSR: off [V+1], adj [2E], each vertex's edge rows ascending (counting sort over the rows in order). */
void dmt_adjacency(int64_t V, int64_t E, const int32_t *edges, int32_t *off, int32_t *adj)
{
    for (int64_t v = 0; v <= V; ++v) off[v] = 0;
    for (int64_t i = 0; i < 2 * E; ++i) off[edges[i] + 1] += 1;
    for (int64_t v = 0; v < V; ++v) off[v + 1] += off[v];
    int32_t *fill = (int32_t *)malloc(sizeof(int32_t) * (size_t)(V + 1));
    for (int64_t v = 0; v <= V; ++v) fill[v] = off[v];
    for (int64_t i = 0; i < 2 * E; ++i) adj[fill[edges[i]]++] = (int32_t)(i / 2);
    free(fill);
}

/* Side N of the UV lattice of T tets: ceil(sqrt((2T + 1) / 2)) as the reference computes it (integer division, then double). */
int64_t dmt_uv_side(int64_t T) { return (int64_t)ceil(sqrt((double)((2 * T + 1) / 2))); }

/* uvs [4 N^2, 2] (always fp32, as the reference): lattice coordinate i = torch.linspace(0, 1 - 1/N, N)[i] (one rounding per element: the
 * first half step * i, the second half end - step * (N - 1 - i)), cell (row y, column x), corners (x, y) (x+p, y) (x+p, y+p) (x, y+p)
 * with p = fl32(0.9 / N). */
void dmt_uvs(int64_t T, float *uvs)
{
    const int64_t N = dmt_uv_side(T);
    const float end = (float)(1.0 - 1.0 / (double)N);
    const float step = N > 1 ? end / (float)(N - 1) : 0.0f;
    const float pad = (float)(0.9 / (double)N);
    float *lin = (float *)malloc(sizeof(float) * (size_t)N);
    for (int64_t i = 0; i < N; ++i) lin[i] = i < N / 2 ? step * (float)i : fmaf(-step, (float)(N - 1 - i), end);
    for (int64_t y = 0; y < N; ++y)
        for (int64_t x = 0; x < N; ++x) {
            float *q = uvs + 8 * (y * N + x);
            const float u = lin[x], v = lin[y];
            q[0] = u; q[1] = v; q[2] = u + pad; q[3] = v; q[4] = u + pad; q[5] = v + pad; q[6] = u; q[7] = v + pad;
        }
    free(lin);
}

/* The extraction.  counts [2] = (M vertices, F faces); vid [E] (-1 where the edge does not cross); verts [<= E, 3]; faces and uv_idx
 * [<= 2T, 3]. */
void dmt_extract(int64_t V, int64_t E, int64_t T, const real *pos, const real *sdf, const int32_t *edges, const int64_t *tet,
                 const int32_t *tet_edges, int64_t *counts, int32_t *vid, real *verts, int64_t *faces, int64_t *uv_idx)
{
    (void)V;
    int64_t M = 0;
    for (int64_t e = 0; e < E; ++e) {
        const int32_t a = edges[2 * e], b = edges[2 * e + 1];
        const real sa = sdf[a], sb = sdf[b];
        if ((sa > 0) == (sb > 0)) { vid[e] = -1; continue; }
        const real D = sa + (-sb);
        const real w0 = (-sb) / D, w1 = sa / D;
        for (int c = 0; c < 3; ++c) verts[3 * M + c] = pos[3 * a + c] * w0 + pos[3 * b + c] * w1;
        vid[e] = (int32_t)M++;
    }
    int64_t F = 0;
    for (int pass = 1; pass <= 2; ++pass)
        for (int64_t t = 0; t < T; ++t) {
            int code = 0;
            for (int k = 0; k < 4; ++k) code |= (sdf[tet[4 * t + k]] > 0) << k;
            if (NTRI[code] != pass) continue;
            for (int k = 0; k < pass; ++k, ++F) {
                for (int j = 0; j < 3; ++j) faces[3 * F + j] = vid[tet_edges[6 * t + TRI[code][3 * k + j]]];
                uv_idx[3 * F] = 4 * t; uv_idx[3 * F + 1] = 4 * t + k + 1; uv_idx[3 * F + 2] = 4 * t + k + 2;
            }
        }
    counts[0] = M;
    counts[1] = F;
}

/* d pos [V,3] and d sdf [V] (overwritten) from d_verts [M,3]; see csrc/dmtet.cu for the order of operations. */
void dmt_backward(int64_t V, int64_t E, const real *pos, const real *sdf, const int32_t *edges, const int32_t *vid, const real *d_verts,
                  real *d_pos, real *d_sdf)
{
    for (int64_t i = 0; i < 3 * V; ++i) d_pos[i] = 0;
    for (int64_t i = 0; i < V; ++i) d_sdf[i] = 0;
    for (int64_t e = 0; e < E; ++e) {
        if (vid[e] < 0) continue;
        const int32_t a = edges[2 * e], b = edges[2 * e + 1];
        const real sa = sdf[a], sb = sdf[b];
        const real D = sa + (-sb);
        const real w0 = (-sb) / D, w1 = sa / D;
        const real *g = d_verts + 3 * (int64_t)vid[e];
        const real *pa = pos + 3 * (int64_t)a, *pb = pos + 3 * (int64_t)b;
        const real dw0 = (g[0] * pa[0] + g[1] * pa[1]) + g[2] * pa[2];
        const real dw1 = (g[0] * pb[0] + g[1] * pb[1]) + g[2] * pb[2];
        const real dD = (-dw0) * (w0 / D) + (-dw1) * (w1 / D);
        for (int c = 0; c < 3; ++c) d_pos[3 * a + c] = d_pos[3 * a + c] + g[c] * w0;
        d_sdf[a] = d_sdf[a] + (dw1 / D + dD);
        for (int c = 0; c < 3; ++c) d_pos[3 * b + c] = d_pos[3 * b + c] + g[c] * w1;
        d_sdf[b] = d_sdf[b] + -(dw0 / D + dD);
    }
}

/* torch.sign's values: 1, -1, and 0 for +-0 and NaN */
static int sgn(real x) { return (int)(0 < x) - (int)(x < 0); }

/* sdf_reg_loss: the two BCE-with-logits means over the edges whose ends differ in sign, summed in double; *m = their count.  NaN when
 * *m = 0. */
double dmt_reg_fwd(int64_t E, const real *sdf, const int32_t *edges, int64_t *m)
{
    double s0 = 0.0, s1 = 0.0;
    int64_t n = 0;
    for (int64_t e = 0; e < E; ++e) {
        const real a = sdf[edges[2 * e]], b = sdf[edges[2 * e + 1]];
        if (sgn(a) == sgn(b)) continue;
        const double x0 = a, x1 = b, y0 = b > 0 ? 1.0 : 0.0, y1 = a > 0 ? 1.0 : 0.0;
        s0 += log1p(exp(-fabs(x0))) + fmax(x0, 0.0) - x0 * y0;
        s1 += log1p(exp(-fabs(x1))) + fmax(x1, 0.0) - x1 * y1;
        ++n;
    }
    *m = n;
    return s0 / (double)n + s1 / (double)n;
}

/* d sdf [V] (overwritten): each masked edge adds ((sigmoid(x) - y) * d_loss) / M to the end whose value is the logit x. */
void dmt_reg_bwd(int64_t V, int64_t E, const real *sdf, const int32_t *edges, real d_loss, real *d_sdf)
{
    int64_t n = 0;
    for (int64_t e = 0; e < E; ++e) n += sgn(sdf[edges[2 * e]]) != sgn(sdf[edges[2 * e + 1]]);
    for (int64_t v = 0; v < V; ++v) d_sdf[v] = 0;
    const real M = (real)n;
    for (int64_t e = 0; e < E; ++e) {
        const int32_t ia = edges[2 * e], ib = edges[2 * e + 1];
        const real a = sdf[ia], b = sdf[ib];
        if (sgn(a) == sgn(b)) continue;
        const real one = 1;
        const real ga = ((one / (one + (real)exp(-(double)a)) - (b > 0 ? one : 0)) * d_loss) / M;
        const real gb = ((one / (one + (real)exp(-(double)b)) - (a > 0 ? one : 0)) * d_loss) / M;
        d_sdf[ia] = d_sdf[ia] + ga;
        d_sdf[ib] = d_sdf[ib] + gb;
    }
}
