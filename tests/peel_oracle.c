/* peel_oracle.c -- CPU twin of depth peeling's ray query, test infrastructure (wrapped by tests/peel_oracle.py).
 *
 * It includes the oracle's source so that the triangle predicate is mt_eval() itself, with the same fixed operation order and the
 * same build flags (-ffp-contract=off): a peeled layer is compared with the GPU bit for bit, like orc_closest_hit.  Only fp32. */
#include "mcoracle.c"

/* Brute-force closest hit with t > sep(t_after[i]), sep(t) = fl32(t * (1 + 2^-16)) (nvdiffrecmc_b200/csrc/bvh_traverse.cuh peel_sep);
 * ties in t go to the lowest triangle id.  t_after[i] = +inf gives a miss.  Outputs as orc_closest_hit: tri_id -1 and t = 1e16 on a miss. */
void orc_closest_hit_after(const OrcScene *s, int n, const real *ro, const real *rd, const real *t_after, int32_t *tri_id, real *tuv)
{
#pragma omp parallel for schedule(dynamic, 64)
    for (int i = 0; i < n; ++i) {
        v3 o = ld3(ro + 3 * (size_t)i), d = ld3(rd + 3 * (size_t)i);
        const real lo = t_after[i] * RC(1.0000152587890625);
        real best = RC(1e16f); int bid = -1; real bu = 0, bv = 0;
        for (int t = 0; t < s->T && lo != (real)INFINITY; ++t) {
            const real *tr = s->tri + 9 * (size_t)t;
            real tt, u, v;
            if (mt_eval(o, d, ld3(tr), ld3(tr + 3), ld3(tr + 6), &tt, &u, &v) && tt > lo && tt < best) { best = tt; bid = t; bu = u; bv = v; }
        }
        tri_id[i] = bid; tuv[3 * (size_t)i] = best; tuv[3 * (size_t)i + 1] = bu; tuv[3 * (size_t)i + 2] = bv;
    }
}

/* Every hit of one ray: t_all[t] = the hit's t for triangle t, or -1 when mt_eval rejects it.  Returns the number of hits. */
int orc_all_hits(const OrcScene *s, const real *ro, const real *rd, real *t_all)
{
    v3 o = ld3(ro), d = ld3(rd);
    int cnt = 0;
    for (int t = 0; t < s->T; ++t) {
        const real *tr = s->tri + 9 * (size_t)t;
        real tt, u, v;
        t_all[t] = RC(-1);
        if (mt_eval(o, d, ld3(tr), ld3(tr + 3), ld3(tr + 6), &tt, &u, &v)) { t_all[t] = tt; ++cnt; }
    }
    return cnt;
}
