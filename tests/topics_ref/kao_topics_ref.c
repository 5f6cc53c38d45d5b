/*
 * TEST INFRASTRUCTURE — plain-C restatement of the per-topic balance rows (docs/MODEL.md §10) on top of the
 * restatement of the search (oracle/kao_ref.c, included unchanged: every call without topic rows stays the oracle's
 * own).  Full evaluation = kao_ref_eval + the topic rows; candidate keys and search are kao_ref_candidate_keys /
 * kao_ref_search with that evaluation.  Never part of the product.
 */
#include "../../oracle/kao_ref.c"

typedef struct {
    int32_t T;
    const int32_t *topic_of;            /* [P] */
    const int32_t *rep_lo, *rep_hi;     /* [T] C3t */
    const int32_t *ldr_lo, *ldr_hi;     /* [T] C4t */
} ref_topics;

static int64_t band(int64_t c, int64_t lo, int64_t hi) { return (c > hi ? c - hi : 0) + (c < lo ? lo - c : 0); }

/* violation of the topic rows: for every topic and BROKER slot (padding slots carry no row), the replicas and the
 * valid leaders (a leader slot the row holds) of the topic's partitions there against [lo, hi] */
int64_t kao_tref_topic_violation(const ref_problem *pb, const ref_topics *tp, const uint32_t *bits, const uint8_t *leader)
{
    ref_layout L;
    if (kao_ref_layout(pb, &L)) return -1;
    const int NSL = L.W * 32;
    int32_t *cnt = (int32_t *)calloc((size_t)tp->T * NSL, 4), *lcnt = (int32_t *)calloc((size_t)tp->T * NSL, 4);
    for (int p = 0; p < pb->P; ++p) {
        const uint32_t *row = bits + (size_t)p * L.W;
        const int t = tp->topic_of[p], ld = leader[p];
        for (int s = 0; s < NSL; ++s)
            if (row_has(row, s)) ++cnt[(size_t)t * NSL + s];
        if (ld < NSL && row_has(row, ld)) ++lcnt[(size_t)t * NSL + ld];
    }
    int64_t v = 0;
    for (int t = 0; t < tp->T; ++t)
        for (int s = 0; s < NSL; ++s) {
            if (s >= KAO_MAX_SLOTS || L.broker_of_slot[s] < 0) continue;
            v += band(cnt[(size_t)t * NSL + s], tp->rep_lo[t], tp->rep_hi[t]);
            v += band(lcnt[(size_t)t * NSL + s], tp->ldr_lo[t], tp->ldr_hi[t]);
        }
    free(cnt);
    free(lcnt);
    return v;
}

void kao_tref_eval(const ref_problem *pb, const ref_topics *tp, const uint32_t *bits, const uint8_t *leader,
                   int64_t *viol_out, int64_t *obj_out)
{
    kao_ref_eval(pb, bits, leader, viol_out, obj_out);
    if (*viol_out >= 0) *viol_out += kao_tref_topic_violation(pb, tp, bits, leader);
}

void kao_tref_candidate_keys(const ref_problem *pb, const ref_topics *tp, const uint32_t *bits, const uint8_t *leader,
                             uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_begin, uint32_t count,
                             uint64_t *keys, int nthreads)
{
    ref_layout L; kao_ref_layout(pb, &L);
    const size_t nb = (size_t)pb->P * L.W;
    ref_aux ax;
    const int obj_bits = kao_ref_obj_bits(pb);
    aux_alloc(pb, L.W, &ax);
    analyse(pb, &L, bits, leader, &ax);
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#else
    (void)nthreads;
#endif
#pragma omp parallel
    {
        uint32_t *sb = (uint32_t *)malloc(nb * 4);
        uint8_t *sl = (uint8_t *)malloc((size_t)pb->P);
#pragma omp for schedule(static)
        for (int64_t i = 0; i < (int64_t)count; ++i) {
            ref_patchset ps; int64_t v, o;
            uint32_t idx = idx_begin + (uint32_t)i;
            gen_patches(pb, &L, &ax, bits, leader, seed, round, idx, round_size, &ps);
            memcpy(sb, bits, nb * 4); memcpy(sl, leader, (size_t)pb->P);
            apply_patches(L.W, &ps, sb, sl);
            kao_tref_eval(pb, tp, sb, sl, &v, &o);
            keys[i] = kao_ref_pack(v, o, idx, obj_bits);
        }
        free(sb); free(sl);
    }
    aux_free(&ax);
}

uint64_t kao_tref_search(const ref_problem *pb, const ref_topics *tp, uint32_t *bits, uint8_t *leader, uint64_t seed,
                         uint32_t first_round, uint32_t rounds, uint32_t round_size, uint64_t *round_keys, int nthreads)
{
    uint64_t last = KEY_NONE;
    uint64_t *keys = (uint64_t *)malloc((size_t)round_size * 8);
    for (uint32_t i = 0; i < rounds; ++i) {                 /* round first_round + i mod 2^32 (docs/MODEL.md §6) */
        const uint32_t t = first_round + i;
        uint64_t best = KEY_NONE;
        kao_tref_candidate_keys(pb, tp, bits, leader, seed, t, round_size, 0, round_size, keys, nthreads);
        for (uint32_t j = 0; j < round_size; ++j) if (keys[j] < best) best = keys[j];
        kao_ref_gen(pb, bits, leader, seed, t, (uint32_t)(best & ((1u << IDX_BITS) - 1)), round_size, bits, leader);
        if (round_keys) round_keys[i] = best;
        last = best;
    }
    free(keys);
    return last;
}
