/*
 * TEST INFRASTRUCTURE — plain-C restatement of the per-partition replication rows (docs/MODEL.md §11) on top of the
 * restatement of the search (oracle/kao_ref.c) and of the topic rows (tests/topics_ref), both included unchanged.
 * Full evaluation = kao_ref_eval with row p's C1 / C7 terms taken against rf[p] / ppr_lo[p]..ppr_hi[p] instead of
 * RF / ppr_lo..ppr_hi, plus the topic rows when given; candidate keys and search are kao_ref_candidate_keys /
 * kao_ref_search with that evaluation; the initial base keeps / completes row p to rf[p].  Never part of the product.
 */
#include "../topics_ref/kao_topics_ref.c"

typedef struct {
    const int32_t *rf, *ppr_lo, *ppr_hi;    /* [P] */
} ref_replication;

/* C1 + C7 terms of one row against (n, lo, hi) */
static int64_t rf_terms(const ref_problem *pb, const ref_layout *L, const uint32_t *row, int n, int lo, int hi)
{
    int pr[KAO_MAX_R] = {0}, cnt = 0;
    for (int s = 0; s < L->W * 32; ++s)
        if (row_has(row, s)) { ++cnt; if (s / L->S < pb->R) ++pr[s / L->S]; }
    int64_t v = abs(cnt - n);
    for (int r = 0; r < pb->R; ++r) v += (pr[r] > hi ? pr[r] - hi : 0) + (pr[r] < lo ? lo - pr[r] : 0);
    return v;
}

void kao_rref_eval(const ref_problem *pb, const ref_topics *tp, const ref_replication *rp, const uint32_t *bits,
                   const uint8_t *leader, int64_t *viol_out, int64_t *obj_out)
{
    if (tp) kao_tref_eval(pb, tp, bits, leader, viol_out, obj_out);
    else kao_ref_eval(pb, bits, leader, viol_out, obj_out);
    if (*viol_out < 0) return;
    ref_layout L; kao_ref_layout(pb, &L);
    for (int p = 0; p < pb->P; ++p) {
        const uint32_t *row = bits + (size_t)p * L.W;
        *viol_out += rf_terms(pb, &L, row, rp->rf[p], rp->ppr_lo[p], rp->ppr_hi[p]) -
                     rf_terms(pb, &L, row, pb->RF, pb->ppr_lo, pb->ppr_hi);
    }
}

void kao_rref_candidate_keys(const ref_problem *pb, const ref_topics *tp, const ref_replication *rp,
                             const uint32_t *bits, const uint8_t *leader, uint64_t seed, uint32_t round,
                             uint32_t round_size, uint32_t idx_begin, uint32_t count, uint64_t *keys, int nthreads)
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
            kao_rref_eval(pb, tp, rp, sb, sl, &v, &o);
            keys[i] = kao_ref_pack(v, o, idx, obj_bits);
        }
        free(sb); free(sl);
    }
    aux_free(&ax);
}

uint64_t kao_rref_search(const ref_problem *pb, const ref_topics *tp, const ref_replication *rp, uint32_t *bits,
                         uint8_t *leader, uint64_t seed, uint32_t first_round, uint32_t rounds, uint32_t round_size,
                         uint64_t *round_keys, int nthreads)
{
    uint64_t last = KEY_NONE;
    uint64_t *keys = (uint64_t *)malloc((size_t)round_size * 8);
    for (uint32_t i = 0; i < rounds; ++i) {                 /* round first_round + i mod 2^32 (docs/MODEL.md §6) */
        const uint32_t t = first_round + i;
        uint64_t best = KEY_NONE;
        kao_rref_candidate_keys(pb, tp, rp, bits, leader, seed, t, round_size, 0, round_size, keys, nthreads);
        for (uint32_t j = 0; j < round_size; ++j) if (keys[j] < best) best = keys[j];
        kao_ref_gen(pb, bits, leader, seed, t, (uint32_t)(best & ((1u << IDX_BITS) - 1)), round_size, bits, leader);
        if (round_keys) round_keys[i] = best;
        last = best;
    }
    free(keys);
    return last;
}

/* kao_ref_init_base with row p kept / completed to rf[p] */
void kao_rref_init_base(const ref_problem *pb, const ref_replication *rp, uint32_t *bits, uint8_t *leader)
{
    ref_layout L; kao_ref_layout(pb, &L);
    const int P = pb->P, B = pb->B, W = L.W;
    int32_t load[KAO_MAX_SLOTS] = {0};
    memset(bits, 0, (size_t)P * W * 4);
    for (int p = 0; p < P; ++p) {
        uint32_t *row = bits + (size_t)p * W;
        int n = 0, ld = -1;
        for (int i = 0; i < pb->RFcur && n < rp->rf[p]; ++i) {
            int b = pb->cur[(size_t)p * pb->RFcur + i];
            if (b < 0 || b >= B || row_has(row, L.slot_of_broker[b])) continue;
            row_set(row, L.slot_of_broker[b]); ++n; ++load[b];
            if (ld < 0) ld = L.slot_of_broker[b];
        }
        leader[p] = (uint8_t)(ld < 0 ? 0xFF : ld);
    }
    for (int p = 0; p < P; ++p) {
        uint32_t *row = bits + (size_t)p * W;
        int n = row_count(row, W);
        while (n < rp->rf[p] && n < B) {
            int pr[KAO_MAX_R] = {0};
            for (int b = 0; b < B; ++b) if (row_has(row, L.slot_of_broker[b])) ++pr[pb->rack_of[b]];
            int best = -1;
            for (int b = 0; b < B; ++b) {
                if (row_has(row, L.slot_of_broker[b])) continue;
                if (best < 0) { best = b; continue; }
                int ra = pr[pb->rack_of[b]], rb = pr[pb->rack_of[best]];
                if (ra < rb || (ra == rb && load[b] < load[best])) best = b;
            }
            /* a row without survivors is led from its first added replica (not "leader byte 0xFF": that is slot
             * 255 when every slot holds a broker) */
            if (n == 0) leader[p] = (uint8_t)L.slot_of_broker[best];
            row_set(row, L.slot_of_broker[best]); ++load[best]; ++n;
        }
    }
}
