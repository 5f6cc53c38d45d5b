/*
 * TEST INFRASTRUCTURE — plain-C restatement of the candidate-search hot path.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * build, load or call this file.  The product (kafka_assignment_optimizer_b200/csrc) never links
 * it and has no CPU fallback.
 *
 * PARITY STATUS: parity unpinned against lp_solve (see oracle/model.py header: the reference
 * snapshot holds no code; lp_solve 5.5, /root/reference/README.md:135-136, is not available).
 * This file restates, with scalar loops and no bit tricks, the SAME deterministic search the CUDA
 * engine runs (docs/MODEL.md): counter-based candidate stream (Philox4x32-10 keyed by seed,
 * counter = (index, round)), full evaluation of C1..C7 + objective per candidate
 * (README.md:144-185), packed (violation, cost, index) argmin per round, winner becomes the next
 * base.  Same seed => bit-identical winner, per-candidate keys and trajectory.  The model
 * semantics are validated against oracle/model.py (HiGHS), which is pinned on the README
 * known-answer vector (README.md:83-91).
 *
 * Build: oracle/Makefile (gcc -O2 -fopenmp -shared).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define KAO_MAX_SLOTS 256
#define KAO_MAX_R 32
#define KAO_MAX_W 8
#define KAO_MAX_OPS 3
#define KAO_HOME 4

typedef struct {
    int32_t P, B, R, RF, RFcur;
    const uint8_t *rack_of;          /* [B] */
    const uint16_t *wF, *wL;         /* [P*B] README.md:145-146 */
    const int32_t *rep_lo, *rep_hi;  /* [B] C3 README.md:158-161 */
    const int32_t *ldr_lo, *ldr_hi;  /* [B] C4 README.md:163-166 */
    const int32_t *rack_lo, *rack_hi;/* [R] C6 README.md:173-176 */
    int32_t ppr_lo, ppr_hi;          /*     C7 README.md:178-180 */
    const int32_t *cur;              /* [P*RFcur] dense broker index, -1 = absent */
} ref_problem;

#define KEY_BITS 63             /* keys stay below 2^63: they order the same as signed int64 */
#define IDX_BITS 24
#define KEY_NONE 0x7FFFFFFFFFFFFFFFull

/* ---------------------------------------------------------------- slot space (docs/MODEL.md §2) */
/* Brokers are re-indexed rack-major into aligned slots: slot = rack*S + rank-in-rack, S = the
 * smallest power of two >= max(8, largest rack).  `order` = position in rack-major order. */
typedef struct {
    int S, NS, W;
    int slot_of_broker[KAO_MAX_SLOTS];
    int broker_of_slot[KAO_MAX_SLOTS]; /* -1 = padding slot */
    int slot_of_order[KAO_MAX_SLOTS];
    int order_of_slot[KAO_MAX_SLOTS];
} ref_layout;

int kao_ref_layout(const ref_problem *pb, ref_layout *L)
{
    int size[KAO_MAX_R] = {0}, maxsz = 0;
    if (pb->R < 1 || pb->R > KAO_MAX_R || pb->B < 1 || pb->B > KAO_MAX_SLOTS) return -1;
    for (int b = 0; b < pb->B; ++b) { if (pb->rack_of[b] >= pb->R) return -1; ++size[pb->rack_of[b]]; }
    for (int r = 0; r < pb->R; ++r) if (size[r] > maxsz) maxsz = size[r];
    int S = 8; while (S < maxsz) S <<= 1;
    L->S = S; L->NS = pb->R * S;
    if (L->NS > KAO_MAX_SLOTS) return -1;
    int w = (L->NS + 31) / 32, W = 1; while (W < w) W <<= 1;
    L->W = W;
    for (int s = 0; s < KAO_MAX_SLOTS; ++s) { L->broker_of_slot[s] = -1; L->order_of_slot[s] = -1; }
    int rank[KAO_MAX_R] = {0};
    for (int b = 0; b < pb->B; ++b) {
        int r = pb->rack_of[b], s = r * S + rank[r]++;
        L->slot_of_broker[b] = s; L->broker_of_slot[s] = b;
    }
    int o = 0;
    for (int s = 0; s < L->NS; ++s)
        if (L->broker_of_slot[s] >= 0) { L->slot_of_order[o] = s; L->order_of_slot[s] = o; ++o; }
    return 0;
}
int kao_ref_words(const ref_problem *pb) { ref_layout L; return kao_ref_layout(pb, &L) ? -1 : L.W; }

/* ---------------------------------------------------------------- Philox4x32-10 (Random123) */
void kao_ref_philox(const uint32_t ctr_in[4], const uint32_t key_in[2], uint32_t out[4])
{
    uint32_t c0 = ctr_in[0], c1 = ctr_in[1], c2 = ctr_in[2], c3 = ctr_in[3];
    uint32_t k0 = key_in[0], k1 = key_in[1];
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        uint32_t n1 = (uint32_t)p1;
        uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

/* ---------------------------------------------------------------- bit helpers (scalar) */
static int row_has(const uint32_t *row, int s) { return (row[s >> 5] >> (s & 31)) & 1u; }
static void row_set(uint32_t *row, int s) { row[s >> 5] |= 1u << (s & 31); }
static void row_clr(uint32_t *row, int s) { row[s >> 5] &= ~(1u << (s & 31)); }
static int row_count(const uint32_t *row, int W)
{
    int n = 0;
    for (int j = 0; j < W; ++j) n += __builtin_popcount(row[j]);
    return n;
}
/* k-th (0-based) set bit in ascending slot order, -1 if fewer */
static int row_kth(const uint32_t *row, int W, int k)
{
    for (int s = 0; s < W * 32; ++s)
        if (row_has(row, s)) { if (k == 0) return s; --k; }
    return -1;
}

/* ---------------------------------------------------------------- full evaluation (docs/MODEL.md §3) */
/* Candidate = bits[P][W] over slots + leader slot per partition.  violation = sum over every row
 * of C1..C7 of the amount by which it is missed; objective = README.md:145-146.  A leader that is
 * not one of the partition's replicas violates C2 by 1 and earns no leader weight.  Replicas on
 * padding slots count for C1/C7/C6 and violate C3 (their bound is [0,0]). */
void kao_ref_eval(const ref_problem *pb, const uint32_t *bits, const uint8_t *leader,
                  int64_t *viol_out, int64_t *obj_out)
{
    ref_layout L;
    if (kao_ref_layout(pb, &L)) { *viol_out = -1; *obj_out = -1; return; }
    const int P = pb->P, R = pb->R, W = L.W, S = L.S;
    int64_t viol = 0, obj = 0;
    int32_t cnt[KAO_MAX_SLOTS] = {0}, lcnt[KAO_MAX_SLOTS] = {0}, rc[KAO_MAX_R] = {0};
    for (int p = 0; p < P; ++p) {
        const uint32_t *row = bits + (size_t)p * W;
        int pr[KAO_MAX_R] = {0};
        int n = 0, ld = leader[p];
        int ld_ok = (ld < W * 32) && row_has(row, ld);
        for (int j = 0; j < W; ++j) {
            for (uint32_t w = row[j]; w; w &= w - 1) {              /* every replica of p */
                int s = j * 32 + __builtin_ctz(w);
                ++n; ++cnt[s];
                if (s / S < R) { ++pr[s / S]; ++rc[s / S]; }
                int b = L.broker_of_slot[s];
                if (b >= 0 && !(ld_ok && s == ld)) obj += pb->wF[(size_t)p * pb->B + b];
            }
        }
        viol += abs(n - pb->RF);                                   /* C1 */
        if (ld_ok) {
            ++lcnt[ld];
            if (L.broker_of_slot[ld] >= 0) obj += pb->wL[(size_t)p * pb->B + L.broker_of_slot[ld]];
        } else viol += 1;                                          /* C2 (+C5) */
        for (int r = 0; r < R; ++r) {                              /* C7 */
            if (pr[r] > pb->ppr_hi) viol += pr[r] - pb->ppr_hi;
            if (pr[r] < pb->ppr_lo) viol += pb->ppr_lo - pr[r];
        }
    }
    for (int s = 0; s < W * 32; ++s) {
        int b = (s < KAO_MAX_SLOTS) ? L.broker_of_slot[s] : -1;
        int rlo = b >= 0 ? pb->rep_lo[b] : 0, rhi = b >= 0 ? pb->rep_hi[b] : 0;
        int llo = b >= 0 ? pb->ldr_lo[b] : 0, lhi = b >= 0 ? pb->ldr_hi[b] : 0;
        if (cnt[s] > rhi) viol += cnt[s] - rhi;                    /* C3 */
        if (cnt[s] < rlo) viol += rlo - cnt[s];
        if (lcnt[s] > lhi) viol += lcnt[s] - lhi;                  /* C4 */
        if (lcnt[s] < llo) viol += llo - lcnt[s];
    }
    for (int r = 0; r < R; ++r) {                                  /* C6 */
        if (rc[r] > pb->rack_hi[r]) viol += rc[r] - pb->rack_hi[r];
        if (rc[r] < pb->rack_lo[r]) viol += pb->rack_lo[r] - rc[r];
    }
    *viol_out = viol; *obj_out = obj;
}

/* Packed key (docs/MODEL.md 3): violation | (objmax - objective) | index, smaller is better.  The
 * cost field is obj_bits wide = the bit length of the largest objective the model can reach
 * (P * RF * largest weight); the violation field takes the remaining 63 - 24 - obj_bits bits
 * (at most 31) and saturates. */
int kao_ref_obj_bits(const ref_problem *pb)
{
    uint64_t maxw = 0, top;
    int bits = 1;
    for (size_t i = 0; i < (size_t)pb->P * pb->B; ++i) {
        if (pb->wF[i] > maxw) maxw = pb->wF[i];
        if (pb->wL[i] > maxw) maxw = pb->wL[i];
    }
    top = (uint64_t)pb->P * pb->RF * maxw;
    while (top >> bits) ++bits;
    return bits;
}
uint64_t kao_ref_pack(int64_t viol, int64_t obj, uint32_t idx, int obj_bits)
{
    const int vbits = KEY_BITS - IDX_BITS - obj_bits;
    const uint64_t vcap = vbits >= 31 ? 0x7FFFFFFFull : ((1ull << vbits) - 1);
    const uint64_t omax = (1ull << obj_bits) - 1;
    uint64_t v = viol < 0 ? 0 : ((uint64_t)viol > vcap ? vcap : (uint64_t)viol);
    uint64_t c = (obj < 0 || (uint64_t)obj > omax) ? 0 : omax - (uint64_t)obj;
    return (v << (IDX_BITS + obj_bits)) | (c << IDX_BITS) | (idx & ((1u << IDX_BITS) - 1));
}

/* ---------------------------------------------------------------- replica lists <-> bit-plane */
/* replicas[P*RF]: dense broker indices, leader first, -1 padded (README.md:52-63 order) */
void kao_ref_encode(const ref_problem *pb, const int32_t *replicas, uint32_t *bits, uint8_t *leader)
{
    ref_layout L; kao_ref_layout(pb, &L);
    memset(bits, 0, (size_t)pb->P * L.W * 4);
    for (int p = 0; p < pb->P; ++p) {
        int have = 0;
        leader[p] = 0xFF;
        for (int i = 0; i < pb->RF; ++i) {
            int b = replicas[(size_t)p * pb->RF + i];
            if (b < 0 || b >= pb->B) continue;
            row_set(bits + (size_t)p * L.W, L.slot_of_broker[b]);
            if (!have) { leader[p] = (uint8_t)L.slot_of_broker[b]; have = 1; }
        }
    }
}
/* leader first, then followers in ascending dense broker index (README.md:65-78,:88) */
void kao_ref_decode(const ref_problem *pb, const uint32_t *bits, const uint8_t *leader,
                    int32_t *replicas)
{
    ref_layout L; kao_ref_layout(pb, &L);
    for (int p = 0; p < pb->P; ++p) {
        const uint32_t *row = bits + (size_t)p * L.W;
        int32_t *out = replicas + (size_t)p * pb->RF;
        int n = 0, ld = leader[p], ldb = -1;
        for (int i = 0; i < pb->RF; ++i) out[i] = -1;
        if (ld < L.W * 32 && row_has(row, ld) && L.broker_of_slot[ld] >= 0)
            out[n++] = ldb = L.broker_of_slot[ld];
        for (int b = 0; b < pb->B && n < pb->RF; ++b)
            if (b != ldb && row_has(row, L.slot_of_broker[b])) out[n++] = b;
    }
}

/* ---------------------------------------------------------------- initial base (docs/MODEL.md §4) */
/* cur restricted to the target brokers, order kept (leader = first survivor); surplus replicas
 * (RF lowered) dropped from the tail; missing replicas (broker removed / RF raised) added one at
 * a time, partitions in ascending order, on the broker minimising (replicas of p already in that
 * rack, current load, dense broker index). */
void kao_ref_init_base(const ref_problem *pb, uint32_t *bits, uint8_t *leader)
{
    ref_layout L; kao_ref_layout(pb, &L);
    const int P = pb->P, B = pb->B, W = L.W;
    int32_t load[KAO_MAX_SLOTS] = {0};
    memset(bits, 0, (size_t)P * W * 4);
    for (int p = 0; p < P; ++p) {
        uint32_t *row = bits + (size_t)p * W;
        int n = 0, ld = -1;
        for (int i = 0; i < pb->RFcur && n < pb->RF; ++i) {
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
        while (n < pb->RF && n < B) {
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

/* ---------------------------------------------------------------- base analysis (docs/MODEL.md §5.1) */
/* home[p] = slots of the surviving entries among the first KAO_HOME positions of cur[p]; home0[p] = slot of cur[p][0]
 * if that broker survives, else -1.  D = ascending list of the partitions whose row lacks at
 * least one home slot ("displaced"); DL = ascending list of the partitions that hold a replica on
 * home0 but are led from elsewhere ("leader displaced"). */
typedef struct { int nD, nL; int32_t *D, *DL; uint32_t *home; /* [P*W] home masks */ int32_t *home0; /* [P] */ } ref_aux;

static void home_mask(const ref_problem *pb, const ref_layout *L, int p, uint32_t *m)
{
    memset(m, 0, (size_t)L->W * 4);
    for (int i = 0; i < pb->RFcur && i < KAO_HOME; ++i) {
        int b = pb->cur[(size_t)p * pb->RFcur + i];
        if (b >= 0 && b < pb->B) row_set(m, L->slot_of_broker[b]);
    }
}
static void analyse(const ref_problem *pb, const ref_layout *L, const uint32_t *bits,
                    const uint8_t *leader, ref_aux *ax)
{
    ax->nD = ax->nL = 0;
    for (int p = 0; p < pb->P; ++p) {
        uint32_t *m = ax->home + (size_t)p * L->W;
        home_mask(pb, L, p, m);
        int miss = 0;
        for (int j = 0; j < L->W; ++j) if (m[j] & ~bits[(size_t)p * L->W + j]) miss = 1;
        if (miss) ax->D[ax->nD++] = p;
        int b0 = pb->cur[(size_t)p * pb->RFcur];
        int h0 = (b0 >= 0 && b0 < pb->B) ? L->slot_of_broker[b0] : -1;
        ax->home0[p] = h0;
        if (h0 >= 0 && row_has(bits + (size_t)p * L->W, h0) && leader[p] != h0) ax->DL[ax->nL++] = p;
    }
}
static void aux_alloc(const ref_problem *pb, int W, ref_aux *ax)
{
    ax->D = (int32_t *)malloc((size_t)pb->P * 4);
    ax->DL = (int32_t *)malloc((size_t)pb->P * 4);
    ax->home0 = (int32_t *)malloc((size_t)pb->P * 4);
    ax->home = (uint32_t *)malloc((size_t)pb->P * W * 4);
}
static void aux_free(ref_aux *ax) { free(ax->D); free(ax->DL); free(ax->home0); free(ax->home); }

/* ---------------------------------------------------------------- candidate generator (docs/MODEL.md §5) */
static uint32_t mulhi32(uint32_t a, uint32_t n) { return (uint32_t)(((uint64_t)a * n) >> 32); }

typedef struct { int32_t p; uint32_t row[KAO_MAX_W]; uint8_t leader; } ref_patch;
typedef struct { int n; ref_patch e[KAO_MAX_OPS]; } ref_patchset;

static void view_row(int W, const uint32_t *bits, const uint8_t *leader,
                     const ref_patchset *ps, int p, uint32_t *row, int *ld)
{
    memcpy(row, bits + (size_t)p * W, (size_t)W * 4);
    *ld = leader[p];
    for (int i = 0; i < ps->n; ++i)
        if (ps->e[i].p == p) { memcpy(row, ps->e[i].row, (size_t)W * 4); *ld = ps->e[i].leader; }
}
static int touched(const ref_patchset *ps, int p)
{
    for (int i = 0; i < ps->n; ++i) if (ps->e[i].p == p) return 1;
    return 0;
}
static void push_patch(int W, ref_patchset *ps, int p, const uint32_t *row, int ld)
{
    for (int i = 0; i < ps->n; ++i)
        if (ps->e[i].p == p) { memcpy(ps->e[i].row, row, (size_t)W * 4); ps->e[i].leader = (uint8_t)ld; return; }
    ref_patch *e = &ps->e[ps->n++];
    e->p = p; memset(e->row, 0, sizeof e->row); memcpy(e->row, row, (size_t)W * 4); e->leader = (uint8_t)ld;
}

/* REPLACE: in partition p the replica on slot a moves to the first broker, in rack-major order
 * starting at order index o (cyclic), that p does not already use; a leader replica keeps its
 * leadership on the new broker. */
static int op_replace(const ref_problem *pb, const ref_layout *L, const uint32_t *bits,
                      const uint8_t *leader, ref_patchset *ps, int p, int a, int o, int *s_out)
{
    uint32_t row[KAO_MAX_W]; int ld;
    view_row(L->W, bits, leader, ps, p, row, &ld);
    if (a < 0 || !row_has(row, a)) return 0;
    int tries = 0;
    while (row_has(row, L->slot_of_order[o])) { o = (o + 1 == pb->B) ? 0 : o + 1; if (++tries > pb->B) return 0; }
    int s = L->slot_of_order[o];
    row_clr(row, a); row_set(row, s);
    if (ld == a) ld = s;
    push_patch(L->W, ps, p, row, ld);
    *s_out = s;
    return 1;
}
/* LEADER: partition p is led from slot `want` if that is one of its non-leader replicas, else
 * from its k-th (ascending slot) non-leader replica.  Returns the new leader slot or -1. */
static int op_leader(const ref_layout *L, const uint32_t *bits, const uint8_t *leader,
                     ref_patchset *ps, int p, int want, uint32_t rnd)
{
    uint32_t row[KAO_MAX_W]; int ld;
    view_row(L->W, bits, leader, ps, p, row, &ld);
    int n = row_count(row, L->W);
    int has_ld = (ld < L->W * 32) && row_has(row, ld);
    int m = n - (has_ld ? 1 : 0);
    if (m < 1) return -1;
    if (want >= 0 && want < L->W * 32 && want != ld && row_has(row, want)) { push_patch(L->W, ps, p, row, want); return want; }
    int k = (int)mulhi32(rnd, (uint32_t)m);
    for (int s = 0; s < L->W * 32; ++s) {
        if (!row_has(row, s) || s == ld) continue;
        if (k-- == 0) { push_patch(L->W, ps, p, row, s); return s; }
    }
    return -1;
}
/* first partition q >= p0 (cyclic), not yet patched, with a non-leader replica on slot src */
static int find_follower(const ref_problem *pb, int W, const uint32_t *bits, const uint8_t *leader,
                         const ref_patchset *ps, int p0, int src)
{
    if (src < 0 || src >= W * 32) return -1;
    for (int k = 0; k < pb->P; ++k) {
        int q = p0 + k; if (q >= pb->P) q -= pb->P;
        if (touched(ps, q)) continue;
        if (leader[q] != src && row_has(bits + (size_t)q * W, src)) return q;
    }
    return -1;
}
/* first partition q >= p0 (cyclic), not yet patched, whose leader is slot src */
static int find_led_by(const ref_problem *pb, const uint8_t *leader, const ref_patchset *ps,
                       int p0, int src)
{
    for (int k = 0; k < pb->P; ++k) {
        int q = p0 + k; if (q >= pb->P) q -= pb->P;
        if (touched(ps, q)) continue;
        if (leader[q] == src) return q;
    }
    return -1;
}
/* first partition q >= p0 (cyclic), not yet patched, that has a replica on slot src */
static int find_holder(const ref_problem *pb, int W, const uint32_t *bits, const ref_patchset *ps,
                       int p0, int src)
{
    if (src < 0 || src >= W * 32) return -1;
    for (int k = 0; k < pb->P; ++k) {
        int q = p0 + k; if (q >= pb->P) q -= pb->P;
        if (touched(ps, q)) continue;
        if (row_has(bits + (size_t)q * W, src)) return q;
    }
    return -1;
}

/* Row patches that turn the base into candidate (round, idx).  idx == round_size-1 is the
 * identity.  Pure function of (base, seed, round, idx).  docs/MODEL.md §5:
 *   control word c = r0:  bits 0-1 -> number of ops (0:1, 1-2:2, 3:3); bit 2 first op is LEADER;
 *   bit 3 guided first op; per later op k: 2 bits link type (0 R-push, 1 R-pull, 2 L-push,
 *   3 L-pull) and 1 bit "close".
 * The chain keeps (lo, hi) = (slot that lost, slot that gained) a replica / a leadership:
 *   R-push  a holder of hi moves that replica to lo (close) or to a random broker   -> hi = target
 *   R-pull  a random partition moves a replica (its leader replica if close) to lo  -> lo = source
 *   L-push  a partition led by hi is led by lo (close, if lo follows there) / its first broker /
 *           a random follower                                                        -> hi = new leader
 *   L-pull  a partition where lo follows is led by lo                                -> lo = old leader
 * Guided first op: REPLACE restores a displaced partition (list D) to a missing home broker;
 * LEADER hands a leader-displaced partition (list DL) back to its first broker. */
static void gen_patches(const ref_problem *pb, const ref_layout *L, const ref_aux *ax,
                        const uint32_t *bits, const uint8_t *leader,
                        uint64_t seed, uint32_t round, uint32_t idx, uint32_t round_size,
                        ref_patchset *ps)
{
    const int P = pb->P, B = pb->B, W = L->W;
    ps->n = 0;
    if (idx + 1 == round_size) return;
    uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
    uint32_t c0[4] = {idx, round, 0, 0x4B414F21u}, c1[4] = {idx, round, 1, 0x4B414F21u};
    uint32_t r[4], s[4];
    kao_ref_philox(c0, key, r);
    kao_ref_philox(c1, key, s);
    /* every fourth round (round mod 4 = 3) is a cycle round: three ops, guided REPLACE first, R-pull, R-push with close */
    const int cycle = (round & 3u) == 3u;
    const uint32_t ctl = cycle ? ((r[0] & ~(0x4u | 0x20u | 0x80u | 0x100u)) | 0x21Bu) : r[0];
    const int nops = (ctl & 3u) == 0 ? 1 : ((ctl & 3u) == 3 ? 3 : 2);
    int moved_leader = 0;                                  /* the last REPLACE moved a leader replica */
    const int first_leader = (ctl >> 2) & 1u, gbit = (ctl >> 3) & 1u;
    uint32_t row[KAO_MAX_W]; int ld;
    int lo, hi;
    if (first_leader) {
        const int guided = gbit && ax->nL > 0;
        const int p = guided ? ax->DL[mulhi32(r[1], (uint32_t)ax->nL)] : (int)mulhi32(r[1], (uint32_t)P);
        lo = leader[p];
        hi = op_leader(L, bits, leader, ps, p, guided ? ax->home0[p] : -1, r[2]);
        if (hi < 0) return;
    } else {
        const int guided = gbit && ax->nD > 0;
        const int p = guided ? ax->D[mulhi32(r[1], (uint32_t)ax->nD)] : (int)mulhi32(r[1], (uint32_t)P);
        view_row(W, bits, leader, ps, p, row, &ld);
        const int n = row_count(row, W);
        if (n == 0) return;
        int a = row_kth(row, W, (int)mulhi32(r[2], (uint32_t)n));
        int o = (int)mulhi32(r[3], (uint32_t)B);
        if (guided) {
            uint32_t miss[KAO_MAX_W], nonhome[KAO_MAX_W];
            const uint32_t *hm = ax->home + (size_t)p * W;
            for (int j = 0; j < W; ++j) { miss[j] = hm[j] & ~row[j]; nonhome[j] = row[j] & ~hm[j]; }
            int nm = row_count(miss, W), nn = row_count(nonhome, W);
            if (nm > 0) {
                o = L->order_of_slot[row_kth(miss, W, (int)mulhi32(r[3], (uint32_t)nm))];
                if (nn > 0) a = row_kth(nonhome, W, (int)mulhi32(r[2], (uint32_t)nn));
            }
        }
        moved_leader = (ld == a);
        if (!op_replace(pb, L, bits, leader, ps, p, a, o, &hi)) return;
        lo = a;
    }
    for (int k = 1; k < nops; ++k) {
        const uint32_t link = (ctl >> (4 + 3 * (k - 1))) & 3u;
        const int close = (ctl >> (6 + 3 * (k - 1))) & 1u;
        const uint32_t ra = s[2 * (k - 1)], rb = s[2 * (k - 1) + 1];
        const int start = (int)mulhi32(ra, (uint32_t)P);
        int olo = (lo < KAO_MAX_SLOTS) ? L->order_of_slot[lo] : -1;
        if (olo < 0) olo = 0;
        /* cycle rounds, bits 11 / 13: the op moves a replica of the same role (leader / follower) as the one before */
        const int match = cycle && ((ctl >> (11 + 2 * (k - 1))) & 1u);
        if (link == 0) {                                   /* R-push */
            int q, t;
            if (!match) q = find_holder(pb, W, bits, ps, start, hi);
            else q = moved_leader ? find_led_by(pb, leader, ps, start, hi) : find_follower(pb, W, bits, leader, ps, start, hi);
            if (q < 0) return;
            if (hi < 0 || hi >= W * 32 || !row_has(bits + (size_t)q * W, hi)) return;
            moved_leader = (leader[q] == hi);
            if (!op_replace(pb, L, bits, leader, ps, q, hi, close ? olo : (int)mulhi32(rb, (uint32_t)B), &t)) return;
            hi = t;
        } else if (link == 1) {                            /* R-pull */
            int q = start, lq, t;
            if (touched(ps, q)) return;
            uint32_t rq[KAO_MAX_W];
            view_row(W, bits, leader, ps, q, rq, &lq);
            const int nq = row_count(rq, W);
            if (nq == 0) return;
            int src = row_kth(rq, W, (int)mulhi32(rb, (uint32_t)nq));
            const int led = lq < W * 32 && row_has(rq, lq);
            if (close && led) src = lq;
            if (match && led) {
                if (moved_leader) src = lq;
                else if (nq > 1) {
                    uint32_t fol[KAO_MAX_W];
                    memcpy(fol, rq, (size_t)W * 4);
                    row_clr(fol, lq);
                    src = row_kth(fol, W, (int)mulhi32(rb, (uint32_t)(nq - 1)));
                }
            }
            moved_leader = (src == lq);
            if (!op_replace(pb, L, bits, leader, ps, q, src, olo, &t)) return;
            lo = src;
        } else if (link == 2) {                            /* L-push */
            int q = find_led_by(pb, leader, ps, start, hi);
            if (q < 0) return;
            int t = op_leader(L, bits, leader, ps, q, close ? lo : ax->home0[q], rb);
            if (t < 0) return;
            hi = t;
        } else {                                           /* L-pull */
            int q = find_follower(pb, W, bits, leader, ps, start, lo);
            if (q < 0) return;
            const int old = leader[q];
            if (op_leader(L, bits, leader, ps, q, lo, rb) < 0) return;
            lo = old;
        }
    }
}

static void apply_patches(int W, const ref_patchset *ps, uint32_t *bits, uint8_t *leader)
{
    for (int i = 0; i < ps->n; ++i) {
        memcpy(bits + (size_t)ps->e[i].p * W, ps->e[i].row, (size_t)W * 4);
        leader[ps->e[i].p] = ps->e[i].leader;
    }
}

/* materialise candidate (round, idx) of base (bits, leader) into (out_bits, out_leader) */
void kao_ref_gen(const ref_problem *pb, const uint32_t *bits, const uint8_t *leader,
                 uint64_t seed, uint32_t round, uint32_t idx, uint32_t round_size,
                 uint32_t *out_bits, uint8_t *out_leader)
{
    ref_layout L; kao_ref_layout(pb, &L);
    ref_aux ax; ref_patchset ps;
    aux_alloc(pb, L.W, &ax);
    analyse(pb, &L, bits, leader, &ax);
    gen_patches(pb, &L, &ax, bits, leader, seed, round, idx, round_size, &ps);
    if (out_bits != bits) memcpy(out_bits, bits, (size_t)pb->P * L.W * 4);
    if (out_leader != leader) memcpy(out_leader, leader, (size_t)pb->P);
    apply_patches(L.W, &ps, out_bits, out_leader);
    aux_free(&ax);
}

/* keys of candidates idx_begin..idx_begin+count-1 of one round, each materialised and evaluated
 * in full (the per-candidate parity vector, T3) */
void kao_ref_candidate_keys(const ref_problem *pb, const uint32_t *bits, const uint8_t *leader,
                            uint64_t seed, uint32_t round, uint32_t round_size,
                            uint32_t idx_begin, uint32_t count, uint64_t *keys, int nthreads)
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
            kao_ref_eval(pb, sb, sl, &v, &o);
            keys[i] = kao_ref_pack(v, o, idx, obj_bits);
        }
        free(sb); free(sl);
    }
    aux_free(&ax);
}

/* ---------------------------------------------------------------- search (docs/MODEL.md §6) */
/* rounds x round_size candidates; per round the minimum key wins and becomes the next base.
 * bits/leader: in = base, out = final base.  round_keys (optional) receives each round's key. */
uint64_t kao_ref_search(const ref_problem *pb, uint32_t *bits, uint8_t *leader, uint64_t seed,
                        uint32_t first_round, uint32_t rounds, uint32_t round_size,
                        uint64_t *round_keys, int nthreads)
{
    ref_layout L; kao_ref_layout(pb, &L);
    const size_t nb = (size_t)pb->P * L.W;
    uint64_t last = KEY_NONE;
    uint64_t *keys = (uint64_t *)malloc((size_t)round_size * 8);
    /* round numbers are u32: call i runs round first_round + i mod 2^32 (docs/MODEL.md §6) */
    for (uint32_t i = 0; i < rounds; ++i) {
        const uint32_t t = first_round + i;
        uint64_t best = KEY_NONE;
        kao_ref_candidate_keys(pb, bits, leader, seed, t, round_size, 0, round_size, keys, nthreads);
        for (uint32_t j = 0; j < round_size; ++j) if (keys[j] < best) best = keys[j];
        uint32_t widx = (uint32_t)(best & ((1u << IDX_BITS) - 1));
        kao_ref_gen(pb, bits, leader, seed, t, widx, round_size, bits, leader);
        if (round_keys) round_keys[i] = best;
        last = best;
    }
    free(keys);
    (void)nb;
    return last;
}

int kao_ref_max_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
