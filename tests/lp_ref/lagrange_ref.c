/* lagrange_ref.c — plain-C restatement of the Lagrangian LP bound (docs/MODEL.md §9): the bit-exact reference
 * that the CUDA kernel (csrc/kao_lagrange.cu) is compared with.  Sequential and written for clarity; it shares
 * no code with the engine.
 *
 * Multipliers: u[0..B) C3 (replicas per broker), u[B..2B) C4 (leaders per broker), u[2B..2B+R) C6 (replicas per
 * rack), int64 with LR_F fractional bits, clamped to [-LR_U, LR_U].  Every quantity below is an exact integer. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define LR_F 20
#define LR_U ((int64_t)1 << 34)
#define LR_NEG INT64_MIN
#define LR_MAXRF 8

typedef struct {
    int P, B, R, RF, ppr_lo, ppr_hi;
    const uint8_t *rack_of;
    const uint16_t *wF, *wL;
    int *rstart;     /* [R+1] racks' ranges in `order` */
    int *order;      /* [B] brokers grouped by rack, ascending index inside a rack */
    int64_t *a3, *a4;/* [B] what a follower / a leader on broker b pays: u3 + u6, u3 + u4 + u6 */
    char *intop;     /* [B] scratch */
} Inst;

/* best_p of partition p under the current a3/a4 (docs/MODEL.md §9), counts of its argmax added to c3/c4/c6;
 * returns LR_NEG when the partition has no row satisfying C1, C2, C5 and C7 */
static int64_t best_row(const Inst *in, int p, int64_t *c3, int64_t *c4, int64_t *c6)
{
    const int RF = in->RF, R = in->R;
    int64_t dp[LR_MAXRF + 1][2], nd[LR_MAXRF + 1][2];
    unsigned char ch[32][LR_MAXRF + 1][2];
    int topj[32][LR_MAXRF], gpos[32][LR_MAXRF + 1], restj[32], Kr[32];
    for (int n = 0; n <= RF; ++n) dp[n][0] = dp[n][1] = LR_NEG;
    dp[0][0] = 0;
#define FW(b) (((int64_t)in->wF[(size_t)p * in->B + (b)] << LR_F) - in->a3[b])
#define LW(b) (((int64_t)in->wL[(size_t)p * in->B + (b)] << LR_F) - in->a4[b])
    for (int r = 0; r < R; ++r) {
        const int j0 = in->rstart[r], j1 = in->rstart[r + 1], size = j1 - j0;
        int K = size < RF ? size : RF;
        if (in->ppr_hi < K) K = in->ppr_hi;
        Kr[r] = K;
        /* the K best followers: descending reduced follower weight, ties by ascending broker index */
        int64_t tv[LR_MAXRF];
        int len = 0;
        for (int j = j0; j < j1; ++j) {
            const int b = in->order[j];
            const int64_t v = FW(b);
            int pos = len;
            while (pos > 0 && tv[pos - 1] < v) --pos;
            if (pos >= K) continue;
            for (int i = (len < K ? len : K - 1); i > pos; --i) { tv[i] = tv[i - 1]; topj[r][i] = topj[r][i - 1]; }
            tv[pos] = v; topj[r][pos] = b;
            if (len < K) ++len;
        }
        int64_t S[LR_MAXRF + 1], G[LR_MAXRF + 1];
        S[0] = 0;
        for (int i = 0; i < K; ++i) S[i + 1] = S[i] + tv[i];
        /* the best leader among the rack's other brokers: largest reduced leader weight, first by broker index */
        for (int i = 0; i < K; ++i) in->intop[topj[r][i]] = 1;
        restj[r] = -1;
        int64_t restv = 0;
        for (int j = j0; j < j1; ++j) {
            const int b = in->order[j];
            if (in->intop[b]) continue;
            const int64_t v = LW(b);
            if (restj[r] < 0 || v > restv) { restj[r] = b; restv = v; }
        }
        for (int i = 0; i < K; ++i) in->intop[topj[r][i]] = 0;
        /* G[k]: a leader and k - 1 followers in this rack; candidates in follower rank order, then the rest */
        for (int k = 1; k <= K; ++k) {
            int64_t best = 0;
            int bp = -1;
            for (int i = 0; i < K; ++i) {
                const int64_t v = (i < k ? S[k] - tv[i] : S[k - 1]) + LW(topj[r][i]);
                if (bp < 0 || v > best) { best = v; bp = i; }
            }
            if (restj[r] >= 0 && S[k - 1] + restv > best) { best = S[k - 1] + restv; bp = K; }
            G[k] = best; gpos[r][k] = bp;
        }
        /* one DP step: k replicas of the partition in rack r, ppr_lo <= k <= K */
        for (int n = 0; n <= RF; ++n) nd[n][0] = nd[n][1] = LR_NEG;
        for (int n = 0; n <= RF; ++n)
            for (int l = 0; l < 2; ++l) {
                if (dp[n][l] == LR_NEG) continue;
                for (int k = in->ppr_lo; k <= K && n + k <= RF; ++k) {
                    const int64_t v = dp[n][l] + S[k];
                    if (v > nd[n + k][l]) { nd[n + k][l] = v; ch[r][n + k][l] = (unsigned char)k; }
                    if (l == 0 && k >= 1) {
                        const int64_t w = dp[n][0] + G[k];
                        if (w > nd[n + k][1]) { nd[n + k][1] = w; ch[r][n + k][1] = (unsigned char)(k | 16); }
                    }
                }
            }
        memcpy(dp, nd, sizeof(dp));
    }
#undef FW
#undef LW
    const int64_t best = dp[RF][1];
    if (best == LR_NEG) return LR_NEG;
    int n = RF, l = 1;
    for (int r = R - 1; r >= 0; --r) {
        const int c = ch[r][n][l], k = c & 15, lead = c >> 4;
        c6[r] += k;
        if (!lead) {
            for (int i = 0; i < k; ++i) c3[topj[r][i]] += 1;
        } else {
            /* the leader (a position of the top list, or K = the best other broker) and the first k - 1 of the
             * top list without it */
            const int gp = gpos[r][k], leader = gp < Kr[r] ? topj[r][gp] : restj[r];
            c3[leader] += 1; c4[leader] += 1;
            for (int i = 0, nf = 0; i < k && nf < k - 1; ++i)
                if (i != gp) { c3[topj[r][i]] += 1; ++nf; }
        }
        n -= k; l -= lead;
    }
    return best;
}

/* The integer iteration of docs/MODEL.md §9.  T: objective of a feasible assignment.  Returns 0, or -1 when a
 * partition has no admissible row (then no assignment is feasible). */
int lagrange_ref(int P, int B, int R, int RF, const uint8_t *rack_of, const uint16_t *wF, const uint16_t *wL,
                 const int32_t *rep_lo, const int32_t *rep_hi, const int32_t *ldr_lo, const int32_t *ldr_hi,
                 const int32_t *rack_lo, const int32_t *rack_hi, int ppr_lo, int ppr_hi, int64_t T,
                 uint32_t max_iterations, int64_t *bound, uint32_t *iterations_run, int64_t *multipliers)
{
    const int NR = 2 * B + R;
    Inst in = {P, B, R, RF, ppr_lo, ppr_hi, rack_of, wF, wL, NULL, NULL, NULL, NULL, NULL};
    in.rstart = calloc(R + 1, sizeof(int));
    in.order = calloc(B, sizeof(int));
    in.a3 = calloc(B, sizeof(int64_t));
    in.a4 = calloc(B, sizeof(int64_t));
    in.intop = calloc(B, 1);
    int64_t *u = calloc(NR, sizeof(int64_t)), *ub = calloc(NR, sizeof(int64_t)), *lo = calloc(NR, sizeof(int64_t)),
            *hi = calloc(NR, sizeof(int64_t)), *cnt = calloc(NR, sizeof(int64_t)), *g = calloc(NR, sizeof(int64_t));
    for (int b = 0; b < B; ++b) ++in.rstart[rack_of[b] + 1];
    for (int r = 0; r < R; ++r) in.rstart[r + 1] += in.rstart[r];
    {
        int *fill = calloc((size_t)NR, sizeof(int));
        for (int b = 0; b < B; ++b) in.order[in.rstart[rack_of[b]] + fill[rack_of[b]]++] = b;
        free(fill);
    }
    /* rows and their bounds; an upper bound above what any assignment reaches is lowered to that (same rows) */
    const int64_t tot = (int64_t)P * RF;
    for (int b = 0; b < B; ++b) {
        lo[b] = rep_lo[b]; hi[b] = rep_hi[b] < tot ? rep_hi[b] : tot;
        lo[B + b] = ldr_lo[b]; hi[B + b] = ldr_hi[b] < P ? ldr_hi[b] : P;
    }
    for (int r = 0; r < R; ++r) { lo[2 * B + r] = rack_lo[r]; hi[2 * B + r] = rack_hi[r] < tot ? rack_hi[r] : tot; }
    int rc = 0;
    int64_t best = INT64_MAX;
    uint32_t it = 0;
    for (;;) {
        ++it;
        for (int b = 0; b < B; ++b) { in.a3[b] = u[b] + u[2 * B + rack_of[b]]; in.a4[b] = in.a3[b] + u[B + b]; }
        memset(cnt, 0, NR * sizeof(int64_t));
        int64_t L = 0;
        for (int p = 0; p < P; ++p) {
            const int64_t v = best_row(&in, p, cnt, cnt + B, cnt + 2 * B);
            if (v == LR_NEG) { rc = -1; goto out; }
            L += v;
        }
        int64_t n2 = 0;
        for (int i = 0; i < NR; ++i) {
            L += u[i] > 0 ? u[i] * hi[i] : u[i] * lo[i];
            const int64_t c = cnt[i], cl = c < lo[i] ? lo[i] : c > hi[i] ? hi[i] : c;
            g[i] = (u[i] > 0 ? hi[i] : u[i] < 0 ? lo[i] : cl) - c;
            n2 += g[i] * g[i];
        }
        if (L < best) { best = L; memcpy(ub, u, NR * sizeof(int64_t)); }
        if ((best >> LR_F) <= T || n2 == 0 || it >= max_iterations) break;
        int64_t s = (L - (T << LR_F)) / n2;
        if (s <= 0) break;
        if (s > 2 * LR_U) s = 2 * LR_U;      /* any larger step clamps every moved multiplier to +-U as well */
        for (int i = 0; i < NR; ++i) {
            const int64_t v = u[i] - s * g[i];
            u[i] = v < -LR_U ? -LR_U : v > LR_U ? LR_U : v;
        }
    }
    *bound = best >> LR_F;
    *iterations_run = it;
    if (multipliers) memcpy(multipliers, ub, NR * sizeof(int64_t));
out:
    free(in.rstart); free(in.order); free(in.a3); free(in.a4); free(in.intop);
    free(u); free(ub); free(lo); free(hi); free(cnt); free(g);
    return rc;
}

int lagrange_ref_fraction_bits(void) { return LR_F; }
int64_t lagrange_ref_box(void) { return LR_U; }
