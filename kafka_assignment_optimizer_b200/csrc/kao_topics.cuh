// kao_topics.cuh — the per-topic balance rows of a topic session (docs/MODEL.md §10, DESIGN.md §7.2) on the device:
// the tables (TopicArgs) and how a candidate or a winner changes their counts and violation.  The HBM-base search
// kernel (kao_large.cu) uses these functions, and the host emulator (tests/emu) compiles the same ones.
#pragma once
#include "kao_device.cuh"

// Per-topic balance rows of a topic session, all in HBM.  The counts are those of the base over broker slots (padding
// slots are never counted nor read); CTA 0 patches them and tviol from each round's winner before the second grid
// barrier.
struct TopicArgs {
    int T;
    const uint16_t *topic_of;       // [Ppad] topic of each partition
    const int4 *bnd;                // [T] (C3t lo, C3t hi, C4t lo, C4t hi)
    uint16_t *tcnt, *tlcnt;         // [T][32 W] replicas / valid leaders of each topic per slot
    int *tviol;                     // the base's violation of the topic rows
};

namespace kao {

// slot s holds a broker (is no padding slot) and so has a topic row: its order index is below B.  Padding slots have
// order index 0xFF in Consts, which with B = 256 would be slot 255's own index, so the test is never "!= 0xFF".
__device__ __forceinline__ bool broker_slot(const Consts *cs, int B, int s) { return cs->order_of_slot[s] < B; }

__device__ __forceinline__ int band_int(int c, int lo, int hi) { return max(c - hi, 0) + max(lo - c, 0); }

// The topic events of a candidate (docs/MODEL.md §10): a patched row differs from the base by at most one replica
// move and one leader change, so it gives at most one -1 / +1 replica event and one -1 / +1 valid-leader event, each on
// the cell topic * 32 W + slot.  Padding slots carry no topic row: -1 (no event) there.
// Events of patched row i (partition p, leader ldo -> ldn, words old_word(w) -> new_word(w)) into entries 2 i, 2 i + 1.
template <int W, class Old, class New>
__device__ __forceinline__ void topic_row_events(const TopicArgs &ta, const Consts *cs, int B, int i, int p, int ldo,
                                                 int ldn, Old old_word, New new_word, int (&rc)[2 * kMaxOps],
                                                 int (&lc)[2 * kMaxOps])
{
    constexpr int NSL = 32 * W;
    auto cell = [&](int t, int s) { return (s >= 0 && broker_slot(cs, B, s)) ? t * NSL + s : -1; };
    const int t = ta.topic_of[p];
    // one word at a time (no row copies: the W = 8 kernel has no registers to spare)
    int rs = -1, as = -1;
    bool oko = false, okn = false;
#pragma unroll
    for (int w = 0; w < W; ++w) {
        const uint32_t o = old_word(w), n = new_word(w);
        if (o & ~n) rs = 32 * w + __ffs(o & ~n) - 1;
        if (n & ~o) as = 32 * w + __ffs(n & ~o) - 1;
        if ((ldo >> 5) == w) oko = (o >> (ldo & 31)) & 1u;
        if ((ldn >> 5) == w) okn = (n >> (ldn & 31)) & 1u;
    }
    rc[2 * i] = cell(t, rs);
    rc[2 * i + 1] = cell(t, as);
    lc[2 * i] = cell(t, oko ? ldo : -1);
    lc[2 * i + 1] = cell(t, okn ? ldn : -1);
}

// the events of a candidate against the base: entry 2 i is row i's -1 event, 2 i + 1 its +1 event (-1: none)
template <int W>
__device__ __forceinline__ void topic_events(const Params &d, const TopicArgs &ta, const Consts *cs, const PatchSet &ps,
                                             const uint32_t (&rows)[kMaxOps][W], int (&rc)[2 * kMaxOps],
                                             int (&lc)[2 * kMaxOps])
{
#pragma unroll
    for (int i = 0; i < kMaxOps; ++i) {
        rc[2 * i] = rc[2 * i + 1] = lc[2 * i] = lc[2 * i + 1] = -1;
        if (i < ps.n) {
            const int p = ps.p[i];
            topic_row_events<W>(ta, cs, d.B, i, p, d.leader[p], (int)ps.ld[i],
                                [&](int w) { return d.bitsT[(size_t)w * d.Ppad + p]; },
                                [&](int w) { return rows[i][w]; }, rc, lc);
        }
    }
}

// change of the topic-row violation from the base to the candidate: the events netted per cell, <= 12 counts read
template <int W>
__device__ __forceinline__ int topic_delta(const TopicArgs &ta, const int (&rc)[2 * kMaxOps], const int (&lc)[2 * kMaxOps])
{
    constexpr int LOG2_NSL = W == 1 ? 5 : W == 2 ? 6 : W == 4 ? 7 : 8;
    int val[2 * kMaxOps];
#pragma unroll
    for (int j = 0; j < 2 * kMaxOps; ++j) val[j] = (j & 1) ? 1 : -1;
    int dv = apply_events<2 * kMaxOps>(rc, val, [&](int c, int net) {
        const int4 b = __ldg(ta.bnd + (c >> LOG2_NSL));
        const int n = ta.tcnt[c];
        return band_int(n + net, b.x, b.y) - band_int(n, b.x, b.y);
    });
    dv += apply_events<2 * kMaxOps>(lc, val, [&](int c, int net) {
        const int4 b = __ldg(ta.bnd + (c >> LOG2_NSL));
        const int n = ta.tlcnt[c];
        return band_int(n + net, b.z, b.w) - band_int(n, b.z, b.w);
    });
    return dv;
}

// a winner's events (topic_row_events of its old and new rows) applied to the base: tviol and the counts follow them
template <int W>
__device__ __forceinline__ void topic_apply_events(const TopicArgs &ta, const int (&rc)[2 * kMaxOps],
                                                   const int (&lc)[2 * kMaxOps])
{
    *ta.tviol += topic_delta<W>(ta, rc, lc);
#pragma unroll
    for (int j = 0; j < 2 * kMaxOps; ++j) {
        const int v = (j & 1) ? 1 : -1;
        if (rc[j] >= 0) ta.tcnt[rc[j]] = (uint16_t)(ta.tcnt[rc[j]] + v);
        if (lc[j] >= 0) ta.tlcnt[lc[j]] = (uint16_t)(ta.tlcnt[lc[j]] + v);
    }
}

}  // namespace kao
