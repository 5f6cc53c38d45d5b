// kao_device_t.cuh — column-major ("transposed") full evaluator of one candidate by one warp.
//
// Same result as eval_candidate (kao_device.cuh, docs/MODEL.md §3) for the layout class of the
// headline configuration: rows of up to 64 slots, 8-slot rack fields, "at most one replica of a
// partition per rack" (C7 bounds 0..1), an objective whose non-zero terms fit 8 term planes.
// The base is ALSO kept transposed in shared memory: for every slot s a bitmap over the partitions
// (32 per word), two planes:
//   q = 0  replicas            T0[s] bit p  <=>  partition p has a replica on slot s
//   q = 1  leader one-hot      T1[s] bit p  <=>  ... and is led from s
// and the objective as the reference writes it — a sum over the variables with a non-zero weight
// (README.md:145-146: `max: 1 t1b12p5 + 4 t1b19p6_l + ...`, only existing placements appear) — as up to
// eight TERM PLANES over the partitions (host: kao_host.hpp): all terms of plane j have the value
// z_value[j] and one kind (replica on / leadership of the term's slot), a partition has at most one term
// per plane, and
//   Z[j] bit p  <=>  term j of partition p holds in the base   =>   objective = sum_j z_value[j] * popc(Z[j]).
// The evaluation walks the matrix twice, each time with all data of a constraint inside one lane:
//   rows     (C1, C7, objective)  a lane owns 32 PARTITIONS (one word of every rack-field plane and of every term
//            plane).  Next to T and Z the base is kept as RACK-FIELD PLANES A[b] (bit p <=> partition p holds a
//            replica in the 8-slot rack field b: the (partition x rack) occupancy matrix).  From the words A[b][w] the
//            bit-sliced sum z = racks in use, and C1 + C7 of all rows together as sums: rows with z == RF cost
//            2 n - z - RF each (n from the column totals), the few with z != RF are corrected one by one from
//            the row-major base (rows_pass).  No popcount per row.  The objective is one POPC per term plane;
//   columns  (C2-C6)  a lane owns one SLOT per row word: replica and leader totals of its columns are
//            popcount sums over the partition words — no bit-sliced column counters, no cross-lane
//            reduce-scatter.
// The candidate's <= 3 patched rows are scored from the patch itself by the thread that generated the candidate:
// their C1 / C7 terms and objective terms (patch_terms) and, per slot, what they change in the column totals
// (patch_column_deltas: replicas and valid leaderships of the patched rows of the candidate minus those of the same
// rows of the base).  The row pass masks the patched partitions out of the base, the column pass sums the base's
// planes in full and every lane adds the delta of its own slot — so every row of the candidate is evaluated, none
// is taken from a previous evaluation.  Model: /root/reference/README.md:144-185.
#pragma once
#include "kao_device.cuh"

namespace kao {

// kNW: partition words per slot fixed at compile time (32 = 1024 padded partitions, the headline
// shape: every shared-memory offset of the evaluator is then an immediate), 0 = read at run time.
// The other parameters are SCHEDULES of the same arithmetic (kao_set_schedule; results identical):
//   kSync      how the warps of a CTA meet before an evaluation: 0 block barrier (all warps walk the
//              evaluator together), 1 warp only (one warp's generator overlaps another's evaluation), 2 warp only
//              with the column loop kept a loop (a third less evaluator code for the instruction cache), 3 / 4 that loop
//              unrolled by 2 / 4
//   kPop       how the two popcount streams (column totals, leader totals) trade POPC (XU pipe, 8 cycles
//              a warp) for carry-save LOP3 (ALU pipe, 2 cycles): one hex digit per stream, 0 = a POPC per
//              word, 1 = three per four words, 2 = two, 3 = one (Harley-Seal accumulators carried across
//              the whole column)
//              a third hex digit picks where the sums are formed: 0 = the popcount streams above, 1 = on the tensor
//              cores, a binary MMA over a batch of 32 candidates (kao_device_mma.cuh; the two low digits and kSync
//              then play no part)
//              with the third digit 3 the MMA epilogue scores two candidates per instruction in 16 x 2 halfword pairs
//              (kao_device_mma.cuh, eval_batch_mma); a fourth hex digit 1 keeps it in 32 bits per candidate
//   kThreads   threads per CTA (0 = threads_for<W>()); fewer threads = more registers per thread
template <int W_, int kNW_ = 0, int kSync_ = 1, int kPop_ = 0x22, int kThreads_ = 0>
struct EvalCfgT {
    static constexpr int W = W_, NPH = 5, kRack = 3, kObj = 3, kNW = kNW_;
    static constexpr int kSync = kSync_, kPop = kPop_, kThreads = kThreads_;
    static constexpr int kSums = (kPop_ >> 8) & 15;
    static constexpr bool kPacked = kSums == 3 && !((kPop_ >> 12) & 1);
    static_assert(!((kPop_ >> 12) & 1) || kSums == 3, "the 32-bit epilogue digit applies to the sorted-batch body");
    static constexpr bool kTrans = true;
};
constexpr int kTPlanes = 2;
constexpr int kZPlanes = 8;          // term planes of the objective: [kZPlanes][nW] words behind the transposed planes
template <int W> __host__ __device__ constexpr int kAPlanes() { return 4 * W; }     // rack-field planes behind the term planes

// C1 + C7 of one row held row-major (a patched row of the candidate, or a row the vertical pass
// flagged): same terms as row_rack_terms<W, 3>
template <int W> __device__ __forceinline__ int row_terms_hi1_s8(const uint32_t (&x)[W], int RF)
{
    int n = 0, nz = 0;
#pragma unroll
    for (int t = 0; t < W; ++t) {
        n += __popc(x[t]);
        nz += __popc((((x[t] & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x[t]) & 0x80808080u);
    }
    return abs(n - RF) + (n - nz);
}

#if defined(KAO_HOST_EMU)
inline long long emu_rows_charged_one_by_one = 0;
#endif
// ------------------------------------------------------------------------------------------
// rows: C1 + C7 of every partition that is not patched, 32 partitions per lane — as sums, not row by row.
// With "at most one replica per rack" a row of n replicas in z racks costs |n - RF| (C1) + (n - z) (C7).
// Per 8-slot rack field one word `any` (the field holds a replica: the rack-field planes) and the bit-sliced sum z of these
// words.  Rows with z == RF have n >= RF, so over them  sum |n - RF| + (n - z)  =  2 sum n - sum z - RF * #rows;
// rows with z != RF (`flagged`, rare: short rows, rows with a doubled rack) are charged the difference to their
// exact terms one by one from the row-major base.  sum n over the unpatched rows is (sum of the column totals) -
// (replicas in the patched rows): the column pass has it anyway.  So this pass returns, per lane,
//     - sum_b popc(any_b) - RF * popc(scored partitions)  +  for every flagged row  |n - RF| - n + RF
// and the caller adds twice its column totals minus twice the replicas of the patched rows.  Exact for every
// bit-plane (also rows with more than RF replicas); no popcount per row, no search for doubled fields.
// ------------------------------------------------------------------------------------------
template <int W, bool kShared, int kNW>
__device__ __forceinline__ int rows_pass(const Params &d, const MemRef<kShared> &Z, const MemRef<kShared> &bitsT,
                                         int nW_rt, int lane, const PatchSet &ps, int &obj)
{
    const int Ppad = d.Ppad, P = d.P, RF = d.RF;
    const int nW = kNW ? kNW : nW_rt;
    constexpr int NB = 4 * W;                       // 8-slot blocks = rack fields
    int viol = 0;
    const uint32_t rf0 = d.rf_mask[0], rf1 = d.rf_mask[1], rf2 = d.rf_mask[2], rf3 = d.rf_mask[3];   // kernel parameters: constant-bank operands
#pragma unroll 1
    for (int w = lane; w < nW; w += 32) {
        const int left = P - 32 * w;                // partitions of this word that exist
        uint32_t valid = left >= 32 ? ~0u : (left <= 0 ? 0u : ((1u << left) - 1u));
#pragma unroll
        for (int i = 0; i < kMaxOps; ++i)           // unused patches hold -1: (-1 >> 5) never equals w
            valid &= ((ps.p[i] >> 5) == w) ? ~(1u << (ps.p[i] & 31)) : ~0u;
        // objective: the terms that hold, one POPC per term plane (planes nz.. are empty and weigh nothing)
#pragma unroll
        for (int j = 0; j < 4; ++j) obj += __popc(Z.ld32((uint32_t)(j * nW + w) * 4u) & valid) * d.z_value[j];
        if (d.nz > 4) {
#pragma unroll
            for (int j = 4; j < kZPlanes; ++j) obj += __popc(Z.ld32((uint32_t)(j * nW + w) * 4u) & valid) * d.z_value[j];
        }
        // rack-field planes of the base (behind the term planes): bit p of A[b][w] <=> partition p holds a replica in
        // rack field b — the (partition x rack) occupancy matrix, kept in step with the base like T and Z
        uint32_t any[NB];
#pragma unroll
        for (int b = 0; b < NB; ++b) any[b] = Z.ld32((uint32_t)((kZPlanes + b) * nW + w) * 4u) & valid;
        // z = number of rack fields in use, bit-sliced (0..8)
        uint32_t z1, z2, z4 = 0, z8 = 0;
        if constexpr (NB == 4) {
            uint32_t c1, s1;
            csa(c1, s1, any[0], any[1], any[2]);
            z1 = s1 ^ any[3];
            const uint32_t c2 = s1 & any[3];
            z2 = c1 ^ c2;
            z4 = c1 & c2;
        } else {
            uint32_t c1, s1, c2, s2, c3, s3, e1, t1;
            csa(c1, s1, any[0], any[1], any[2]);
            csa(c2, s2, any[3], any[4], any[5]);
            csa(c3, s3, s1, s2, any[6]);
            z1 = s3 ^ any[7];
            const uint32_t c4 = s3 & any[7];
            csa(e1, t1, c1, c2, c3);
            z2 = t1 ^ c4;
            const uint32_t e2 = t1 & c4;
            z4 = e1 ^ e2;
            z8 = e1 & e2;
        }
        // sum of z over the scored rows = racks in use, from the bit planes of z (4 popcounts instead of one per field)
        viol -= __popc(z1) + 2 * __popc(z2) + 4 * __popc(z4) + 8 * __popc(z8) + RF * __popc(valid);
        const uint32_t flagged = ((z1 ^ rf0) | (z2 ^ rf1) | (z4 ^ rf2) | (z8 ^ rf3)) & valid;    // z != RF
        for (uint32_t m = flagged; m; m &= m - 1) { // rare: the row's exact C1 term in place of the n >= RF form
#if defined(KAO_HOST_EMU)
            ++emu_rows_charged_one_by_one;          // tests/emu: a well-formed row must never come here
#endif
            const int p = 32 * w + __ffs(m) - 1;
            int n = 0;
#pragma unroll
            for (int t = 0; t < W; ++t) n += __popc(bitsT.ld32((uint32_t)(t * Ppad + p) * 4u));
            viol += abs(n - RF) - n + RF;
        }
    }
    return viol;
}

// One popcount stream of the column pass: words arrive four at a time (one 128-bit load), the total is
// read once per candidate.  kLvl picks how many of the four popcounts are replaced by carry-save adders:
//   0  popc(a) + popc(b) + popc(c) + popc(d)                                            4 POPC
//   1  a + b + c = 2 maj + xor                                                          3 POPC, 2 LOP3
//   2  a running `ones` word absorbs the words two at a time, the carries are counted   2 POPC, 4 LOP3
//   3  Harley-Seal: running `ones` and `twos`, only the weight-4 carry is counted       1 POPC, 6 LOP3
template <int kLvl> struct PopStream {
    uint32_t ones = 0, twos = 0;
    int n1 = 0, n2 = 0, n4 = 0;
    __device__ __forceinline__ void add4(uint32_t a, uint32_t b, uint32_t c, uint32_t d)
    {
        if constexpr (kLvl == 0) {
            n1 += __popc(a) + __popc(b) + __popc(c) + __popc(d);
        } else if constexpr (kLvl == 1) {
            uint32_t h, l;
            csa(h, l, a, b, c);
            n1 += __popc(l) + __popc(d);
            n2 += __popc(h);
        } else if constexpr (kLvl == 2) {
            uint32_t c1, c2;
            csa(c1, ones, ones, a, b);
            csa(c2, ones, ones, c, d);
            n2 += __popc(c1) + __popc(c2);
        } else {
            uint32_t c1, c2, f;
            csa(c1, ones, ones, a, b);
            csa(c2, ones, ones, c, d);
            csa(f, twos, twos, c1, c2);
            n4 += __popc(f);
        }
    }
    __device__ __forceinline__ int total() const
    {
        if constexpr (kLvl <= 1) return n1 + 2 * n2;
        else if constexpr (kLvl == 2) return __popc(ones) + 2 * n2;
        else return __popc(ones) + 2 * __popc(twos) + 4 * n4;
    }
};

// ------------------------------------------------------------------------------------------
// C1 / C7 terms and objective terms of the candidate's patched rows, from the rows themselves (one thread:
// the per-thread generator of the search kernels calls this for its own candidate)
// ------------------------------------------------------------------------------------------
template <int W>
__device__ __forceinline__ void patch_terms(const Params &d, const PatchSet &ps, const uint32_t (&rows)[kMaxOps][W], int &pviol, int &pobj,
                                            int &pcount)
{
    pviol = 0;
    pobj = 0;
    pcount = 0;                                     // replicas in the patched rows (the column totals include them)
#pragma unroll
    for (int i = 0; i < kMaxOps; ++i) {
        if (ps.p[i] < 0) continue;
        pviol += row_terms_hi1_s8<W>(rows[i], d.RF);
        pcount += row_count<W>(rows[i]);
        const uint32_t *zs = reinterpret_cast<const uint32_t *>(d.zslot + (size_t)ps.p[i] * kZPlanes);
        const uint32_t z03 = zs[0], z47 = d.nz > 4 ? zs[1] : 0xFFFFFFFFu;
#pragma unroll
        for (int j = 0; j < kZPlanes; ++j) {
            if (j >= 4 && d.nz <= 4) break;
            const int slot = (int)(((j < 4 ? z03 : z47) >> (8 * (j & 3))) & 0xFFu);      // 0xFF (no term) is never a slot of the row
            const bool has = row_has<W>(rows[i], slot);
            const bool on = ((d.z_on_leader >> j) & 1) ? (has && (int)ps.ld[i] == slot) : has;
            pobj += on ? d.z_value[j] : 0;
        }
    }
}

// ------------------------------------------------------------------------------------------
// What the candidate's patched rows change in the column totals, per slot: one byte per slot, low nibble =
// 4 + (replicas on the slot in the patched rows of the candidate) - (... in the same rows of the base), high
// nibble = the same for valid leaderships (|net| <= kMaxOps).  Computed from the rows themselves by the thread
// that generated the candidate (like patch_terms) and parked next to it; the column pass sums the base's planes
// in full and every lane adds the byte of its own slot.  out: [32 * W] bytes, private to the calling thread.
// ------------------------------------------------------------------------------------------
constexpr uint32_t kDeltaBias = 0x44444444u;
template <int W>
__device__ __forceinline__ void patch_column_deltas(const Params &d, const PatchSet &ps, const uint32_t (&rows)[kMaxOps][W],
                                                    const uint32_t *bitsT, const uint8_t *leader, uint8_t *out)
{
    static_assert(kMaxOps <= 3, "a nibble holds 4 +- kMaxOps");
    uint32_t *ow = reinterpret_cast<uint32_t *>(out);
#pragma unroll
    for (int k = 0; k < 8 * W; ++k) ow[k] = kDeltaBias;
#pragma unroll
    for (int i = 0; i < kMaxOps; ++i) {
        const int p = ps.p[i];
        if (p < 0) continue;
        uint32_t old[W];
#pragma unroll
        for (int t = 0; t < W; ++t) old[t] = bitsT[(size_t)t * d.Ppad + p];
        const int old_ld = leader[p], new_ld = (int)ps.ld[i];
#pragma unroll
        for (int t = 0; t < W; ++t)
            for (uint32_t m = rows[i][t] ^ old[t]; m; m &= m - 1) {
                const int s = 32 * t + __ffs(m) - 1;
                out[s] = (uint8_t)(out[s] + (row_has<W>(rows[i], s) ? 1 : -1));
            }
        if (old_ld < 32 * W && row_has<W>(old, old_ld)) out[old_ld] = (uint8_t)(out[old_ld] - 0x10);
        if (new_ld < 32 * W && row_has<W>(rows[i], new_ld)) out[new_ld] = (uint8_t)(out[new_ld] + 0x10);
    }
}

// The bounds a lane checks its own columns against, read once per round: C3 / C4 of slots `lane` and `lane + 32`,
// and (used by the first lane of every 8-lane rack group) C6 of those slots' racks — a rack field beyond R gets
// [0, INT_MAX], which no total violates.  Rack bounds are whatever the caller passed (any int32), so they stay whole words.
template <int W> struct LaneBounds {
    int rep_lo[W], rep_hi[W], ldr_lo[W], ldr_hi[W], rack_lo[W], rack_hi[W];
    __device__ __forceinline__ void load(const Consts *cs, int lane, int R)
    {
#pragma unroll
        for (int t = 0; t < W; ++t) {
            const int s = lane + 32 * t, rk = s >> 3;
            rep_lo[t] = (int)(cs->bnd_rep[s] & 0xFFFFu); rep_hi[t] = (int)(cs->bnd_rep[s] >> 16);
            ldr_lo[t] = (int)(cs->bnd_ldr[s] & 0xFFFFu); ldr_hi[t] = (int)(cs->bnd_ldr[s] >> 16);
            rack_lo[t] = rk < R ? cs->rack_lo[rk] : 0;
            rack_hi[t] = rk < R ? cs->rack_hi[rk] : 0x7FFFFFFF;
        }
    }
};

// ------------------------------------------------------------------------------------------
// the whole candidate.  T: the two transposed planes; Z: the term planes [kZPlanes][nW]; bits: the row-major
// base; lb: this lane's bounds; pdelta: patch_column_deltas of this candidate; pviol / pobj / pcount: patch_terms of its patched rows
// ------------------------------------------------------------------------------------------
template <class Cfg, bool kShared>
__device__ void eval_candidate_t(const Params &d, const uint32_t *Tp, int nW_rt, const uint32_t *bitsT, const uint32_t *Zp,
                                 const LaneBounds<Cfg::W> &lb, const PatchSet &ps, const uint8_t *pdelta, int pviol, int pobj, int pcount,
                                 int lane, int &viol_out, int &obj_out)
{
    constexpr int W = Cfg::W, kNW = Cfg::kNW;
    constexpr int NSL = 32 * W;
    const int nW = kNW ? kNW : nW_rt;
    const MemRef<kShared> T(Tp), B(bitsT), Z(Zp);
    // ---- rows: unpatched partitions from the transposed bit-plane and the term planes, patched ones from the patch
    int obj = 0;
    int viol = rows_pass<W, kShared, kNW>(d, Z, B, nW, lane, ps, obj);
    if (lane == 0) { viol += pviol - 2 * pcount; obj += pobj; }    // the patched rows' own terms; their replicas are not the row pass's
    // ---- columns: this lane owns slot `lane` of every row word.  The planes of the base are summed in full; what
    // the candidate's patched rows change in this lane's columns is one byte of pdelta (patch_column_deltas)
    PopStream<(Cfg::kPop >> 0) & 15> cnt[W];
    PopStream<(Cfg::kPop >> 4) & 15> lcnt[W];
    const int nch = nW >> 2;                        // chunks of 128 partitions
    const bool swz = t_swizzled(nW);
    const uint32_t rot = swz ? 16u * (uint32_t)(lane & 7) : 0u;     // byte offset XORed into the chunk offset
    auto load = [&](int j, uint4 (&col)[W], uint4 (&oh)[W]) {
        const uint32_t off = ((uint32_t)j * 16u) ^ rot;             // logical chunk j of this lane's slots
#pragma unroll
        for (int t = 0; t < W; ++t) {
            const int s = lane + 32 * t;
            col[t] = T.ld128((uint32_t)((0 * NSL + s) * nW) * 4u + off);
            oh[t] = T.ld128((uint32_t)((1 * NSL + s) * nW) * 4u + off);
        }
    };
    auto add = [&](const uint4 (&col)[W], const uint4 (&oh)[W]) {
#pragma unroll
        for (int t = 0; t < W; ++t) {
            cnt[t].add4(col[t].x, col[t].y, col[t].z, col[t].w);
            lcnt[t].add4(oh[t].x, oh[t].y, oh[t].z, oh[t].w);
        }
    };
    if constexpr (kNW == 32 && Cfg::kSync < 2) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { uint4 c[W], o[W]; load(j, c, o); add(c, o); }
    } else if constexpr (Cfg::kSync == 3) {          // nch is even (t_words rounds to whole groups of 8 words)
#pragma unroll 2
        for (int j = 0; j < nch; ++j) { uint4 c[W], o[W]; load(j, c, o); add(c, o); }
    } else if constexpr (Cfg::kSync == 4) {
#pragma unroll 4
        for (int j = 0; j < nch; ++j) { uint4 c[W], o[W]; load(j, c, o); add(c, o); }
    } else {
#pragma unroll 1
        for (int j = 0; j < nch; ++j) { uint4 c[W], o[W]; load(j, c, o); add(c, o); }
    }
    // ---- C3 / C4 on this lane's columns, C2/C5 as P - sum of valid leaders, C6 per 8-lane rack group
    // (rack totals: the W column totals of a lane travel packed in one word through three butterfly steps
    // inside the 8-lane group — a partial-mask warp reduction would run once per group, one after the other)
    static_assert(W <= 2, "two 16-bit totals per word");
    uint32_t packed = 0;
#pragma unroll
    for (int t = 0; t < W; ++t) {
        const int s = lane + 32 * t;
        const int pd = pdelta[s];
        const int c = cnt[t].total() + (pd & 15) - 4, l = lcnt[t].total() + (pd >> 4) - 4;
        packed |= (uint32_t)c << (16 * t);                      // c <= P < 8192: the sum of 8 lanes stays below 2^16
        viol += 2 * c - l + max(c - lb.rep_hi[t], 0) + max(lb.rep_lo[t] - c, 0) + max(l - lb.ldr_hi[t], 0) + max(lb.ldr_lo[t] - l, 0);   // 2 c: see rows_pass
    }
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) packed += __shfl_xor_sync(0xFFFFFFFFu, packed, o);
    if ((lane & 7) == 0) {
#pragma unroll
        for (int t = 0; t < W; ++t) {
            const int tot = (int)((packed >> (16 * t)) & 0xFFFFu);
            viol += max(tot - lb.rack_hi[t], 0) + max(lb.rack_lo[t] - tot, 0);
        }
    }
    viol_out = __reduce_add_sync(0xFFFFFFFFu, viol) + d.P;
    obj_out = __reduce_add_sync(0xFFFFFFFFu, obj);
}

// ------------------------------------------------------------------------------------------
// keeping the transposed planes in step with the row-major base (search kernels; tests/emu)
// ------------------------------------------------------------------------------------------
// one word (32 partitions) of plane q, slot s, gathered from the row-major tables
template <int W>
__device__ __forceinline__ uint32_t t_gather(int q, int s, int w, const uint32_t *bitsT, const uint8_t *leader, int Ppad)
{
    uint32_t out = 0;
    const int sw = s >> 5, sb = s & 31;
    for (int b = 0; b < 32; ++b) {
        const int p = 32 * w + b;
        if (p >= Ppad) break;                       // padding words of the plane (t_words)
        const uint32_t has = (bitsT[(size_t)sw * Ppad + p] >> sb) & 1u;
        const uint32_t led = has & ((int)leader[p] == s ? 1u : 0u);
        out |= (q == 0 ? has : led) << b;
    }
    return out;
}
// does term j of partition p hold for the row (row, ld)
template <int W>
__device__ __forceinline__ bool z_term_holds(const Params &d, int j, int p, const uint32_t (&row)[W], uint32_t ld)
{
    const int slot = d.zslot[(size_t)p * kZPlanes + j];
    const bool has = row_has<W>(row, slot);                     // 0xFF (no term) is never a slot of the row
    return ((d.z_on_leader >> j) & 1) ? (has && (int)ld == slot) : has;
}
// one word (32 partitions) of term plane j
template <int W>
__device__ __forceinline__ uint32_t z_gather(const Params &d, int j, int w, const uint32_t *bitsT, const uint8_t *leader)
{
    uint32_t out = 0;
    for (int b = 0; b < 32; ++b) {
        const int p = 32 * w + b;
        if (p >= d.P) break;
        uint32_t row[W];
#pragma unroll
        for (int t = 0; t < W; ++t) row[t] = bitsT[(size_t)t * d.Ppad + p];
        out |= (z_term_holds<W>(d, j, p, row, leader[p]) ? 1u : 0u) << b;
    }
    return out;
}
// one word (32 partitions) of rack-field plane b: the partition holds a replica in the 8-slot field b
template <int W>
__device__ __forceinline__ uint32_t a_gather(int b, int w, const uint32_t *bitsT, int Ppad)
{
    uint32_t out = 0;
    for (int i = 0; i < 32; ++i) {
        const int p = 32 * w + i;
        if (p >= Ppad) break;
        out |= (((bitsT[(size_t)(b >> 2) * Ppad + p] >> (8 * (b & 3))) & 0xFFu) ? 1u : 0u) << i;
    }
    return out;
}
// Row p of the base becomes (newrow, newld): every lane rewrites bit p of its own slots' words in both
// transposed planes, lanes 0..7 bit p of one term plane each, the next 4 W lanes bit p of one rack-field plane each,
// with kS the next four bit p of one shortfall plane each (kao_device_mma.cuh)
// (the whole warp calls this; the row-major base itself is patched by the caller).
template <int W, bool kS = false>
__device__ __forceinline__ void t_patch_row(const Params &d, uint32_t *T, uint32_t *Z, int nW, int p, const uint32_t (&newrow)[W],
                                            uint32_t newld, int lane)
{
    constexpr int NSL = 32 * W;
    const int w = p >> 5;
    const uint32_t bit = 1u << (p & 31);
#pragma unroll
    for (int t = 0; t < W; ++t) {
        const int s = lane + 32 * t;
        const bool has = (newrow[t] >> lane) & 1u;
        const bool led = has && ((int)newld == s);
#pragma unroll
        for (int q = 0; q < kTPlanes; ++q) {
            const bool on = q == 0 ? has : led;
            uint32_t &word = T[t_word(q, s, w, nW, NSL)];
            word = on ? (word | bit) : (word & ~bit);
        }
    }
    if (lane < kZPlanes) {
        uint32_t &word = Z[lane * nW + w];
        word = z_term_holds<W>(d, lane, p, newrow, newld) ? (word | bit) : (word & ~bit);
    } else if (lane < kZPlanes + kAPlanes<W>()) {
        const int b = lane - kZPlanes;
        uint32_t &word = Z[lane * nW + w];
        word = ((newrow[b >> 2] >> (8 * (b & 3))) & 0xFFu) ? (word | bit) : (word & ~bit);
    } else if (kS && lane < kZPlanes + kAPlanes<W>() + 4) {
        const int k = lane - kZPlanes - kAPlanes<W>(), short_by = max(d.RF - row_count<W>(newrow), 0);
        uint32_t &word = Z[lane * nW + w];
        word = ((short_by >> k) & 1) ? (word | bit) : (word & ~bit);
    }
}

}  // namespace kao
