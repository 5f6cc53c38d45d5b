// kao_large.cu — the large-instance path (DESIGN.md §7.1): 8,161 .. 65,280 partitions.  Every other search kernel
// stages the base in shared memory for the whole launch, which caps the row count at 8,160; here the base and the
// tables derived from it live in HBM (L2-resident: 7.5 MB at 65,280 x 256 slots) and every CTA keeps only the
// per-slot totals of the base in shared memory.  Same candidate stream, keys and winners as MODEL §5 / §6; candidates
// are scored by delta evaluation (MODEL §8), one thread each.
//
// This translation unit is compiled with -Xptxas -dlcm=cg: plain global loads bypass L1, so the base that CTA 0
// patches between two grid barriers is never read from a stale L1 line by another SM.  (Only the objective table,
// which no kernel writes, is read through the read-only path, __ldg in MemRef<false>.)
#include "kao_large.hpp"

namespace {

constexpr int kLT = 512;     // threads per CTA of the search and evaluation kernels
// the one evaluator configuration of the large path: general rack bounds (for C7 = 0..1 they give the values of the
// 8 / 16-slot forms), objective from packed weight entries or the dense table.  NPH is unused by delta evaluation.
template <int W> using LargeCfg = EvalCfg<W, 5, 0, kObjEntries>;

__device__ __forceinline__ void load_consts(Consts *s, const Consts *g)
{
    const uint4 *src = reinterpret_cast<const uint4 *>(g);
    uint4 *dst = reinterpret_cast<uint4 *>(s);
    for (int i = threadIdx.x; i < (int)(sizeof(Consts) / 16); i += blockDim.x) dst[i] = src[i];
}

template <class T> __device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    return v;
}

// Full evaluation of one assignment by the whole CTA: the per-row terms (C1, C2/C5, C7, objective) of row_eval, the
// replica and valid-leader count per slot and the replica count per rack in shared memory, then the C3 / C4 / C6
// bands.  Leaves cnt / lcnt / rc filled (the totals delta evaluation starts from); acc = (violation, objective).
// kRF: each row's C1 / C7 operands from rftab (docs/MODEL.md §11).
template <int W, bool kRF = false>
__device__ void block_eval(const Params &d, const Consts *cs, const uint32_t *bits, const uint8_t *leader,
                           int *cnt, int *lcnt, int *rc, long long *acc, const uint32_t *rftab = nullptr)
{
    const int tid = threadIdx.x, lane = tid & 31;
    for (int i = tid; i < 256; i += blockDim.x) { cnt[i] = 0; lcnt[i] = 0; if (i < 32) rc[i] = 0; }
    if (tid < 2) acc[tid] = 0;
    __syncthreads();
    const MemRef<false> m_obj(d.swT);
    long long v = 0, o = 0;
    for (int p = tid; p < d.P; p += blockDim.x) {
        uint32_t x[W];
#pragma unroll
        for (int t = 0; t < W; ++t) x[t] = bits[(size_t)t * d.Ppad + p];
        const uint32_t ld = leader[p];
        int rv, ro;
        if constexpr (kRF) row_eval<LargeCfg<W>, false, true>(d, m_obj, p, x, ld, rv, ro, row_rf(rftab, p));
        else row_eval<LargeCfg<W>, false>(d, m_obj, p, x, ld, rv, ro);
        v += rv;
        o += ro;
#pragma unroll
        for (int t = 0; t < W; ++t)
            for (uint32_t m = x[t]; m; m &= m - 1) {
                const int s = 32 * t + __ffs(m) - 1;
                atomicAdd(&cnt[s], 1);
                atomicAdd(&rc[s >> d.log2S], 1);
            }
        if ((int)ld < 32 * W && row_has<W>(x, (int)ld)) atomicAdd(&lcnt[ld], 1);
    }
    v = warp_sum(v);
    o = warp_sum(o);
    if (lane == 0) {
        atomicAdd(reinterpret_cast<unsigned long long *>(&acc[0]), (unsigned long long)v);
        atomicAdd(reinterpret_cast<unsigned long long *>(&acc[1]), (unsigned long long)o);
    }
    __syncthreads();
    if (tid < 32) {
        long long bv = 0;
        for (int s = lane; s < 32 * W; s += 32) bv += band_violation(cnt[s], cs->bnd_rep[s]) + band_violation(lcnt[s], cs->bnd_ldr[s]);
        if (lane < d.R) bv += max(rc[lane] - cs->rack_hi[lane], 0) + max(cs->rack_lo[lane] - rc[lane], 0);
        bv = warp_sum(bv);
        if (lane == 0) acc[0] += bv;
    }
    __syncthreads();
}

// the per-thread generator over the HBM base of the current round (list buffers and counts: LargeRecord::state)
template <int W>
__device__ __forceinline__ Gen<W, true, true> large_gen(const Params &d, const LargeArgs &la, const Consts *cs, const int *st)
{
    Gen<W, true, true> tg;
    tg.bitsT = d.bitsT; tg.leader = d.leader; tg.cs = cs; tg.d = &d; tg.prow = nullptr; tg.lane = 0;
    tg.D = d.D + (size_t)(st[3] & 1) * d.Ppad; tg.DL = d.DL + (size_t)((st[3] >> 1) & 1) * d.Ppad;
    tg.nD = st[0]; tg.nL = st[1];
    tg.T = la.T; tg.tnW = la.tnW; tg.t_leaders_valid = st[2] == 0;     // "first holder of slot s": plane-row scan
    return tg;
}

// membership of partition p (row, leader) in the displaced lists (as rebuild_lists decides it): a home slot is
// missing (D); the first home slot is held but does not lead (DL)
template <int W>
__device__ __forceinline__ void displaced(uint32_t h4, uint32_t hv, const uint32_t (&row)[W], uint32_t ld, bool &miss,
                                          bool &ldis)
{
    miss = false; ldis = false;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int hs = (h4 >> (8 * i)) & 0xFF;
        if (home_ok<W>(hs, hv, i)) {
            const bool has = row_has<W>(row, hs);
            miss |= !has;
            if (i == 0) ldis = has && ((int)ld != hs);
        }
    }
}

// List changes of one round: at most kMaxOps removals and insertions per list
struct ListChanges {
    int nd[2], ni[2];
    int del[2][kMaxOps], ins[2][kMaxOps];
    int less[2][kMaxOps];
};

// CTA 0, whole block: the round's winner (key k) becomes the base.  Re-materialise it, patch the HBM base, the
// transposed planes and the displaced lists (rewritten, ascending, into their other buffer when they change), and
// write the winner record.  st: the state the round was generated from.
template <int W>
__device__ void apply_winner_large(const Params &d, const LargeArgs &la, const Consts *cs, const int *st, uint64_t seed,
                                   uint32_t round, uint32_t round_size, unsigned long long k, LargeRecord &rec,
                                   ListChanges &lc)
{
    constexpr int NSL = 32 * W;
    const int tid = threadIdx.x, lane = tid & 31;
    if (tid < 32) {
        if (lane == 0) {
            // lane 0 alone: it rewrites the rows the generator reads
            const Gen<W, true, true> tg = large_gen<W>(d, la, cs, st);
            PatchSet ps;
            uint32_t rows[kMaxOps][W];
#pragma unroll
            for (int i = 0; i < kMaxOps; ++i)
#pragma unroll
                for (int t = 0; t < W; ++t) rows[i][t] = 0;
            tg.run(seed, round, (uint32_t)(k & kIdxMask), round_size, ps, rows);
            rec.n = ps.n;
            int nbad = st[2];
            lc.nd[0] = lc.nd[1] = lc.ni[0] = lc.ni[1] = 0;
            for (int i = 0; i < kMaxOps; ++i) {
                if (i >= ps.n) { rec.p[i] = -1; continue; }
                const int p = ps.p[i];
                uint32_t xo[W], xn[W];
#pragma unroll
                for (int t = 0; t < W; ++t) {
                    xo[t] = d.bitsT[(size_t)t * d.Ppad + p];
                    xn[t] = rows[i][t];
                    rec.old_row[i][t] = xo[t];
                    rec.new_row[i][t] = xn[t];
                }
                const uint32_t lo = d.leader[p], ln = ps.ld[i];
                rec.p[i] = p; rec.old_ld[i] = lo; rec.new_ld[i] = ln;
                const bool was = (int)lo < NSL && row_has<W>(xo, (int)lo), is = (int)ln < NSL && row_has<W>(xn, (int)ln);
                nbad += (was ? 0 : -1) + (is ? 0 : 1);
                bool mo, lo_dis, mn, ln_dis;
                const uint32_t h4 = d.homeT[p], hv = home_valid<W>(d.homeT, d.Ppad, p);
                displaced<W>(h4, hv, xo, lo, mo, lo_dis);
                displaced<W>(h4, hv, xn, ln, mn, ln_dis);
                if (mo && !mn) lc.del[0][lc.nd[0]++] = p;
                if (!mo && mn) lc.ins[0][lc.ni[0]++] = p;
                if (lo_dis && !ln_dis) lc.del[1][lc.nd[1]++] = p;
                if (!lo_dis && ln_dis) lc.ins[1][lc.ni[1]++] = p;
#pragma unroll
                for (int t = 0; t < W; ++t) d.bitsT[(size_t)t * d.Ppad + p] = xn[t];
                d.leader[p] = (uint8_t)ln;
            }
            rec.state[2] = nbad;
        }
        __syncwarp();
        // transposed planes: lane l rewrites bit p of slot 32 t + l in T0 (replica) and T1 (replica and leader)
        for (int i = 0; i < rec.n; ++i) {
            const int p = rec.p[i], w = p >> 5;
            const uint32_t bit = 1u << (p & 31);
#pragma unroll
            for (int t = 0; t < W; ++t) {
                const int s = 32 * t + lane;
                const bool ho = (rec.old_row[i][t] >> lane) & 1u, hn = (rec.new_row[i][t] >> lane) & 1u;
                const bool lo = ho && (int)rec.old_ld[i] == s, ln = hn && (int)rec.new_ld[i] == s;
                if (ho != hn) la.T[t_word(0, s, w, la.tnW, NSL)] ^= bit;
                if (lo != ln) la.T[t_word(1, s, w, la.tnW, NSL)] ^= bit;
            }
        }
    }
    __syncthreads();
    int bits = st[3];
    for (int L = 0; L < 2; ++L) {
        const int nd = lc.nd[L], ni = lc.ni[L];
        if (nd + ni == 0) { if (tid == 0) rec.state[L] = st[L]; continue; }
        uint16_t *base = L ? d.DL : d.D;
        const uint16_t *src = base + (size_t)((bits >> L) & 1) * d.Ppad;
        uint16_t *dst = base + (size_t)(((bits >> L) & 1) ^ 1) * d.Ppad;
        const int n = st[L];
        if (tid < kMaxOps) lc.less[L][tid] = 0;
        __syncthreads();
        int less[kMaxOps] = {0, 0, 0};
        for (int i = tid; i < n; i += blockDim.x) {
            const int v = src[i];
            bool gone = false;
            int shift = 0;
            for (int j = 0; j < nd; ++j) { gone |= lc.del[L][j] == v; shift -= lc.del[L][j] < v ? 1 : 0; }
            for (int j = 0; j < ni; ++j) { shift += lc.ins[L][j] < v ? 1 : 0; less[j] += v < lc.ins[L][j] ? 1 : 0; }
            if (!gone) dst[i + shift] = (uint16_t)v;
        }
        for (int j = 0; j < ni; ++j) if (less[j]) atomicAdd(&lc.less[L][j], less[j]);
        __syncthreads();
        if (tid < ni) {
            const int v = lc.ins[L][tid];
            int pos = lc.less[L][tid];
            for (int j = 0; j < nd; ++j) pos -= lc.del[L][j] < v ? 1 : 0;
            for (int j = 0; j < ni; ++j) pos += lc.ins[L][j] < v ? 1 : 0;
            dst[pos] = (uint16_t)v;
        }
        if (tid == 0) rec.state[L] = n - nd + ni;
        bits ^= 1 << L;
    }
    if (tid == 0) {
        rec.state[3] = bits;
        *la.rec = rec;
#pragma unroll
        for (int j = 0; j < 4; ++j) d.nD[j] = rec.state[j];
    }
}

// CTA 0, the thread that wrote the winner record (apply_winner_large): the topic counts and the topic-row violation of
// the base follow the record's old and new rows
template <int W>
__device__ __forceinline__ void apply_winner_topics(const TopicArgs &ta, const Consts *cs, int B, const LargeRecord &rec)
{
    int rc[2 * kMaxOps], lc[2 * kMaxOps];
#pragma unroll
    for (int i = 0; i < kMaxOps; ++i) {
        rc[2 * i] = rc[2 * i + 1] = lc[2 * i] = lc[2 * i + 1] = -1;
        if (i < rec.n)
            topic_row_events<W>(ta, cs, B, i, rec.p[i], (int)rec.old_ld[i], (int)rec.new_ld[i],
                                [&](int w) { return rec.old_row[i][w]; }, [&](int w) { return rec.new_row[i][w]; },
                                rc, lc);
    }
    topic_apply_events<W>(ta, rc, lc);
}

// the search kernel; kTopics: the topic rows of ta are part of the violation; kRF: every row's C1 / C7 operands from
// rftab ([Ppad] packed words, replication_table in kao_host.hpp; docs/MODEL.md §11).  ta and rftab are unused otherwise
// and come last, so that the parameters of the plain instantiations are laid out as without them.
template <int W, bool kTopics, bool kRF>
__global__ void __launch_bounds__(kLT, 1)
search_large_kernel(Params d, LargeArgs la, uint64_t seed, uint32_t first_round, uint32_t rounds, uint32_t round_size,
                    unsigned long long *keys, unsigned int *grid_bar, P2P pp, unsigned long long *all_keys, TopicArgs ta,
                    const uint32_t *rftab)
{
    constexpr int kWarps = kLT / 32, NSL = 32 * W;
    __shared__ Consts s_cs;
    __shared__ int s_cnt[256], s_lcnt[256], s_rc[32];
    __shared__ long long s_acc[2];
    __shared__ int s_base[3];                          // (violation, objective) of the base; [2] = 1: taken from the last key
    __shared__ int s_st[4];                            // LargeRecord::state of the current base
    __shared__ unsigned long long s_red[kWarps + 3];   // per-warp minima; stop flag, best (violation, cost), stall
    __shared__ int s_abort;
    __shared__ LargeRecord s_rec;
    __shared__ ListChanges s_lc;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    load_consts(&s_cs, d.consts);
    if (tid < 4) s_st[tid] = __ldcg(d.nD + tid);
    if (tid == 0) {
        s_abort = 0; s_base[2] = 0;
        s_red[kWarps] = 0; s_red[kWarps + 1] = pp.best_in; s_red[kWarps + 2] = pp.stall_in;
    }
    __syncthreads();
    uint32_t barriers = 0;                             // grid barriers passed: two per round with a winner
    for (uint32_t t = 0; t < rounds; ++t) {
        const uint32_t round = first_round + t;
        // the base's own evaluation and totals: a full pass in the first round; afterwards the totals are patched and
        // the evaluation IS the previous winner's key (unless that key was saturated)
        if (t == 0 || s_base[2] == 0) {
            block_eval<W, kRF>(d, &s_cs, d.bitsT, d.leader, s_cnt, s_lcnt, s_rc, s_acc, rftab);
            if constexpr (kTopics) {
                if (tid == 0) s_acc[0] += __ldcg(ta.tviol);
            }
            if (tid == 0) { s_base[0] = (int)min(s_acc[0], (long long)0x7FFFFFFF); s_base[1] = (int)s_acc[1]; }
            __syncthreads();
        }
        unsigned long long best = kKeyNone;
        {
            const Gen<W, true, true> tg = large_gen<W>(d, la, &s_cs, s_st);
            const MemRef<false> m_obj(d.swT);
            const int base_viol = s_base[0], base_obj = s_base[1];
            for (uint32_t idx = pp.idx_lo + blockIdx.x * kLT + tid; idx < pp.idx_hi; idx += gridDim.x * kLT) {
                PatchSet ps;
                uint32_t rows[kMaxOps][W];
                tg.run(seed, round, idx, round_size, ps, rows);
                int viol, obj;
                delta_eval<LargeCfg<W>, false, kRF>(d, d.bitsT, d.leader, m_obj, &s_cs, ps, rows, s_cnt, s_lcnt, s_rc,
                                                    base_viol, base_obj, viol, obj, rftab);
                if constexpr (kTopics) {
                    int rc[2 * kMaxOps], lc[2 * kMaxOps];
                    topic_events<W>(d, ta, &s_cs, ps, rows, rc, lc);
                    viol += topic_delta<W>(ta, rc, lc);
                }
                const unsigned long long key = pack_key(viol, obj, idx, d.key_obj_bits);
                if (all_keys) all_keys[idx - pp.idx_lo] = key;
                best = key < best ? key : best;
            }
        }
        if (all_keys) return;                                       // key dump only: the base stays as it is
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long w = __shfl_xor_sync(0xFFFFFFFFu, best, o);
            best = w < best ? w : best;
        }
        if (lane == 0) s_red[warp] = best;
        __syncthreads();
        if (warp == 0) {
            unsigned long long v = lane < kWarps ? s_red[lane] : kKeyNone;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const unsigned long long w = __shfl_xor_sync(0xFFFFFFFFu, v, o);
                v = w < v ? w : v;
            }
            if (lane == 0) {
                if (v != kKeyNone) atomicMin(keys + t, v);
                // grid barrier 1: every CTA's contribution to keys[t] is visible before anyone reads it
                __threadfence();
                atomicAdd(grid_bar, 1u);
                if (!spin_until(grid_bar, (barriers + 1) * gridDim.x, pp.abort, pp.timeout_ns)) s_abort = 1;
                __threadfence();
            }
        }
        ++barriers;
        __syncthreads();
        if (s_abort) return;
        const unsigned long long k = __ldcg(keys + t);
        if (tid == 0) {
            // early stop (the same decision in every CTA: it only depends on the keys)
            const unsigned long long vc = k >> kIdxBits;
            if (vc < s_red[kWarps + 1]) { s_red[kWarps + 1] = vc; s_red[kWarps + 2] = 0; } else ++s_red[kWarps + 2];
            if (pp.patience && s_red[kWarps + 2] >= pp.patience) s_red[kWarps] = 1;
            if (blockIdx.x == 0 && pp.rounds_run) *pp.rounds_run = t + 1;
            if (blockIdx.x == 0 && pp.carry) { pp.carry[0] = s_red[kWarps + 1]; pp.carry[1] = s_red[kWarps + 2]; }
            const uint32_t kv = key_violation(k, d.key_obj_bits);
            s_base[2] = (k != kKeyNone && (uint64_t)kv < key_viol_cap(d.key_obj_bits)) ? 1 : 0;
            s_base[0] = (int)kv;
            s_base[1] = (int)key_objective(k, d.key_obj_bits);
        }
        if (k == kKeyNone) {
            __syncthreads();
            if (s_red[kWarps]) break;
            continue;
        }
        if (blockIdx.x == 0) apply_winner_large<W>(d, la, &s_cs, s_st, seed, round, round_size, k, s_rec, s_lc);
        if constexpr (kTopics) {
            if (blockIdx.x == 0 && tid == 0) apply_winner_topics<W>(ta, &s_cs, d.B, s_rec);
        }
        // grid barrier 2: the patched HBM state and the winner record are visible before anyone reads them
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            atomicAdd(grid_bar, 1u);
            if (!spin_until(grid_bar, (barriers + 1) * gridDim.x, pp.abort, pp.timeout_ns)) s_abort = 1;
            __threadfence();
        }
        ++barriers;
        __syncthreads();
        if (s_abort) return;
        if (tid == 0) {
            // every CTA patches its totals from the record: the old rows out, the new rows in
            const int n = __ldcg(&la.rec->n);
            for (int i = 0; i < n; ++i) {
                for (int t2 = 0; t2 < W; ++t2) {
                    for (uint32_t m = __ldcg(&la.rec->old_row[i][t2]); m; m &= m - 1) {
                        const int s = 32 * t2 + __ffs(m) - 1;
                        --s_cnt[s]; --s_rc[s >> d.log2S];
                    }
                    for (uint32_t m = __ldcg(&la.rec->new_row[i][t2]); m; m &= m - 1) {
                        const int s = 32 * t2 + __ffs(m) - 1;
                        ++s_cnt[s]; ++s_rc[s >> d.log2S];
                    }
                }
                const int lo = (int)__ldcg(&la.rec->old_ld[i]), ln = (int)__ldcg(&la.rec->new_ld[i]);
                if (lo < NSL && ((__ldcg(&la.rec->old_row[i][lo >> 5]) >> (lo & 31)) & 1u)) --s_lcnt[lo];
                if (ln < NSL && ((__ldcg(&la.rec->new_row[i][ln >> 5]) >> (ln & 31)) & 1u)) ++s_lcnt[ln];
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) s_st[j] = __ldcg(&la.rec->state[j]);
        }
        __syncthreads();
        if (s_red[kWarps]) break;
    }
}

// a topic session's counts: one 32-bit atomic on the word that holds the u16 cell (a cell never exceeds 65,280)
template <int W>
__global__ void topic_count_kernel(Params d, TopicArgs ta)
{
    constexpr int NSL = 32 * W;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < d.P; p += gridDim.x * blockDim.x) {
        const int t = ta.topic_of[p], ld = d.leader[p];
        uint32_t x[W];
#pragma unroll
        for (int w = 0; w < W; ++w) x[w] = d.bitsT[(size_t)w * d.Ppad + p];
        auto bump = [&](uint16_t *c, int s) {
            const size_t i = (size_t)t * NSL + s;
            atomicAdd(reinterpret_cast<unsigned int *>(c + (i & ~(size_t)1)), 1u << (16 * (i & 1)));
        };
#pragma unroll
        for (int w = 0; w < W; ++w)
            for (uint32_t m = x[w]; m; m &= m - 1) {
                const int s = 32 * w + __ffs(m) - 1;
                if (broker_slot(d.consts, d.B, s)) bump(ta.tcnt, s);
            }
        if (ld < NSL && row_has<W>(x, ld) && broker_slot(d.consts, d.B, ld)) bump(ta.tlcnt, ld);
    }
}

// the topic-row violation of the base: every (topic, broker slot) cell once
template <int W>
__global__ void topic_violation_kernel(Params d, TopicArgs ta)
{
    constexpr int NSL = 32 * W;
    __shared__ int s_v;
    if (threadIdx.x == 0) s_v = 0;
    __syncthreads();
    int v = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)ta.T * NSL; i += (size_t)gridDim.x * blockDim.x) {
        const int s = (int)(i & (NSL - 1));
        if (!broker_slot(d.consts, d.B, s)) continue;
        const int4 b = ta.bnd[i / NSL];
        v += band_int(ta.tcnt[i], b.x, b.y) + band_int(ta.tlcnt[i], b.z, b.w);
    }
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(&s_v, v);
    __syncthreads();
    if (threadIdx.x == 0 && s_v) atomicAdd(ta.tviol, s_v);
}

// the transposed planes of the base (every word, the padding words of t_words included)
template <int W>
__global__ void large_t_kernel(const uint32_t *bits, const uint8_t *leader, int Ppad, uint32_t *T, int nW)
{
    constexpr int NSL = 32 * W;
    const int total = kTPlanes * NSL * nW;
    for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < total; o += gridDim.x * blockDim.x) {
        const int w = o % nW, s = (o / nW) % NSL, q = o / (nW * NSL);
        T[t_word(q, s, w, nW, NSL)] = t_gather<W>(q, s, w, bits, leader, Ppad);
    }
}

// the displaced lists into buffer 0, and the number of partitions led from a slot they do not hold
template <int W>
__global__ void __launch_bounds__(1024, 1) large_lists_kernel(Params d)
{
    __shared__ int s_scan[72];
    __shared__ int s_bad;
    rebuild_lists<W, 1024>(d.bitsT, d.leader, d.homeT, d.P, d.Ppad, d.D, d.DL, d.nD, s_scan);
    if (threadIdx.x == 0) s_bad = 0;
    __syncthreads();
    int bad = 0;
    for (int p = threadIdx.x; p < d.P; p += 1024) {
        const int ld = d.leader[p];
        bad += (ld < 32 * W && ((d.bitsT[(size_t)(ld >> 5) * d.Ppad + p] >> (ld & 31)) & 1u)) ? 0 : 1;
    }
    if (bad) atomicAdd(&s_bad, bad);
    __syncthreads();
    if (threadIdx.x == 0) { d.nD[2] = s_bad; d.nD[3] = 0; }
}

template <int W>
__global__ void __launch_bounds__(kLT, 1)
eval_large_kernel(Params d, const uint32_t *bits, const uint8_t *leader, long long *viol, long long *obj)
{
    __shared__ Consts s_cs;
    __shared__ int s_cnt[256], s_lcnt[256], s_rc[32];
    __shared__ long long s_acc[2];
    load_consts(&s_cs, d.consts);
    __syncthreads();
    const size_t a = blockIdx.x;
    block_eval<W>(d, &s_cs, bits + a * W * d.Ppad, leader + a * d.Ppad, s_cnt, s_lcnt, s_rc, s_acc);
    if (threadIdx.x == 0) { viol[a] = s_acc[0]; obj[a] = s_acc[1]; }
}

// the base of a topic or replication session: the evaluation above, with every row's own C1 / C7 operands (kRF), plus
// the topic-row violation kept current with the base when the session has topic rows (ta.tviol != nullptr)
template <int W, bool kRF>
__global__ void __launch_bounds__(kLT, 1)
eval_large_base_kernel(Params d, TopicArgs ta, const uint32_t *rftab, long long *viol, long long *obj)
{
    __shared__ Consts s_cs;
    __shared__ int s_cnt[256], s_lcnt[256], s_rc[32];
    __shared__ long long s_acc[2];
    load_consts(&s_cs, d.consts);
    __syncthreads();
    block_eval<W, kRF>(d, &s_cs, d.bitsT, d.leader, s_cnt, s_lcnt, s_rc, s_acc, rftab);
    if (threadIdx.x == 0) { *viol = s_acc[0] + (ta.tviol ? __ldcg(ta.tviol) : 0); *obj = s_acc[1]; }
}

template <class F> cudaError_t with_w(int W, F &&f)
{
    switch (W) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    default: return f(std::integral_constant<int, 8>{});
    }
}

}  // namespace

cudaError_t large_prepare(int W, const Params &d, const LargeArgs &la, cudaStream_t st)
{
    return with_w(W, [&](auto w) {
        constexpr int kW = decltype(w)::value;
        large_t_kernel<kW><<<264, 256, 0, st>>>(d.bitsT, d.leader, d.Ppad, la.T, la.tnW);
        large_lists_kernel<kW><<<1, 1024, 0, st>>>(d);
        return cudaGetLastError();
    });
}

cudaError_t topics_prepare(int W, const Params &d, const TopicArgs &ta, cudaStream_t st)
{
    const size_t cells = (size_t)ta.T * 32 * W;
    cudaError_t e = cudaMemsetAsync(ta.tcnt, 0, cells * 2, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(ta.tlcnt, 0, cells * 2, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(ta.tviol, 0, sizeof(int), st);
    if (e != cudaSuccess) return e;
    return with_w(W, [&](auto w) {
        constexpr int kW = decltype(w)::value;
        topic_count_kernel<kW><<<264, 256, 0, st>>>(d, ta);
        topic_violation_kernel<kW><<<528, 256, 0, st>>>(d, ta);
        return cudaGetLastError();
    });
}

cudaError_t large_search(int W, int grid, const Params &d, const LargeArgs &la, uint64_t seed, uint32_t first_round,
                         uint32_t rounds, uint32_t round_size, unsigned long long *keys, unsigned int *grid_bar,
                         const P2P &pp, unsigned long long *all_keys, cudaStream_t st, const TopicArgs *ta,
                         const uint32_t *rftab)
{
    Params prm = d;
    LargeArgs a = la;
    P2P p2 = pp;
    TopicArgs t = ta ? *ta : TopicArgs{};
    const uint32_t *rt = rftab;
    void *args[] = {&prm, &a, &seed, &first_round, &rounds, &round_size, &keys, &grid_bar, &p2, &all_keys, &t, &rt};
    return with_w(W, [&](auto w) {
        constexpr int kW = decltype(w)::value;
        // cooperative launch: all CTAs are co-resident, which the grid barriers need
        const void *kern = rftab ? (ta ? reinterpret_cast<const void *>(search_large_kernel<kW, true, true>)
                                       : reinterpret_cast<const void *>(search_large_kernel<kW, false, true>))
                                 : (ta ? reinterpret_cast<const void *>(search_large_kernel<kW, true, false>)
                                       : reinterpret_cast<const void *>(search_large_kernel<kW, false, false>));
        return cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kLT), args, 0, st);
    });
}

cudaError_t large_eval_base(int W, const Params &d, const TopicArgs *ta, const uint32_t *rftab, long long *viol,
                            long long *obj, cudaStream_t st)
{
    const TopicArgs t = ta ? *ta : TopicArgs{};
    return with_w(W, [&](auto w) {
        constexpr int kW = decltype(w)::value;
        if (rftab) eval_large_base_kernel<kW, true><<<1, kLT, 0, st>>>(d, t, rftab, viol, obj);
        else eval_large_base_kernel<kW, false><<<1, kLT, 0, st>>>(d, t, rftab, viol, obj);
        return cudaGetLastError();
    });
}

cudaError_t large_eval(int W, const Params &d, const uint32_t *bits, const uint8_t *leader, int n, long long *viol,
                       long long *obj, cudaStream_t st)
{
    if (n <= 0) return cudaSuccess;
    return with_w(W, [&](auto w) {
        eval_large_kernel<decltype(w)::value><<<n, kLT, 0, st>>>(d, bits, leader, viol, obj);
        return cudaGetLastError();
    });
}
