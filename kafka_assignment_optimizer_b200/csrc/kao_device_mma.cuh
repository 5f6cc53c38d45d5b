// kao_device_mma.cuh — the column-major evaluator with its sums on the tensor cores (schedule pop 0x300,
// kao_device_t.cuh: EvalCfgT).
//
// Every sum the column-major evaluator forms is a count of partitions p that hold in a base plane AND are scored
// for the candidate.  For the 32 candidates c of a warp's batch these counts are one binary matrix product
//     D[r][c] = sum_p  plane_r[p] AND valid_c[p]          (mma.sync.m16n8k256 .b1 .and.popc, SASS BMMA.168256.AND.POPC)
// with valid_c[p] = "partition p is not patched by candidate c".  The rows r of the base (A operand, ldmatrix from
// shared memory) are
//     T0[s]  replicas on slot s             T1[s]  valid leaders on slot s        (2 x 32 W rows, kao_device_t.cuh)
//     Z[j]   term plane j of the objective  A[b]   rack field b in use            (8 + 4 W rows)
//     S[k]   bit k of max(0, RF - n_p): how far row p falls short of RF           (kSPlanes rows)
// and the candidates' masks are the B operand, built in registers from the patched partitions.  Every sum of every
// candidate is formed from the planes with that candidate's own mask (docs/MODEL.md §3.3); the patched rows are
// scored from the patch itself by the thread that generated the candidate (patch_terms, mma_park_patch).
//
// The rows: with "at most one replica per rack" a row of n replicas in z racks costs |n - RF| + (n - z)
// = 2 n - z - RF + 2 max(0, RF - n), exactly, for every row.  So over the unpatched rows
//     C1 + C7 = 2 sum_s D[T0 s] - sum_b D[A b] - RF * #unpatched + 2 sum_k 2^k D[S k]
// and the objective is sum_j z_value[j] D[Z j].  The columns: c_s = D[T0 s] + new_s, l_s = D[T1 s] + newl_s, with
// new_s / newl_s what the candidate's patched rows put on slot s; C3 / C4 per slot, C6 over the 8 slots of a rack,
// C2 / C5 as P - sum_s l_s.
#pragma once
#include "kao_plan.hpp"

namespace kao {

constexpr int kSPlanes = 4;          // max(0, RF - n) < 16 (RF < 16: rf_mask holds four bit slices)

// ------------------------------------------------------------------------------------------
// PTX: ldmatrix of four 8 x 16-byte matrices and the binary MMA.  A fragment (m16 x k256, row):
// a0 = row g, 32-bit word t of the k-step; a1 = row g + 8, word t; a2 / a3 = the same rows, word t + 4.
// B fragment (k256 x n8, col): b0 = column g, word t; b1 = column g, word t + 4.  D: d0 / d1 = row g, columns 2 t,
// 2 t + 1; d2 / d3 = row g + 8.  (g = lane / 4, t = lane % 4.)  tests/emu/mma_emu.hpp restates both.
// ------------------------------------------------------------------------------------------
#if !defined(KAO_HOST_EMU)
__device__ __forceinline__ void ldsm_x4(const uint32_t *row, uint32_t (&a)[4])
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]) : "r"((uint32_t)__cvta_generic_to_shared(row)));
}
__device__ __forceinline__ void bmma_and_popc(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
#else
inline void ldsm_x4(const uint32_t *row, uint32_t (&a)[4]) { emu_ldsm_x4(row, a); }
inline void bmma_and_popc(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) { emu_bmma_and_popc(c, a, b0, b1); }
#endif

// ------------------------------------------------------------------------------------------
// 16 x 2 SIMD for the packed epilogue: per-halfword unsigned max / min, SASS VIMNMX.U16x2,
// one instruction for two candidates.  The host build (test emulation) restates the CUDA semantics: each halfword of
// the result is the max / min of the operands' halfwords, no carry or borrow between the halves.
// ------------------------------------------------------------------------------------------
#if !defined(KAO_HOST_EMU)
__device__ __forceinline__ uint32_t vmax16x2(uint32_t a, uint32_t b) { return __vmaxu2(a, b); }
__device__ __forceinline__ uint32_t vmin16x2(uint32_t a, uint32_t b) { return __vminu2(a, b); }
#else
inline uint32_t vmax16x2(uint32_t a, uint32_t b)
{
    const uint32_t al = a & 0xFFFFu, bl = b & 0xFFFFu, ah = a >> 16, bh = b >> 16;
    return (al > bl ? al : bl) | (ah > bh ? ah : bh) << 16;
}
inline uint32_t vmin16x2(uint32_t a, uint32_t b)
{
    const uint32_t al = a & 0xFFFFu, bl = b & 0xFFFFu, ah = a >> 16, bh = b >> 16;
    return (al < bl ? al : bl) | (ah < bh ? ah : bh) << 16;
}
#endif
// a slot's bounds lo | hi << 16 clamped to P (PP = P | P << 16): lo' and hi' each in both halves
__device__ __forceinline__ void bounds16x2(uint32_t b, uint32_t PP, uint32_t &lo2, uint32_t &hi2)
{
    const uint32_t bc = vmin16x2(b, PP);
    lo2 = __byte_perm(bc, 0u, 0x1010);
    hi2 = __byte_perm(bc, 0u, 0x3232);
}
// what the clamp leaves to a per-launch constant: max(lo - P, 0) - min(hi, P)
__device__ __forceinline__ int bounds16x2_rest(uint32_t b, uint32_t PP)
{
    const uint32_t bc = vmin16x2(b, PP);
    return (int)((b - bc) & 0xFFFFu) - (int)(bc >> 16);
}

// one word (32 partitions) of shortfall plane k: bit k of max(0, RF - replicas of the row), 0 beyond P
template <int W>
__device__ __forceinline__ uint32_t s_gather(const Params &d, int k, int w, const uint32_t *bitsT)
{
    uint32_t out = 0;
    for (int b = 0; b < 32; ++b) {
        const int p = 32 * w + b;
        if (p >= d.P) break;
        int n = 0;
        for (int t = 0; t < W; ++t) n += __popc(bitsT[(size_t)t * d.Ppad + p]);
        out |= (uint32_t)((max(d.RF - n, 0) >> k) & 1) << b;
    }
    return out;
}

// ------------------------------------------------------------------------------------------
// The warp's batch (per warp, 32 * batch_stride_words(W) words, kao_plan.hpp): 32 headers of 4 words — (patched
// partition 0 | 1 << 16), (partition 2 | patched partitions << 16), the C1 / C7 terms and the objective terms of the
// patched rows; 0xFFFF = no patch — then one 32-byte row per slot: byte mma_byte_pos(c) of row s = replicas (low
// nibble) and valid leaderships (high nibble) that candidate c's patched rows put on slot s.  A lane of the MMA
// epilogue holds candidates 8 nt + 2 t + jj (nt = 0..3, jj = 0, 1): they are the 8 bytes at 8 t of the row.
// ------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int mma_byte_pos(int c) { return ((c >> 1) & 3) * 8 + (c >> 3) * 2 + (c & 1); }

// the whole warp clears the slot rows of its batch (before the lanes park their candidates)
template <int W>
__device__ __forceinline__ void mma_clear_batch(uint32_t *batch, int lane)
{
    uint4 *rows = reinterpret_cast<uint4 *>(batch + 32 * kBatchHdr);
#pragma unroll
    for (int i = 0; i < 2 * W; ++i) rows[i * 32 + lane] = make_uint4(0u, 0u, 0u, 0u);
}

// lane c parks its candidate (ps, rows: the generator's patch; pviol / pobj: patch_terms)
template <int W>
__device__ __forceinline__ void mma_park_patch(const PatchSet &ps, const uint32_t (&rows)[kMaxOps][W], int pviol, int pobj,
                                               uint32_t *batch, int lane)
{
    const int p0 = ps.p[0], p1 = ps.p[1], p2 = ps.p[2];
    const int npatched = (p0 >= 0) + (p1 >= 0 && p1 != p0) + (p2 >= 0 && p2 != p0 && p2 != p1);     // rows the masks take out
    uint32_t *mine = batch + lane * kBatchHdr;
    mine[0] = ((uint32_t)p0 & 0xFFFFu) | ((uint32_t)p1 << 16);
    mine[1] = ((uint32_t)p2 & 0xFFFFu) | ((uint32_t)npatched << 16);
    mine[2] = (uint32_t)pviol;
    mine[3] = (uint32_t)pobj;
    uint8_t *col = reinterpret_cast<uint8_t *>(batch + 32 * kBatchHdr) + mma_byte_pos(lane);
#pragma unroll
    for (int i = 0; i < kMaxOps; ++i) {
        if (ps.p[i] < 0) continue;
#pragma unroll
        for (int t = 0; t < W; ++t)
            for (uint32_t m = rows[i][t]; m; m &= m - 1) {
                const int s = 32 * t + __ffs(m) - 1;
                col[32 * s] = (uint8_t)(col[32 * s] + 1);
            }
        const int ld = (int)ps.ld[i];
        if (ld < 32 * W && row_has<W>(rows[i], ld)) col[32 * ld] = (uint8_t)(col[32 * ld] + 0x10);
    }
}

// Sum over the 8 lane groups (lanes with the same t) of 8 values per lane, scattered: afterwards lane (g, t) holds
// the total of value g.  7 shuffles instead of 24.
__device__ __forceinline__ int reduce_scatter8(int (&v)[8], int lane)
{
    const bool h4 = (lane >> 4) & 1, h2 = (lane >> 3) & 1, h1 = (lane >> 2) & 1;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int send = h4 ? v[i] : v[i + 4], keep = h4 ? v[i + 4] : v[i];
        v[i] = keep + (int)__shfl_xor_sync(0xFFFFFFFFu, (uint32_t)send, 16);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int send = h2 ? v[i] : v[i + 2], keep = h2 ? v[i + 2] : v[i];
        v[i] = keep + (int)__shfl_xor_sync(0xFFFFFFFFu, (uint32_t)send, 8);
    }
    const int send = h1 ? v[0] : v[1], keep = h1 ? v[1] : v[0];
    return keep + (int)__shfl_xor_sync(0xFFFFFFFFu, (uint32_t)send, 4);
}

// ------------------------------------------------------------------------------------------
// Sorted batches.  The 32 lanes of a batch run the union of their candidates'
// generator bodies, and every branch of that union is chosen by the candidate's control word (docs/MODEL.md §5),
// which depends on (seed, round, index) alone, not on the base.  So a CTA sorts its candidates of a round by the
// class below before the round starts, and a batch takes 32 neighbours of that order: mostly one body.  The class:
// 0 the identity candidate; in a cycle round 1 + the two role-match bits (every other choice is fixed there); else
// operations << 6 | first-operation LEADER << 5 | guided << 4 | link kind of operation 2 << 2 | of operation 3
// (link kinds of operations a candidate does not have are 0).  Below kCandClasses (kao_plan.hpp).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cand_class(uint64_t seed, uint32_t round, uint32_t idx, uint32_t round_size)
{
    if (idx + 1 == round_size) return 0;
    uint32_t r[4];
    philox4x32_10(idx, round, 0u, kTag, (uint32_t)seed, (uint32_t)(seed >> 32), r);
    const uint32_t ctl = r[0];
    if ((round & 3u) == 3u) return 1u + ((ctl >> 11) & 1u) * 2u + ((ctl >> 13) & 1u);
    const uint32_t nops = (ctl & 3u) == 0 ? 1u : ((ctl & 3u) == 3 ? 3u : 2u);
    return nops << 6 | ((ctl >> 2) & 3u) << 4 | (nops >= 2 ? ((ctl >> 4) & 3u) << 2 : 0u) | (nops == 3 ? (ctl >> 7) & 3u : 0u);
}
// candidate index at position k of a CTA's share of a round: warp k % warps, iteration k / warps
__host__ __device__ __forceinline__ uint32_t cand_at(uint32_t k, uint32_t first, uint32_t stride, uint32_t warps)
{
    return first + k % warps + k / warps * stride;
}
// how many of the positions 0, 1, ... of a CTA's share lie below idx_hi (indices rise with the position)
__host__ __device__ __forceinline__ uint32_t cand_count(uint32_t first, uint32_t stride, uint32_t warps, uint32_t idx_hi)
{
    if (first >= idx_hi) return 0;
    const uint32_t full = (idx_hi - first) / stride, rem = (idx_hi - first) % stride;
    return full * warps + (rem < warps ? rem : warps);
}

// ------------------------------------------------------------------------------------------
// The batch of 32 candidates.  T: the transposed planes; Z: term, rack-field and shortfall planes ([kZPlanes + 4 W +
// kSPlanes][nW]); batch: the warp's parked candidates.  Returns, in lane (g, t), candidate mma_lane_candidate(lane):
// its violation and objective.
// ------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int mma_lane_candidate(int lane) { return ((lane >> 3) & 3) * 8 + 2 * (lane & 3) + ((lane >> 2) & 1); }

template <class Cfg>
__device__ __forceinline__ void eval_batch_mma(const Params &d, const Consts *cs, const uint32_t *T, int nW_rt, const uint32_t *Z,
                                               const uint32_t *batch, int lane, int &viol_out, int &obj_out)
{
    constexpr int W = Cfg::W, kNW = Cfg::kNW, NSL = 32 * W;
    const int nW = kNW ? kNW : nW_rt;
    const int g = lane >> 2, t = lane & 3;
    // ---- B fragments: the masks of candidates 8 nt + g; words t and t + 4 of every k-step of 8 words
    int pw[4][kMaxOps];
    uint32_t pm[4][kMaxOps];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        const uint2 h = *reinterpret_cast<const uint2 *>(batch + (nt * 8 + g) * kBatchHdr);
        const int p[kMaxOps] = {(int)(int16_t)(h.x & 0xFFFFu), (int)(int16_t)(h.x >> 16), (int)(int16_t)(h.y & 0xFFFFu)};
#pragma unroll
        for (int i = 0; i < kMaxOps; ++i) { pw[nt][i] = p[i] >> 5; pm[nt][i] = ~(1u << (p[i] & 31)); }    // -1 >> 5 is never a word
    }
    auto mask = [&](int nt, int w) {
        uint32_t b = ~0u;
#pragma unroll
        for (int i = 0; i < kMaxOps; ++i) b &= pw[nt][i] == w ? pm[nt][i] : ~0u;
        return b;
    };
    constexpr int kKS = kNW ? kNW / 8 : 1;          // k-steps whose masks stay in registers (compile-time word count)
    uint32_t bf[kKS][4][2];
    if constexpr (kNW != 0) {
#pragma unroll
        for (int ks = 0; ks < kKS; ++ks)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) { bf[ks][nt][0] = mask(nt, 8 * ks + t); bf[ks][nt][1] = mask(nt, 8 * ks + t + 4); }
    }
    // ---- one m-tile: 16 rows of the base against the 32 masks.  row: this lane's ldmatrix row (word 0 of the plane
    // row), sx: its swizzle (words XORed into the word index, kao_device.cuh t_word)
    const int lrow = (lane & 7) + ((lane >> 3) & 1) * 8, khalf = 4 * (lane >> 4);
    int acc[4][4];
    auto tile = [&](const uint32_t *row, int sx) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[nt][i] = 0;
        if constexpr (kNW != 0) {
#pragma unroll
            for (int ks = 0; ks < kKS; ++ks) {
                uint32_t a[4];
                ldsm_x4(row + ((8 * ks + khalf) ^ sx), a);
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) bmma_and_popc(acc[nt], a, bf[ks][nt][0], bf[ks][nt][1]);
            }
        } else {
#pragma unroll 1
            for (int ks = 0; ks < nW / 8; ++ks) {
                uint32_t a[4];
                ldsm_x4(row + ((8 * ks + khalf) ^ sx), a);
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) bmma_and_popc(acc[nt], a, mask(nt, 8 * ks + t), mask(nt, 8 * ks + t + 4));
            }
        }
    };
    const bool swz = t_swizzled(nW);
    const uint8_t *cols = reinterpret_cast<const uint8_t *>(batch + 32 * kBatchHdr) + 8 * t;
    // per-lane partial sums of candidates 8 nt + 2 t + jj at [2 nt + jj]; rack terms of candidates 8 (g & 3) + 2 t + jj
    int v[8], o[8], rpen[2] = {0, 0};
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = o[e] = 0;
    // Packed epilogue: d0 / d1 of a lane are candidates 2 t and 2 t + 1 of one slot row, so the pair
    // travels as one register x = x0 | x1 << 16 (PRMT) and its delta bytes are spread into the two halves.  Every
    // column total is 0 <= c <= P <= 8,160, and with the bounds clamped to lo' = min(lo, P), hi' = min(hi, P)
    //     max(c - hi, 0) + max(lo - c, 0) = max(c, hi') + max(c, lo') - c  - hi' + (lo - lo')        (c <= P)
    // so a slot costs two VIMNMX.U16x2 per pair, and - hi' + (lo - lo') summed over the slots is one constant of the
    // launch, added at the end (one warp reduction per batch).
    // The pair sums r = lo + hi << 16 of an m-tile are plain 32-bit adds: each half's total stays in 0 .. 65,535 (bounds
    // at the loops), so no carry crosses the halves.  They widen once per m-tile: v[2 nt] sums r and v[2 nt + 1] sums
    // r >> 16 (one IADD, one LEA.HI); after the last m-tile v[2 nt] - (v[2 nt + 1] << 16) is the sum of the low halves,
    // exact mod 2^32, and that sum is far below 2^31.
    const uint32_t PP = (uint32_t)d.P * 0x10001u;
    auto widen = [&](const uint32_t (&r)[4]) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) { v[2 * nt] = (int)((uint32_t)v[2 * nt] + r[nt]); v[2 * nt + 1] += (int)(r[nt] >> 16); }
    };
    auto pair = [&](int nt, int h) { return __byte_perm((uint32_t)acc[nt][2 * h], (uint32_t)acc[nt][2 * h + 1], 0x5410); };
    // delta nibbles (masked to the low nibble of each byte) of candidates 8 nt + 2 t, + 1: bytes 2 nt, 2 nt + 1 of the row
    auto spread = [](uint32_t nx, uint32_t ny, int nt) { return __byte_perm(nt < 2 ? nx : ny, 0u, (nt & 1) ? 0x4342 : 0x4140); };
    // ---- replicas: 2 D (rows), C3, and the rack totals (C6)
#pragma unroll 1
    for (int mt = 0; mt < 2 * W; ++mt) {
        const int s = 16 * mt + lrow;
        tile(T + (size_t)(0 * NSL + s) * nW, swz ? 4 * (s & 7) : 0);
        int rk[8];
        // per half and slot: 2 D + the C3 terms = max(c, hi') + max(c, lo') + D - delta, in 2 D .. 3 P; two slots
        // <= 6 P = 48,960
        uint32_t r[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int sl = 16 * mt + 8 * h + g;
            uint32_t lo2, hi2;
            bounds16x2(cs->bnd_rep[sl], PP, lo2, hi2);
            const uint2 nb = *reinterpret_cast<const uint2 *>(cols + 32 * sl);
            const uint32_t nx = nb.x & 0x0F0F0F0Fu, ny = nb.y & 0x0F0F0F0Fu;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const uint32_t d2 = pair(nt, h), n2 = spread(nx, ny, nt), c2 = d2 + n2;
                r[nt] += vmax16x2(c2, hi2) + vmax16x2(c2, lo2) + d2 - n2;
                rk[4 * h + nt] = (int)c2;                       // c <= P < 8192: a rack's 8 slots stay below 2^16
            }
        }
        widen(r);
        // rack totals: the 8 slots of a rack are the 8 lane groups; lane (g, t) gets rack 2 mt + (g >> 2) of candidates
        // 8 (g & 3) + 2 t + jj
        const int pk = reduce_scatter8(rk, lane);
        const int rack = 2 * mt + (g >> 2);
        const int lo = rack < d.R ? cs->rack_lo[rack] : 0, hi = rack < d.R ? cs->rack_hi[rack] : 0x7FFFFFFF;
        const int t0 = pk & 0xFFFF, t1 = (int)((uint32_t)pk >> 16);
        rpen[0] += max(t0 - hi, 0) + max(lo - t0, 0);
        rpen[1] += max(t1 - hi, 0) + max(lo - t1, 0);
    }
    // ---- valid leaders: C4 and - l (C2 / C5 = P - sum of the valid leaders)
#pragma unroll 1
    for (int mt = 0; mt < 2 * W; ++mt) {
        const int s = 16 * mt + lrow;
        tile(T + (size_t)(1 * NSL + s) * nW, swz ? 4 * (s & 7) : 0);
        // per half and slot: the C4 terms - l = max(l, hi') + max(l, lo') - 2 l, in 0 .. 2 P; two slots <= 4 P = 32,640
        uint32_t m[4] = {0u, 0u, 0u, 0u}, ls[4] = {0u, 0u, 0u, 0u}, r[4];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int sl = 16 * mt + 8 * h + g;
            uint32_t lo2, hi2;
            bounds16x2(cs->bnd_ldr[sl], PP, lo2, hi2);
            const uint2 nb = *reinterpret_cast<const uint2 *>(cols + 32 * sl);
            const uint32_t nx = (nb.x >> 4) & 0x0F0F0F0Fu, ny = (nb.y >> 4) & 0x0F0F0F0Fu;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const uint32_t l2 = pair(nt, h) + spread(nx, ny, nt);
                m[nt] += vmax16x2(l2, hi2) + vmax16x2(l2, lo2);
                ls[nt] += l2;
            }
        }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) r[nt] = m[nt] - 2u * ls[nt];
        widen(r);
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) v[2 * nt] = (int)((uint32_t)v[2 * nt] - ((uint32_t)v[2 * nt + 1] << 16));
    // ---- term planes (objective), rack-field planes (- z) and shortfall planes (+ 2 * 2^k): rows Z[0..8 + 4 W + 4),
    // one tile at W = 1, two at W = 2 (the second one's rows beyond the shortfall planes repeat them and weigh nothing)
    constexpr int kZRows = kZPlanes + 4 * W + kSPlanes;
#pragma unroll
    for (int zt = 0; zt < (kZRows + 15) / 16; ++zt) {
        const int r = 16 * zt + lrow;
        tile(Z + (size_t)(r < kZRows ? r : kZRows - kSPlanes + (r & 3)) * nW, 0);
        auto weight = [&](int row, int &wv, int &wo) {             // what row `row` of the Z area weighs
            wv = 0; wo = 0;
            if (row < kZPlanes) wo = row < d.nz ? d.z_value[row] : 0;
            else if (row < kZPlanes + 4 * W) wv = -1;
            else if (row < kZRows) wv = 2 << (row - kZPlanes - 4 * W);
        };
        int wv0, wo0, wv1, wo1;
        weight(16 * zt + g, wv0, wo0);
        weight(16 * zt + 8 + g, wv1, wo1);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int jj = 0; jj < 2; ++jj) {
                v[2 * nt + jj] += wv0 * acc[nt][jj] + wv1 * acc[nt][2 + jj];
                o[2 * nt + jj] += wo0 * acc[nt][jj] + wo1 * acc[nt][2 + jj];
            }
    }
    // ---- the rack terms join their candidates' sums; per-candidate totals; the patched rows' own terms
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] += (e >> 1) == (g & 3) ? rpen[e & 1] : 0;
    const int viol = reduce_scatter8(v, lane), obj = reduce_scatter8(o, lane);
    const uint4 h = *reinterpret_cast<const uint4 *>(batch + mma_lane_candidate(lane) * kBatchHdr);
    viol_out = viol + (int)h.z + d.P - d.RF * (d.P - (int)(h.y >> 16));
    obj_out = obj + (int)h.w;
    int k = 0;                                                      // the clamp's constant, over every slot of both tables
#pragma unroll
    for (int sl = lane; sl < NSL; sl += 32) k += bounds16x2_rest(cs->bnd_rep[sl], PP) + bounds16x2_rest(cs->bnd_ldr[sl], PP);
    viol_out += __reduce_add_sync(0xFFFFFFFFu, k);
}

}  // namespace kao
