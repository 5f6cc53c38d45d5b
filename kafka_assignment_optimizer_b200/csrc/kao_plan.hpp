// kao_plan.hpp — shared-memory plan of the search kernels: which table sits where in the dynamic
// shared memory of a CTA.  Host-only arithmetic, shared by the kernels (kao_kernels.cuh), the engine
// (kao_engine.cu: does the mask-plane layout fit, else packed entries) and the host-side emulation
// harness of the device functions (tests/emu).
#pragma once
#include "kao_device.cuh"
#include "kao_device_t.cuh"

#include <cstdint>

using namespace kao;

// ------------------------------------------------------------------------------------------
// shared-memory plan of the search kernel
// ------------------------------------------------------------------------------------------
struct SmemPlan {
    uint32_t off_bits, off_sw, off_z, off_leader, off_consts, off_prow, off_red, off_bar, off_lists, off_totals, off_inv, total;
    uint32_t cap_hold, cap_led;      // delta mode: capacity of the inverted lists (0 = not staged)
};
// Column-major kernels: the 32 lanes of a warp generate 32 candidates at once and park them in the warp's
// scratch.  Per candidate: 4 header words — (partition 0 | partition 1 << 16), (partition 2 | replicas in the patched
// rows << 16), the C1 / C7 terms and the objective terms of the patched rows (patch_terms); 0xFFFF = no patch —
// then 32 * W bytes, one per slot: what the patched rows change in the column totals (patch_column_deltas).
// 16-byte aligned; the stride is an odd multiple of 4 words (the lanes' stores spread over 8 banks).
constexpr int kBatchHdr = 4;
__host__ __device__ constexpr int batch_stride_words(int W) { return kBatchHdr + 8 * W; }
static_assert(batch_stride_words(1) % 8 == 4 && batch_stride_words(2) % 8 == 4, "odd multiple of 4 words");

// prow_words_per_warp: per-warp scratch for patched rows (kMaxOps * W), or a whole batch of candidates
// lists: 1 stage the inverted lists of the per-thread generator if they fit, 0 never, -1 = for rows of up to 64 slots
// round_tables: the per-round tables of the delta kernels (at off_totals; the MMA column-major plan has none)
inline SmemPlan make_plan(int W, int Ppad, int warps, int obj_words_per_row, int P, int RF, bool oh_plane,
                          int prow_words_per_warp = 0, int lists = -1, int z_bytes = 0, bool round_tables = true)
{
    if (prow_words_per_warp <= 0) prow_words_per_warp = kMaxOps * W;
    SmemPlan s;
    uint32_t o = 0;
    s.off_bits = o;   o += (uint32_t)W * Ppad * 4;
    if (oh_plane) o += (uint32_t)W * Ppad * 4;            // leader one-hot plane, directly behind the bit-plane
    s.off_sw = o;     o += (uint32_t)obj_words_per_row * Ppad * 4;
    s.off_z = o;      o += (uint32_t)z_bytes;               // term planes of the column-major evaluator
    s.off_leader = o; o += (uint32_t)Ppad;
    s.off_consts = o; o += (uint32_t)sizeof(Consts);
    o = (o + 15u) & ~15u;
    s.off_prow = o;   o += (uint32_t)warps * prow_words_per_warp * 4;
    o = (o + 15u) & ~15u;
    s.off_red = o;    o += (uint32_t)(warps + 4) * 8;      // + early-stop state behind the per-warp minima
    s.off_bar = o;    o += 16;
    s.off_lists = o;  o += (uint32_t)Ppad * 4 + 16 + 2 * 36 * 4;   // D, DL (u16 each), counts, scan scratch
    s.off_totals = o; o += round_tables ? (256 + 256 + 32 + 4 + 256 + 2 * 258 + 4) * 4 : 0;  // per-round tables (kao_kernels.cuh, RoundTables): cnt,
                                                                           // lcnt, rc, base (viol, obj), led counts, list offsets, flag
    s.off_inv = o;
    s.cap_hold = s.cap_led = 0;
    if (lists < 0 ? W <= 2 : lists > 0) {   // inverted lists (u16 partitions) if they fit next to everything else
        const uint32_t nthreads = (uint32_t)warps * 32 > 512u ? (uint32_t)warps * 32 : 512u;      // (segment, slot) counts: one per thread
        const uint32_t need = ((uint32_t)P * RF + 258 + (uint32_t)P + 2 + 8) * 2 + 2 * nthreads * 4 + 16;
        if (o + need <= 227u * 1024u) {
            s.cap_hold = ((uint32_t)P * RF + 256 + 1) & ~1u;    // even counts keep the int scratch behind them aligned
            s.cap_led = ((uint32_t)P + 1) & ~1u;
            o += (need + 15u) & ~15u;
        }
    }
    s.total = o;
    return s;
}

// shared-memory plan of a column-major kernel: the two transposed planes + the term planes in place of the
// objective table, a batch of candidates per warp (the per-thread generator scans the transposed planes: no inverted lists).
// mma: the tensor-core form (kao_device_mma.cuh) keeps four shortfall planes behind the rack-field planes
// (16 nW bytes, at most 4 KB) and has no per-round tables (5,296 bytes): it fits wherever the other form does.
// cands: a sorted-batch schedule (kao_kernels.cuh, build_cand_list) keeps the class histogram, a CTA's share of a
// round — cands candidate indices sorted by class — and their class bytes behind everything else (at off_inv) if they
// fit: cand_list_cap(plan) entries, else none.
constexpr uint32_t kCandClasses = 256;
inline SmemPlan make_plan_t(int W, int Ppad, int threads, int P, int RF, bool mma = false, uint32_t cands = 0)
{
    // make_plan sizes the area at off_sw in words per partition of Ppad: the transposed planes hold t_words(Ppad)
    // words per slot, which is Ppad / 32 or (more than 1024 partitions) up to 31 words more — one extra word per
    // partition covers that for every Ppad the evaluator accepts
    const int nW = t_words(Ppad);
    const int per_row = (kTPlanes * W * 32 * nW + Ppad - 1) / Ppad;
    SmemPlan s = make_plan(W, Ppad, threads / 32, per_row, P, RF, false, 32 * batch_stride_words(W), 0,
                           (kZPlanes + 4 * W + (mma ? 4 : 0)) * nW * 4, !mma);  // term planes + rack-field planes (+ shortfall planes)
    const uint64_t need = ((uint64_t)kCandClasses + ((cands + 31u) & ~31ull)) * 5;      // + one class byte per candidate
    if (mma && cands > 0 && s.total + need <= 227u * 1024u) s.total += (uint32_t)need;
    return s;
}
// entries of the sorted candidate list of a tensor-core plan (0: none, the kernel walks its candidates unsorted)
__host__ __device__ inline uint32_t cand_list_cap(const SmemPlan &s)
{
    return s.total > s.off_inv + kCandClasses * 5 ? (s.total - s.off_inv) / 5 - kCandClasses : 0;
}
// does the column-major evaluator cover this layout (kao_create; tests/emu asks the same question)
inline bool column_major_fits(int W, int Ppad, int threads, int P, int RF)
{
    const SmemPlan s = make_plan_t(W, Ppad, threads, P, RF);
    return s.total <= 227u * 1024u;
}

// shared-memory plan of a delta kernel for rows wider than 64 slots: the base, the per-round tables and the
// inverted lists; the objective table stays in HBM / L2 (it is read for the <= 3 patched rows of a candidate)
inline SmemPlan make_plan_delta_wide(int W, int Ppad, int threads, int P, int RF)
{
    return make_plan(W, Ppad, threads / 32, 0, P, RF, false, 0, 1);
}
