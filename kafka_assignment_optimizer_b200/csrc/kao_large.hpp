// kao_large.hpp — host interface of the large-instance path (kao_large.cu, DESIGN.md §7.1): sessions of
// more than kSmemRowsMax partitions keep their base in HBM (L2-resident) instead of shared memory and are searched
// with delta evaluation only.  Everything else of the engine (kao_engine.cu) stays as it is below that size.
#pragma once
#include "kao_kernels.cuh"
#include "kao_topics.cuh"

#include <cstdint>
#include <cuda_runtime.h>

// the largest row count the shared-memory resident kernels take (the base of every other kernel is staged per CTA)
constexpr int kSmemRowsMax = 8160;
// the largest row count of the large path: the largest multiple of 256 below 2^16, so that u16 partition ids, the
// 0xFFFF sentinel and Ppad stay valid
constexpr int kLargeRowsMax = 65280;

// What the winner of a round changes, written by CTA 0 after it has patched the HBM state and read by every CTA
// after the second grid barrier (each patches its own per-slot totals from it).
struct LargeRecord {
    int n;                          // patched partitions (0: no winner this round)
    int p[kMaxOps];
    uint32_t old_row[kMaxOps][8], new_row[kMaxOps][8];
    uint32_t old_ld[kMaxOps], new_ld[kMaxOps];
    int state[4];                   // |D|, |DL|, partitions led from a slot they do not hold, list buffer bits
};

// HBM state of a large session beyond Params: the transposed planes T0 / T1 ([2][32 W][tnW] words, the XOR swizzle of
// kao_device.cuh t_word) and the winner record.  Params.D / Params.DL hold two buffers of Ppad entries each (the list
// is rewritten into the other buffer when it changes); Params.nD = the four words of LargeRecord::state.
struct LargeArgs {
    uint32_t *T;
    int tnW;
    LargeRecord *rec;
};

// the HBM state derived from the base (transposed planes, displaced lists in buffer 0, leader validity count) after
// the base itself was uploaded
cudaError_t large_prepare(int W, const Params &d, const LargeArgs &la, cudaStream_t st);
// a topic session's counts and topic-row violation of the base, from scratch
cudaError_t topics_prepare(int W, const Params &d, const TopicArgs &ta, cudaStream_t st);
// rounds first_round .. first_round + rounds - 1 of a delta search in one cooperative launch (one CTA per SM);
// P2P: rank 0 of 1 (idx_lo / idx_hi, early stop, abort flag, rounds run).  all_keys != nullptr: one round, every
// candidate's key dumped, the base left as it is.  ta != nullptr: with the topic rows.  rftab != nullptr: every row's
// C1 / C7 operands from that per-partition table (docs/MODEL.md §11, replication_table in kao_host.hpp)
cudaError_t large_search(int W, int grid, const Params &d, const LargeArgs &la, uint64_t seed, uint32_t first_round,
                         uint32_t rounds, uint32_t round_size, unsigned long long *keys, unsigned int *grid_bar,
                         const P2P &pp, unsigned long long *all_keys, cudaStream_t st, const TopicArgs *ta = nullptr,
                         const uint32_t *rftab = nullptr);
// full evaluation of a topic or replication session's base: with its topic rows when ta != nullptr, with its
// per-partition rows when rftab != nullptr
cudaError_t large_eval_base(int W, const Params &d, const TopicArgs *ta, const uint32_t *rftab, long long *viol,
                            long long *obj, cudaStream_t st);
// full evaluation of n explicit assignments (bits [n][W][Ppad], leaders [n][Ppad]): one CTA each
cudaError_t large_eval(int W, const Params &d, const uint32_t *bits, const uint8_t *leader, int n, long long *viol,
                       long long *obj, cudaStream_t st);
