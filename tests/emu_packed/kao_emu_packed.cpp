// kao_emu_packed.cpp — TEST INFRASTRUCTURE.  The packed MMA epilogue (csrc/kao_device_mma.cuh, the sorted-batch
// schedule pop 0x300) compiled for the host: the tensor-core emulation of tests/emu_mma with eval_batch_mma instantiated
// for pop 0x300, whose 16 x 2 SIMD runs as the header's host restatement.  32 candidates are generated one per lane,
// parked and evaluated together as one warp of the search kernel does it (batches in index order, so every shape and
// round size reaches the epilogue); winners patch the planes as in tests/emu_mma.  tests/test_packed_epilogue.py checks
// it against the oracle restatement.  Never linked into libkao.so.
#include "../emu_mma/kao_emu_mma.cpp"

namespace {

constexpr int kPackedPop = 0x300;
static_assert(EvalCfgT<1, 0, 1, kPackedPop>::kPacked && !EvalCfgT<1, 0, 1, 0x1300>::kPacked, "pop 0x300 is the packed epilogue");

// candidates idx0 .. idx0 + count - 1 (count <= 32): one batch of the search kernel
template <int W> void packed_keys_batch(MmaEmu &x, uint64_t seed, uint32_t round, uint32_t idx0, uint32_t count, uint32_t round_size,
                                        unsigned long long *out)
{
    Emu &e = *x.e;
    alignas(16) uint32_t batch[32 * batch_stride_words(W)];
    emu::run_warp([&](int lane) {
        mma_clear_batch<W>(batch, lane);
        __syncwarp();
        PatchSet ps;
        uint32_t rows[kMaxOps][W];
        ps.n = 0;
        for (int i = 0; i < kMaxOps; ++i) {
            ps.p[i] = -1; ps.ld[i] = 0xFF;
            for (int t = 0; t < W; ++t) rows[i][t] = 0;
        }
        if ((uint32_t)lane < count) make_gen<W>(x).run(seed, round, idx0 + lane, round_size, ps, rows);
        int pviol, pobj, pcount;
        patch_terms<W>(e.prm, ps, rows, pviol, pobj, pcount);
        mma_park_patch<W>(ps, rows, pviol, pobj, batch, lane);
        __syncwarp();
        int viol, obj;
        if (e.nW == 32) eval_batch_mma<EvalCfgT<W, 32, 1, kPackedPop>>(e.prm, &e.cs, x.T.data(), e.nW, x.Z.data(), batch, lane, viol, obj);
        else eval_batch_mma<EvalCfgT<W, 0, 1, kPackedPop>>(e.prm, &e.cs, x.T.data(), e.nW, x.Z.data(), batch, lane, viol, obj);
        const uint32_t j = (uint32_t)mma_lane_candidate(lane);
        if (j < count) out[j] = pack_key(viol, obj, idx0 + j, e.prm.key_obj_bits);
    });
}

template <int W> void packed_keys(MmaEmu &x, uint64_t seed, uint32_t round, uint32_t idx0, uint32_t count, uint32_t round_size,
                                  unsigned long long *out)
{
    for (uint32_t i = 0; i < count; i += 32) packed_keys_batch<W>(x, seed, round, idx0 + i, std::min(32u, count - i), round_size, out + i);
}

}  // namespace

extern "C" {

// keys of candidates idx_begin .. idx_begin + count - 1 by the packed epilogue (h: kao_emu_mma_create)
void kao_emu_packed_candidate_keys(void *h, uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_begin, uint32_t count,
                                   uint64_t *out)
{
    auto &x = *static_cast<MmaEmu *>(h);
    with_w(x, [&](auto w) {
        packed_keys<decltype(w)::value>(x, seed, round, idx_begin, count, round_size, reinterpret_cast<unsigned long long *>(out));
        return 0;
    });
}

// whole rounds: argmin of the keys, the winner becomes the base (kao_search, one GPU, no early stop)
void kao_emu_packed_search(void *h, uint64_t seed, uint32_t first_round, uint32_t rounds, uint32_t round_size, uint64_t *round_keys)
{
    auto &x = *static_cast<MmaEmu *>(h);
    with_w(x, [&](auto w) {
        constexpr int W = decltype(w)::value;
        std::vector<unsigned long long> all(round_size);
        for (uint32_t t = 0; t < rounds; ++t) {
            packed_keys<W>(x, seed, first_round + t, 0, round_size, round_size, all.data());
            unsigned long long best = kKeyNone;
            for (uint32_t i = 0; i < round_size; ++i) best = std::min(best, all[i]);
            if (round_keys) round_keys[t] = best;
            if (best != kKeyNone) apply<W>(x, seed, first_round + t, (uint32_t)(best & kIdxMask), round_size);
        }
        return 0;
    });
}

// the host forms of the epilogue's intrinsics one by one: op 0 vmax16x2, 1 vmin16x2, 2 __byte_perm(a, b, sel)
void kao_emu_simd(int op, const uint32_t *a, const uint32_t *b, uint32_t sel, uint32_t *out, int n)
{
    for (int i = 0; i < n; ++i)
        out[i] = op == 0 ? kao::vmax16x2(a[i], b[i]) : op == 1 ? kao::vmin16x2(a[i], b[i]) : __byte_perm(a[i], b[i], sel);
}

}  // extern "C"
