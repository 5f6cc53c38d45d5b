// kao_emu_mma.cpp — TEST INFRASTRUCTURE.  The tensor-core form of the column-major evaluator
// (csrc/kao_device_mma.cuh, schedules with pop 0x100) compiled for the host: the emulator of tests/emu (host model,
// base, per-thread generator, row-major evaluator) plus the batched body, ldmatrix and the binary MMA restated by
// mma_emu.hpp.  As one warp of the search kernel does it, 32 candidates are generated one per lane, parked in the
// warp's batch and evaluated together; winners patch the transposed, term, rack-field and shortfall planes with
// t_patch_row.  tests/test_mma_emulation.py checks it against the oracle restatement.  Never linked into libkao.so.
#define KAO_HOST_EMU 1
#include "mma_emu.hpp"
#include "../emu/kao_emu.cpp"
#include "../../kafka_assignment_optimizer_b200/csrc/kao_device_mma.cuh"

namespace {

struct MmaEmu {
    Emu *e = nullptr;
    std::vector<uint32_t> T, Z;          // transposed planes; term, rack-field and shortfall planes
};

template <int W> void build_planes(MmaEmu &x)
{
    Emu &e = *x.e;
    const int nW = e.nW, Ppad = e.hm.Ppad;
    x.T.assign((size_t)kTPlanes * 32 * W * nW, 0);
    for (int q = 0; q < kTPlanes; ++q)
        for (int s = 0; s < 32 * W; ++s)
            for (int w = 0; w < nW; ++w) x.T[t_word(q, s, w, nW, 32 * W)] = t_gather<W>(q, s, w, e.bits.data(), e.leader.data(), Ppad);
    x.Z.assign((size_t)(kZPlanes + kAPlanes<W>() + kSPlanes) * nW, 0);
    for (int j = 0; j < kZPlanes; ++j)
        for (int w = 0; w < nW; ++w) x.Z[(size_t)j * nW + w] = z_gather<W>(e.prm, j, w, e.bits.data(), e.leader.data());
    for (int b = 0; b < kAPlanes<W>(); ++b)
        for (int w = 0; w < nW; ++w) x.Z[(size_t)(kZPlanes + b) * nW + w] = a_gather<W>(b, w, e.bits.data(), Ppad);
    for (int k = 0; k < kSPlanes; ++k)
        for (int w = 0; w < nW; ++w) x.Z[(size_t)(kZPlanes + kAPlanes<W>() + k) * nW + w] = s_gather<W>(e.prm, k, w, e.bits.data());
}

template <int W> Gen<W, true, true> make_gen(MmaEmu &x)
{
    Emu &e = *x.e;
    Gen<W, true, true> tg;
    tg.bitsT = e.bits.data(); tg.leader = e.leader.data(); tg.cs = &e.cs; tg.d = &e.prm; tg.prow = nullptr; tg.lane = 0;
    tg.D = e.D.data(); tg.DL = e.DL.data(); tg.nD = e.nD; tg.nL = e.nL;
    tg.T = x.T.data(); tg.tnW = e.nW; tg.t_leaders_valid = e.n_invalid == 0;
    return tg;
}

// candidates idx0 .. idx0 + count - 1 (count <= 32): one batch of the search kernel
template <int W> void keys_batch(MmaEmu &x, uint64_t seed, uint32_t round, uint32_t idx0, uint32_t count, uint32_t round_size,
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
        if (e.nW == 32) eval_batch_mma<EvalCfgT<W, 32, 1, 0x100>>(e.prm, &e.cs, x.T.data(), e.nW, x.Z.data(), batch, lane, viol, obj);
        else eval_batch_mma<EvalCfgT<W, 0, 1, 0x100>>(e.prm, &e.cs, x.T.data(), e.nW, x.Z.data(), batch, lane, viol, obj);
        const uint32_t j = (uint32_t)mma_lane_candidate(lane);
        if (j < count) out[j] = pack_key(viol, obj, idx0 + j, e.prm.key_obj_bits);
    });
}

template <int W> void keys(MmaEmu &x, uint64_t seed, uint32_t round, uint32_t idx0, uint32_t count, uint32_t round_size,
                           unsigned long long *out)
{
    for (uint32_t i = 0; i < count; i += 32) keys_batch<W>(x, seed, round, idx0 + i, std::min(32u, count - i), round_size, out + i);
}

// the winner becomes the base: every lane rewrites its words of the planes (t_patch_row with the shortfall planes),
// the row-major base and the lists follow (search_persistent_kernel, after the grid barrier)
template <int W> void apply(MmaEmu &x, uint64_t seed, uint32_t round, uint32_t idx, uint32_t round_size)
{
    Emu &e = *x.e;
    PatchSet win;
    uint32_t wrows[kMaxOps][W];
    emu::run_warp([&](int lane) {
        PatchSet ps;
        uint32_t rows[kMaxOps][W];
        for (int i = 0; i < kMaxOps; ++i)
            for (int t = 0; t < W; ++t) rows[i][t] = 0;
        make_gen<W>(x).run(seed, round, idx, round_size, ps, rows);
        if (lane == 0) {
            win = ps;
            std::memcpy(wrows, rows, sizeof(rows));
        }
    });
    const int Ppad = e.hm.Ppad;
    for (int i = 0; i < win.n; ++i) {
        for (int lane = 0; lane < 32; ++lane)
            t_patch_row<W, true>(e.prm, x.T.data(), x.Z.data(), e.nW, win.p[i], wrows[i], win.ld[i], lane);
        for (int w = 0; w < W; ++w) {
            e.bits[(size_t)w * Ppad + win.p[i]] = wrows[i][w];
            if (e.oh) e.bits[(size_t)(W + w) * Ppad + win.p[i]] = oh_word(wrows[i][w], win.ld[i], w);
        }
        e.leader[win.p[i]] = (uint8_t)win.ld[i];
    }
    rebuild_lists(e);
}

template <class F> auto with_w(MmaEmu &x, F f) { return x.e->hm.W == 1 ? f(std::integral_constant<int, 1>{}) : f(std::integral_constant<int, 2>{}); }

}  // namespace

extern "C" {

// nullptr (kao_emu_last_error) unless the column-major evaluator covers the layout
void *kao_emu_mma_create(const kao_problem *pb)
{
    Emu *e = static_cast<Emu *>(kao_emu_create(pb));
    if (!e) return nullptr;
    if (!e->trans_ok) {
        g_err = "column-major evaluator: unsupported layout";
        delete e;
        return nullptr;
    }
    auto *x = new MmaEmu;
    x->e = e;
    with_w(*x, [&](auto w) { build_planes<decltype(w)::value>(*x); return 0; });
    return x;
}

void kao_emu_mma_destroy(void *h)
{
    auto *x = static_cast<MmaEmu *>(h);
    delete x->e;
    delete x;
}

void kao_emu_mma_set_base(void *h, const int32_t *replicas)
{
    auto &x = *static_cast<MmaEmu *>(h);
    kao_emu_set_base(x.e, replicas);
    with_w(x, [&](auto w) { build_planes<decltype(w)::value>(x); return 0; });
}

// replica lists of the base and its evaluation by the row-major evaluator (the identity candidate)
void kao_emu_mma_get_base(void *h, int32_t *replicas, int64_t *violation, int64_t *objective, int32_t *moves)
{
    kao_emu_get_base(static_cast<MmaEmu *>(h)->e, replicas, violation, objective, moves);
}

void kao_emu_mma_candidate_keys(void *h, uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_begin, uint32_t count,
                                uint64_t *out)
{
    auto &x = *static_cast<MmaEmu *>(h);
    with_w(x, [&](auto w) {
        keys<decltype(w)::value>(x, seed, round, idx_begin, count, round_size, reinterpret_cast<unsigned long long *>(out));
        return 0;
    });
}

// whole rounds: argmin of the keys, the winner becomes the base (kao_search, one GPU, no early stop)
void kao_emu_mma_search(void *h, uint64_t seed, uint32_t first_round, uint32_t rounds, uint32_t round_size, uint64_t *round_keys)
{
    auto &x = *static_cast<MmaEmu *>(h);
    with_w(x, [&](auto w) {
        constexpr int W = decltype(w)::value;
        std::vector<unsigned long long> all(round_size);
        for (uint32_t t = 0; t < rounds; ++t) {
            keys<W>(x, seed, first_round + t, 0, round_size, round_size, all.data());
            unsigned long long best = kKeyNone;
            for (uint32_t i = 0; i < round_size; ++i) best = std::min(best, all[i]);
            if (round_keys) round_keys[t] = best;
            if (best != kKeyNone) apply<W>(x, seed, first_round + t, (uint32_t)(best & kIdxMask), round_size);
        }
        return 0;
    });
}

}  // extern "C"
