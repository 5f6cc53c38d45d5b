// kao_emu.cpp — TEST INFRASTRUCTURE.  The engine's own device code (csrc/kao_device.cuh: candidate
// generator, full evaluator, delta evaluator) compiled for the host on top of warp_emu.hpp, with the
// engine's own host model (csrc/kao_host.hpp) and shared-memory plan (csrc/kao_plan.hpp) deciding
// layout and evaluator configuration exactly as kao_create / dispatch do.  tests/test_device_emulation.py
// checks it against the committed golden streams and the oracle restatement, so the arithmetic of the
// CUDA path is exercised by the CPU suite as well; the kernels themselves (staging, grid barrier,
// cross-GPU exchange) are only tested on the GPU.  Replication sessions (kao_emu_create_replication) run the kRF forms
// of the row and delta evaluators on the HBM-base kernels' configuration (tests/test_replication_emulation.py); topic
// sessions (kao_emu_create_topics) add the topic rows of csrc/kao_topics.cuh to it (tests/test_slot255_cpu.py).
// tensor_core.cpp (the tensor-core body) and reduce_fixed.cpp (the fixed-partition reduction) are included at the end:
// one translation unit, one library, tests/emu/_build/libkao_emu.so.  Never linked into libkao.so.
#define KAO_HOST_EMU 1
#include "warp_emu.hpp"

#include "../../kafka_assignment_optimizer_b200/csrc/kao_device.cuh"
#include "../../kafka_assignment_optimizer_b200/csrc/kao_device_t.cuh"
#include "../../kafka_assignment_optimizer_b200/csrc/kao_topics.cuh"
#include "../../kafka_assignment_optimizer_b200/csrc/kao_plan.hpp"
#include "../../kafka_assignment_optimizer_b200/csrc/kao_host.hpp"

#include <cstring>
#include <memory>
#include <string>
#include <vector>

using namespace kao;

namespace {

struct Emu {
    HostModel hm;
    Params prm{};
    Consts cs{};
    bool oh = false;                     // leader one-hot plane kept behind the bit-plane (has_oh_plane)
    int nph = 3, rack = 0, obj = 0;      // evaluator configuration (EvalCfg<W, NPH, kRack, kObj>)
    std::vector<uint32_t> bits;          // [W or 2W][Ppad]
    std::vector<uint8_t> leader;         // [Ppad]
    std::vector<uint16_t> D, DL;
    int nD = 0, nL = 0;
    std::vector<uint32_t> prow;          // [kMaxOps * W]
    // column-major evaluator (kao_device_t.cuh): supported shape, in use, the five transposed planes
    bool trans_ok = false;
    int trans = 0;                       // 0 row-major evaluator, 1.. forms (schedules) of the column-major one
    int nW = 0;
    std::vector<uint32_t> T, Z;          // transposed planes, term planes of the objective
    int n_invalid = 0;                   // partitions led from a slot that holds none of their replicas (s_counts[2] of the kernel)
    // a replication session (kao_create_replication): every row's C1 / C7 operands from rftab, evaluated as the
    // HBM-base kernels do (kao_large.cu: LargeCfg<W>, block_eval / delta_eval with kRF)
    bool rf = false;
    std::vector<uint32_t> rftab;         // [Ppad] rf | ppr_lo << 8 | ppr_hi << 16 (replication_table)
    // a topic session (kao_create_topics): the same kernels with the topic rows; the counts and tviol of the base are
    // rebuilt by set_base and patched winner by winner, as topics_prepare / apply_winner_topics keep them
    bool topics = false;
    HostTopics ht;
    std::vector<int4> tbnd;              // [T]
    std::vector<uint16_t> tcnt, tlcnt;   // [T][32 W]
    int tviol = 0;
    TopicArgs ta{};
    std::string err;
};

template <int W> void build_T(Emu &e)
{
    const HostModel &m = e.hm;
    e.T.assign((size_t)kTPlanes * 32 * W * e.nW, 0);
    for (int q = 0; q < kTPlanes; ++q)
        for (int s = 0; s < 32 * W; ++s)
            for (int w = 0; w < e.nW; ++w)
                e.T[t_word(q, s, w, e.nW, 32 * W)] = t_gather<W>(q, s, w, e.bits.data(), e.leader.data(), m.Ppad);
    e.Z.assign((size_t)(kZPlanes + kAPlanes<W>()) * e.nW, 0);
    for (int j = 0; j < kZPlanes; ++j)
        for (int w = 0; w < e.nW; ++w) e.Z[(size_t)j * e.nW + w] = z_gather<W>(e.prm, j, w, e.bits.data(), e.leader.data());
    for (int b = 0; b < kAPlanes<W>(); ++b)
        for (int w = 0; w < e.nW; ++w) e.Z[(size_t)(kZPlanes + b) * e.nW + w] = a_gather<W>(b, w, e.bits.data(), m.Ppad);
}

uint32_t oh_word(uint32_t x, uint32_t ld, int w) { return ((int)(ld >> 5) == w) ? (x & (1u << (ld & 31u))) : 0u; }

// partitions led from a slot that holds none of their replicas, counted over the whole base (the kernel's staging pass)
int count_invalid(const Emu &e)
{
    const HostModel &m = e.hm;
    int n = 0;
    for (int p = 0; p < m.P; ++p) {
        const int ld = e.leader[p];
        if (!(ld < 32 * m.W && ((e.bits[(size_t)(ld >> 5) * m.Ppad + p] >> (ld & 31)) & 1u))) ++n;
    }
    return n;
}

// s_counts[2] after a winner's row i replaces partition p's row and leader, as search_persistent_kernel updates it
// (before the row is written): -1 if the old leader was invalid, +1 if the new one is
void patch_invalid(Emu &e, int p, const uint32_t *newrow, int ln)
{
    const int W = e.hm.W, lo = e.leader[p];
    const bool was = lo < W * 32 && ((e.bits[(size_t)(lo >> 5) * e.hm.Ppad + p] >> (lo & 31)) & 1u);
    const bool is = ln < W * 32 && ((newrow[ln >> 5] >> (ln & 31)) & 1u);
    e.n_invalid += (was ? 0 : -1) + (is ? 0 : 1);
}

// rebuild_lists of kao_kernels.cuh: ascending partitions that miss a home slot (D) / hold home slot
// 0 without being led from it (DL)
void rebuild_lists(Emu &e)
{
    const HostModel &m = e.hm;
    e.nD = e.nL = 0;
    for (int p = 0; p < m.P; ++p) {
        const uint32_t h4 = m.homeT[p];
        const uint32_t hv = m.W == 8 ? home_valid<8>(m.homeT.data(), m.Ppad, p) : 0u;
        bool miss = false, ldis = false;
        for (int i = 0; i < 4; ++i) {
            const int hs = (h4 >> (8 * i)) & 0xFF;
            if (!(m.W == 8 ? home_ok<8>(hs, hv, i) : home_ok<4>(hs, hv, i))) continue;
            const bool has = (e.bits[(size_t)(hs >> 5) * m.Ppad + p] >> (hs & 31)) & 1u;
            miss |= !has;
            if (i == 0) ldis = has && ((int)e.leader[p] != hs);
        }
        if (miss) e.D[e.nD++] = (uint16_t)p;
        if (ldis) e.DL[e.nL++] = (uint16_t)p;
    }
}

// topics_prepare: the base's replicas and valid leaders per (topic, broker slot) (topic_count_kernel), then the
// topic-row violation over every such cell (topic_violation_kernel)
void count_topics(Emu &e)
{
    const HostModel &m = e.hm;
    const int NSL = 32 * m.W;
    e.tcnt.assign((size_t)e.ht.T * NSL, 0);
    e.tlcnt.assign((size_t)e.ht.T * NSL, 0);
    for (int p = 0; p < m.P; ++p) {
        const size_t t = e.ht.topic_of[p];
        const int ld = e.leader[p];
        for (int s = 0; s < NSL; ++s) {
            if (!((e.bits[(size_t)(s >> 5) * m.Ppad + p] >> (s & 31)) & 1u) || !broker_slot(&e.cs, m.B, s)) continue;
            ++e.tcnt[t * NSL + s];
            if (s == ld) ++e.tlcnt[t * NSL + s];
        }
    }
    e.tviol = 0;
    for (size_t i = 0; i < e.tcnt.size(); ++i) {
        if (!broker_slot(&e.cs, m.B, (int)(i % NSL))) continue;
        const int4 b = e.tbnd[i / NSL];
        e.tviol += band_int(e.tcnt[i], b.x, b.y) + band_int(e.tlcnt[i], b.z, b.w);
    }
    e.ta.tcnt = e.tcnt.data();
    e.ta.tlcnt = e.tlcnt.data();
}

void set_base(Emu &e, const std::vector<uint32_t> &bitsT, const std::vector<uint8_t> &leader)
{
    const HostModel &m = e.hm;
    e.bits.assign((size_t)(e.oh ? 2 : 1) * m.W * m.Ppad, 0);
    std::copy(bitsT.begin(), bitsT.end(), e.bits.begin());
    e.leader = leader;
    if (e.oh)
        for (int p = 0; p < m.Ppad; ++p)
            for (int w = 0; w < m.W; ++w)
                e.bits[(size_t)(m.W + w) * m.Ppad + p] = oh_word(e.bits[(size_t)w * m.Ppad + p], e.leader[p], w);
    e.prm.bitsT = e.bits.data();
    e.prm.leader = e.leader.data();
    rebuild_lists(e);
    e.n_invalid = count_invalid(e);
    if (e.trans_ok) { if (m.W == 1) build_T<1>(e); else build_T<2>(e); }
    if (e.topics) count_topics(e);
}

// State a search patches winner by winner, against the same state rebuilt from the current bits / leader: the one-hot
// plane, the count of invalid leaders, the displaced lists.  0, or 3.. (kao_emu_check_state) with the first differing
// index in *at and a message in g_err.
int check_state_msg(int code, const char *what, long long at, long long *out_at, std::string &err)
{
    *out_at = at;
    err = std::string("patched ") + what + " differs from the rebuilt one at index " + std::to_string(at);
    return code;
}

int check_base_state(Emu &e, long long *at, std::string &err)
{
    const HostModel &m = e.hm;
    if (e.oh)
        for (int w = 0; w < m.W; ++w)
            for (int p = 0; p < m.Ppad; ++p) {
                const size_t i = (size_t)(m.W + w) * m.Ppad + p;
                if (e.bits[i] != oh_word(e.bits[(size_t)w * m.Ppad + p], e.leader[p], w))
                    return check_state_msg(3, "leader one-hot plane", (long long)i, at, err);
            }
    const int n_inv = count_invalid(e);
    if (n_inv != e.n_invalid) {
        *at = e.n_invalid;
        err = "patched count of invalid leaders " + std::to_string(e.n_invalid) + ", rebuilt " + std::to_string(n_inv);
        return 4;
    }
    const std::vector<uint16_t> D = e.D, DL = e.DL;
    const int nD = e.nD, nL = e.nL;
    rebuild_lists(e);
    int rc = 0;
    if (nD != e.nD || nL != e.nL) {
        *at = nD != e.nD ? 0 : 1;
        err = "patched list lengths (" + std::to_string(nD) + ", " + std::to_string(nL) + "), rebuilt (" +
              std::to_string(e.nD) + ", " + std::to_string(e.nL) + ")";
        rc = 5;
    }
    for (int i = 0; rc == 0 && i < nD; ++i)
        if (D[i] != e.D[i]) rc = check_state_msg(6, "list D", i, at, err);
    for (int i = 0; rc == 0 && i < nL; ++i)
        if (DL[i] != e.DL[i]) rc = check_state_msg(7, "list DL", i, at, err);
    e.D = D; e.DL = DL; e.nD = nD; e.nL = nL;        // the session keeps the state it patched
    return rc;
}

// the first index at which two plane arrays differ, or -1
long long first_diff(const std::vector<uint32_t> &a, const std::vector<uint32_t> &b)
{
    if (a.size() != b.size()) return (long long)std::min(a.size(), b.size());
    for (size_t i = 0; i < a.size(); ++i)
        if (a[i] != b[i]) return (long long)i;
    return -1;
}

template <class Cfg> struct Run {
    static constexpr int W = Cfg::W;
    template <bool kSmall> static Gen<W, false, kSmall> make_gen(Emu &e, int lane)
    {
        Gen<W, false, kSmall> g;
        g.bitsT = e.bits.data(); g.leader = e.leader.data(); g.cs = &e.cs; g.d = &e.prm;
        g.prow = e.prow.data(); g.lane = lane;
        g.D = e.D.data(); g.DL = e.DL.data(); g.nD = e.nD; g.nL = e.nL;
        return g;
    }
    // the per-thread generator of the column-major kernels: every lane generates the candidate for itself ("first holder
    // of slot s" = scan of the transposed planes), lane 0 parks the patched rows where the evaluator reads them
    static void gen_thread(Emu &e, int lane, uint64_t seed, uint32_t round, uint32_t idx, uint32_t round_size, PatchSet &ps)
    {
        Gen<W, true, true> tg;
        tg.bitsT = e.bits.data(); tg.leader = e.leader.data(); tg.cs = &e.cs; tg.d = &e.prm; tg.prow = nullptr; tg.lane = 0;
        tg.D = e.D.data(); tg.DL = e.DL.data(); tg.nD = e.nD; tg.nL = e.nL;
        tg.T = e.T.data(); tg.tnW = e.nW; tg.t_leaders_valid = e.n_invalid == 0;
        uint32_t rows[kMaxOps][W];
        for (int i = 0; i < kMaxOps; ++i)
            for (int t = 0; t < W; ++t) rows[i][t] = 0;
        tg.run(seed, round, idx, round_size, ps, rows);
        if (lane == 0)
            for (int i = 0; i < kMaxOps; ++i)
                for (int t = 0; t < W; ++t) e.prow[i * W + t] = rows[i][t];
    }
    // generate + evaluate in full, as one warp of the search kernels does
    static unsigned long long key(Emu &e, uint64_t seed, uint32_t round, uint32_t idx, uint32_t round_size)
    {
        unsigned long long out = 0;
        const uint32_t *objT = Cfg::kObj > 0 ? e.prm.planesT : e.prm.swT;
        emu::run_warp([&](int lane) {
            uint32_t no_rows[kMaxOps][W];
            PatchSet ps;
            if constexpr (W <= 2) {
                if (e.trans) gen_thread(e, lane, seed, round, idx, round_size, ps);               // as the column-major kernels
                else make_gen<false>(e, lane).run(seed, round, idx, round_size, ps, no_rows);
            } else {
                make_gen<false>(e, lane).run(seed, round, idx, round_size, ps, no_rows);
            }
            __syncwarp();                                     // __syncthreads() of the kernels
            int viol, obj;
            if constexpr (W <= 2) {
                // forms of the column-major evaluator: 1 as the engine picks it (32-word specialisation where it
                // applies, default popcount streams), 2 run-time word count, 3 a POPC per word, 4 three POPC per four
                // words, 5 Harley-Seal on the column totals, 6 Harley-Seal on both streams
                const bool fixed = e.nW == 32;
                uint32_t prows[kMaxOps][W];
                for (int i = 0; i < kMaxOps; ++i)
                    for (int t = 0; t < W; ++t) prows[i][t] = ps.p[i] >= 0 ? e.prow[i * W + t] : 0u;
                int pviol = 0, pobj = 0, pcount = 0;
                LaneBounds<W> lb;
                lb.load(&e.cs, lane, e.prm.R);
                alignas(16) uint8_t pdelta[32 * W];                                      // every fiber keeps its own copy (the kernel: the warp's batch)
                if (e.trans) {                                                           // per candidate, as the per-thread generator does
                    patch_terms<W>(e.prm, ps, prows, pviol, pobj, pcount);
                    patch_column_deltas<W>(e.prm, ps, prows, e.bits.data(), e.leader.data(), pdelta);
                }
#define KAO_EMU_T(NW_, POP_) eval_candidate_t<EvalCfgT<W, NW_, 1, POP_>, true>(e.prm, e.T.data(), e.nW, e.bits.data(), e.Z.data(), lb, ps, pdelta, pviol, pobj, pcount, lane, viol, obj)
                if (e.trans == 1 && fixed) KAO_EMU_T(32, 0x22);
                else if (e.trans == 1 || e.trans == 2) KAO_EMU_T(0, 0x22);
                else if (e.trans == 3 && fixed) KAO_EMU_T(32, 0x00);
                else if (e.trans == 3) KAO_EMU_T(0, 0x00);
                else if (e.trans == 4 && fixed) KAO_EMU_T(32, 0x11);
                else if (e.trans == 4) KAO_EMU_T(0, 0x11);
                else if (e.trans == 5 && fixed) KAO_EMU_T(32, 0x23);
                else if (e.trans == 5) KAO_EMU_T(0, 0x23);
                else if (e.trans == 6 && fixed) KAO_EMU_T(32, 0x33);
                else if (e.trans == 6) KAO_EMU_T(0, 0x33);
#undef KAO_EMU_T
                else eval_candidate<Cfg, true>(e.prm, e.bits.data(), e.leader.data(), objT, &e.cs, ps, e.prow.data(), lane, viol, obj);
            } else {
                eval_candidate<Cfg, true>(e.prm, e.bits.data(), e.leader.data(), objT, &e.cs, ps, e.prow.data(), lane, viol, obj);
            }
            if (lane == 0) out = pack_key(viol, obj, idx, e.prm.key_obj_bits);
        });
        return out;
    }
    // the winner becomes the base (search_persistent_kernel, after the grid barrier)
    static void apply(Emu &e, uint64_t seed, uint32_t round, uint32_t idx, uint32_t round_size)
    {
        PatchSet win;
        emu::run_warp([&](int lane) {
            uint32_t no_rows[kMaxOps][W];
            PatchSet ps;
            if constexpr (W <= 2) {
                if (e.trans) gen_thread(e, lane, seed, round, idx, round_size, ps);
                else make_gen<false>(e, lane).run(seed, round, idx, round_size, ps, no_rows);
            } else {
                make_gen<false>(e, lane).run(seed, round, idx, round_size, ps, no_rows);
            }
            if (lane == 0) win = ps;
        });
        const int Ppad = e.hm.Ppad;
        for (int i = 0; i < win.n; ++i) {
            if constexpr (W <= 2) {
                if (e.trans_ok) {                   // as the kernel does: every lane rewrites its own slots' words
                    uint32_t newrow[W];
                    for (int w = 0; w < W; ++w) newrow[w] = e.prow[i * W + w];
                    for (int lane = 0; lane < 32; ++lane)
                        t_patch_row<W>(e.prm, e.T.data(), e.Z.data(), e.nW, win.p[i], newrow, win.ld[i], lane);
                }
            }
            patch_invalid(e, win.p[i], &e.prow[(size_t)i * W], win.ld[i]);
            for (int w = 0; w < W; ++w) {
                const uint32_t v = e.prow[i * W + w];
                e.bits[(size_t)w * Ppad + win.p[i]] = v;
                if (e.oh) e.bits[(size_t)(W + w) * Ppad + win.p[i]] = oh_word(v, win.ld[i], w);
            }
            e.leader[win.p[i]] = (uint8_t)win.ld[i];
        }
        rebuild_lists(e);
    }
    // the base's own evaluation as the delta kernel's full pass computes it (identity candidate, row-major
    // evaluator): the raw violation, which a packed key would cap at its field width
    static void base_eval(Emu &e, int &viol, int &obj)
    {
        const uint32_t *objT = Cfg::kObj > 0 ? e.prm.planesT : e.prm.swT;
        emu::run_warp([&](int lane) {
            PatchSet id;
            id.n = 0;
            for (int i = 0; i < kMaxOps; ++i) { id.p[i] = -1; id.ld[i] = 0xFF; }
            int v, o;
            eval_candidate<Cfg, true>(e.prm, e.bits.data(), e.leader.data(), objT, &e.cs, id, e.prow.data(), lane, v, o);
            if (lane == 0) { viol = v; obj = o; }
        });
    }
    // delta mode (search_persistent_kernel<..., kDelta>): per-thread generator + delta evaluator on
    // the base's totals; no inverted lists here (the generator's linear-scan form)
    static unsigned long long key_delta(Emu &e, uint64_t seed, uint32_t round, uint32_t idx, uint32_t round_size,
                                        const int *cnt, const int *lcnt, const int *rc, int base_viol, int base_obj)
    {
        Gen<W, true> tg;
        tg.bitsT = e.bits.data(); tg.leader = e.leader.data(); tg.cs = &e.cs; tg.d = &e.prm; tg.prow = nullptr; tg.lane = 0;
        tg.D = e.D.data(); tg.DL = e.DL.data(); tg.nD = e.nD; tg.nL = e.nL;
        const uint32_t *objT = Cfg::kObj > 0 ? e.prm.planesT : e.prm.swT;
        const MemRef<true> m_obj(objT);
        PatchSet ps;
        uint32_t rows[kMaxOps][W];
        tg.run(seed, round, idx, round_size, ps, rows);
        int viol, obj;
        delta_eval<Cfg>(e.prm, e.bits.data(), e.leader.data(), m_obj, &e.cs, ps, rows, cnt, lcnt, rc, base_viol, base_obj, viol, obj);
        return pack_key(viol, obj, idx, e.prm.key_obj_bits);
    }
};

// explicit candidate from HBM-style buffers (eval_batch_kernel): general rack form, packed entries
template <int W, int NPH> void eval_explicit(Emu &e, const uint32_t *cb, const uint8_t *cl, long long &viol, long long &obj)
{
    int v = 0, o = 0;
    emu::run_warp([&](int lane) {
        PatchSet ps;
        ps.n = 0;
        for (int i = 0; i < kMaxOps; ++i) { ps.p[i] = -1; ps.ld[i] = 0xFF; }
        int lv, lo;
        eval_candidate<EvalCfg<W, NPH, 0, kObjEntries>, false>(e.prm, cb, cl, e.prm.swT, &e.cs, ps, nullptr, lane, lv, lo);
        if (lane == 0) { v = lv; o = lo; }
    });
    viol = v; obj = o;
}

// kao_engine.cu: dispatch / dispatch_w / dispatch_obj.  X(W, NPH, rack form, objective planes) for every
// evaluator configuration the engine instantiates (kao_kernels.cuh: KAO_FOR_CFGS_*, kao_inst.cu)
#define KAO_EMU_RACKS(X, W_, NPH_, O_) X(W_, NPH_, 0, O_) X(W_, NPH_, 3, O_) X(W_, NPH_, 4, O_) X(W_, NPH_, 5, O_)
#define KAO_EMU_NARROW(X, W_, NPH_) KAO_EMU_RACKS(X, W_, NPH_, 0) KAO_EMU_RACKS(X, W_, NPH_, 3)
#define KAO_EMU_CFGS(X) \
    KAO_EMU_NARROW(X, 1, 5) KAO_EMU_NARROW(X, 2, 5) KAO_EMU_RACKS(X, 4, 5, 0) KAO_EMU_RACKS(X, 8, 5, 0) KAO_EMU_NARROW(X, 1, 6)
template <class F> auto dispatch(Emu &e, F f)
{
#define KAO_EMU_CASE(W_, NPH_, R_, O_) \
    if (e.hm.W == W_ && e.nph == NPH_ && e.rack == R_ && e.obj == O_) return f(Run<EvalCfg<W_, NPH_, R_, O_>>{});
    KAO_EMU_CFGS(KAO_EMU_CASE)
#undef KAO_EMU_CASE
    fprintf(stderr, "kao_emu: no evaluator configuration W=%d NPH=%d rack=%d obj=%d\n", e.hm.W, e.nph, e.rack, e.obj);
    abort();
    return f(Run<EvalCfg<1, 5, 0, 0>>{});
}

// The HBM-base kernels of a replication or topic session (kao_large.cu: search_large_kernel<W, kTopics, kRF>,
// eval_large_base_kernel<W, kRF>): their one evaluator configuration; kRF: every row's C1 / C7 operands from rftab;
// e.topics: the topic rows of kao_topics.cuh on top.
template <int W> using LargeCfg = EvalCfg<W, 5, 0, kObjEntries>;

template <int W, bool kRF> struct RunLarge {
    struct Totals {
        std::vector<int> cnt = std::vector<int>(256, 0), lcnt = std::vector<int>(256, 0), rc = std::vector<int>(32, 0);
        long long viol = 0, obj = 0;                   // raw, as block_eval leaves them in acc
    };
    // block_eval<W, true>: row_eval with each row's own operands, the replica / valid-leader count per slot and the
    // replica count per rack, then the C3 / C4 / C6 bands
    static Totals base(const Emu &e)
    {
        const Params &d = e.prm;
        const MemRef<false> m_obj(d.swT);
        Totals t;
        for (int p = 0; p < d.P; ++p) {
            uint32_t x[W];
            for (int w = 0; w < W; ++w) x[w] = e.bits[(size_t)w * d.Ppad + p];
            const uint32_t ld = e.leader[p];
            int rv, ro;
            if constexpr (kRF) row_eval<LargeCfg<W>, false, true>(d, m_obj, p, x, ld, rv, ro, row_rf(e.rftab.data(), p));
            else row_eval<LargeCfg<W>, false>(d, m_obj, p, x, ld, rv, ro);
            t.viol += rv;
            t.obj += ro;
            for (int w = 0; w < W; ++w)
                for (uint32_t m = x[w]; m; m &= m - 1) {
                    const int s = 32 * w + __ffs(m) - 1;
                    ++t.cnt[s];
                    ++t.rc[s >> d.log2S];
                }
            if ((int)ld < 32 * W && row_has<W>(x, (int)ld)) ++t.lcnt[ld];
        }
        for (int s = 0; s < 32 * W; ++s)
            t.viol += band_violation(t.cnt[s], e.cs.bnd_rep[s]) + band_violation(t.lcnt[s], e.cs.bnd_ldr[s]);
        for (int r = 0; r < d.R; ++r)
            t.viol += std::max(t.rc[r] - e.cs.rack_hi[r], 0) + std::max(e.cs.rack_lo[r] - t.rc[r], 0);
        if (e.topics) t.viol += e.tviol;              // the search kernel adds tviol to block_eval's total
        return t;
    }
    // the per-thread generator on the base (its linear-scan form), as large_gen hands it to each thread
    static void gen(const Emu &e, uint64_t seed, uint32_t round, uint32_t idx, uint32_t round_size, PatchSet &ps,
                    uint32_t (&rows)[kMaxOps][W])
    {
        Gen<W, true> tg;
        tg.bitsT = e.bits.data(); tg.leader = e.leader.data(); tg.cs = &e.cs; tg.d = &e.prm; tg.prow = nullptr; tg.lane = 0;
        tg.D = e.D.data(); tg.DL = e.DL.data(); tg.nD = e.nD; tg.nL = e.nL;
        tg.run(seed, round, idx, round_size, ps, rows);
    }
    // one candidate of the search kernel: delta_eval<LargeCfg<W>, false, true> on the base's totals
    static unsigned long long key(const Emu &e, const Totals &t, int base_viol, int base_obj, uint64_t seed,
                                  uint32_t round, uint32_t idx, uint32_t round_size)
    {
        PatchSet ps;
        uint32_t rows[kMaxOps][W];
        gen(e, seed, round, idx, round_size, ps, rows);
        int viol, obj;
        delta_eval<LargeCfg<W>, false, kRF>(e.prm, e.bits.data(), e.leader.data(), MemRef<false>(e.prm.swT), &e.cs, ps,
                                            rows, t.cnt.data(), t.lcnt.data(), t.rc.data(), base_viol, base_obj, viol,
                                            obj, kRF ? e.rftab.data() : nullptr);
        if (e.topics) {
            int rc[2 * kMaxOps], lc[2 * kMaxOps];
            topic_events<W>(e.prm, e.ta, &e.cs, ps, rows, rc, lc);
            viol += topic_delta<W>(e.ta, rc, lc);
        }
        return pack_key(viol, obj, idx, e.prm.key_obj_bits);
    }
    // the base's (violation, objective) as the kernel hands it to delta_eval: the full pass, the violation clamped to int
    static void base_key_fields(const Totals &t, int &bv, int &bo)
    {
        bv = (int)std::min(t.viol, (long long)0x7FFFFFFF);
        bo = (int)t.obj;
    }
    static void keys(Emu &e, uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_begin, uint32_t count,
                     uint64_t *out)
    {
        const Totals t = base(e);
        int bv, bo;
        base_key_fields(t, bv, bo);
        for (uint32_t i = 0; i < count; ++i) out[i] = key(e, t, bv, bo, seed, round, idx_begin + i, round_size);
    }
    // whole rounds as search_large_kernel runs them: after a winner the base's evaluation IS the winner's key, unless
    // that key is saturated, then the next round evaluates the base in full (the totals are rebuilt here every round,
    // the kernel patches them: the same counts)
    static void search(Emu &e, uint64_t seed, uint32_t first_round, uint32_t rounds, uint32_t round_size,
                       uint64_t *round_keys)
    {
        bool from_key = false;
        int bv = 0, bo = 0;
        for (uint32_t t = 0; t < rounds; ++t) {
            const uint32_t round = first_round + t;
            const Totals tot = base(e);
            if (!from_key) base_key_fields(tot, bv, bo);
            unsigned long long best = kKeyNone;
            for (uint32_t idx = 0; idx < round_size; ++idx) best = std::min(best, key(e, tot, bv, bo, seed, round, idx, round_size));
            if (round_keys) round_keys[t] = best;
            const uint32_t kv = key_violation(best, e.prm.key_obj_bits);
            from_key = best != kKeyNone && (uint64_t)kv < key_viol_cap(e.prm.key_obj_bits);
            bv = (int)kv;
            bo = (int)key_objective(best, e.prm.key_obj_bits);
            if (best == kKeyNone) continue;
            PatchSet win;
            uint32_t rows[kMaxOps][W];
            gen(e, seed, round, (uint32_t)(best & kIdxMask), round_size, win, rows);
            if (e.topics) {                           // apply_winner_topics: the winner's events against the base
                int rc[2 * kMaxOps], lc[2 * kMaxOps];
                topic_events<W>(e.prm, e.ta, &e.cs, win, rows, rc, lc);
                topic_apply_events<W>(e.ta, rc, lc);
            }
            for (int i = 0; i < win.n; ++i) {
                for (int w = 0; w < W; ++w) e.bits[(size_t)w * e.hm.Ppad + win.p[i]] = rows[i][w];
                e.leader[win.p[i]] = (uint8_t)win.ld[i];
            }
            rebuild_lists(e);
        }
    }
};

template <bool kRF, class F> auto with_w_rf(const Emu &e, F f)
{
    switch (e.hm.W) {
    case 1: return f(RunLarge<1, kRF>{});
    case 2: return f(RunLarge<2, kRF>{});
    case 4: return f(RunLarge<4, kRF>{});
    default: return f(RunLarge<8, kRF>{});
    }
}

template <class F> auto with_w(const Emu &e, F f) { return e.rf ? with_w_rf<true>(e, f) : with_w_rf<false>(e, f); }

// the device-side tables and Params of a session whose host model and evaluator configuration are set; its initial base
void start(Emu &e)
{
    const HostModel &m = e.hm;
    e.nW = t_words(m.Ppad);
    fill_consts(m, e.cs);
    Params &p = e.prm;
    p.P = m.P; p.Ppad = m.Ppad; p.B = m.B; p.R = m.R; p.RF = m.RF; p.NS = m.NS; p.log2S = m.log2S;
    set_rf_masks(p);
    p.key_obj_bits = m.key_obj_bits;
    p.ppr_lo = m.ppr_lo; p.ppr_hi = m.ppr_hi; p.dense = m.dense ? 1 : 0;
    p.nentries = m.nentries; p.nplanes = m.nplanes; p.plane_on_leader = m.plane_on_leader;
    for (int c = 0; c < 6; ++c) p.plane_value[c] = m.plane_value[c];
    p.swT = m.swT.data();
    p.planesT = m.nplanes > 0 ? m.planesT.data() : nullptr;
    p.dense_w = m.dense ? m.dense_w.data() : nullptr;
    p.homeT = m.homeT.data();
    p.nz = m.z_ok ? m.nz : 0; p.z_on_leader = m.z_on_leader; p.zslot = m.z_ok ? m.zslot.data() : nullptr;
    for (int j = 0; j < 8; ++j) p.z_value[j] = m.z_value[j];
    p.consts = &e.cs;
    e.D.assign(m.Ppad, 0);
    e.DL.assign(m.Ppad, 0);
    e.prow.assign((size_t)kMaxOps * m.W, 0);
    std::vector<uint32_t> bitsT;
    std::vector<uint8_t> leader;
    initial_base(m, bitsT, leader);
    set_base(e, bitsT, leader);
}

thread_local std::string g_err;

}  // namespace

extern "C" {

const char *kao_emu_last_error(void) { return g_err.c_str(); }

void *kao_emu_create(const kao_problem *pb)
{
    auto e = std::make_unique<Emu>();
    if (!build_host_model(*pb, e->hm, g_err)) return nullptr;
    HostModel &m = e->hm;
    // kao_create: do mask planes + one-hot plane fit next to the base, else packed entries
    const int threads = m.W <= 2 ? 768 : 256;
    SmemPlan plan = make_plan(m.W, m.Ppad, threads / 32, m.nplanes > 0 ? m.nplanes * m.W : 4, m.P, m.RF, m.nplanes > 0);
    if (plan.total > 227u * 1024u && m.nplanes > 0) {
        m.nplanes = 0;
        plan = make_plan(m.W, m.Ppad, threads / 32, 4, m.P, m.RF, false);
    }
    if (plan.total > 227u * 1024u) { g_err = "problem too large for the shared-memory resident search kernel"; return nullptr; }
    e->nph = counter_nph(m.Ppad);                     // counter depth (kao_engine.cu: dispatch)
    e->rack = !m.hi1 ? 0 : (m.log2S == 3 ? 3 : (m.log2S == 4 ? 4 : 5));
    e->obj = (m.W <= 2 && m.nplanes == 3) ? 3 : 0;
    e->oh = m.W <= 2 && e->obj > 0;
    // kao_set_evaluator: the column-major evaluator covers 8-slot rack fields with C7 = "at most one
    // replica per rack" and an objective of up to eight term planes
    e->trans_ok = m.W <= 2 && m.hi1 && m.log2S == 3 && m.z_ok && column_major_fits(m.W, m.Ppad, 1024, m.P, m.RF);
    start(*e);
    return e.release();
}

// kao_create_replication: the host model with every row's C1 / C7 operands, always on the HBM-base path (no
// shared-memory plan; objective from packed entries or the dense table; general rack form whatever hi1 says)
void *kao_emu_create_replication(const kao_problem *pb, const kao_replication *rp)
{
    auto e = std::make_unique<Emu>();
    if (!build_host_model(*pb, e->hm, g_err) || !build_host_replication(*rp, e->hm, g_err)) return nullptr;
    e->hm.nplanes = 0;
    e->hm.z_ok = false;
    e->rf = true;
    e->rftab = replication_table(e->hm);
    e->nph = 5; e->rack = 0; e->obj = kObjEntries;
    start(*e);
    return e.release();
}

// kao_create_topics: a plain host model with topic rows, on the HBM-base path like a replication session; the rows as
// build_host_topics checks them, the session's TopicArgs on the emulator's own tables
void *kao_emu_create_topics(const kao_problem *pb, const kao_topics *tp)
{
    auto e = std::make_unique<Emu>();
    if (!build_host_model(*pb, e->hm, g_err) || !build_host_topics(*pb, *tp, e->hm.Ppad, e->ht, g_err))
        return nullptr;
    e->hm.nplanes = 0;
    e->hm.z_ok = false;
    e->topics = true;
    e->tbnd.resize(e->ht.T);
    for (int t = 0; t < e->ht.T; ++t)
        e->tbnd[t] = make_int4(e->ht.bnd[4 * t], e->ht.bnd[4 * t + 1], e->ht.bnd[4 * t + 2], e->ht.bnd[4 * t + 3]);
    e->ta.T = e->ht.T;
    e->ta.topic_of = e->ht.topic_of.data();
    e->ta.bnd = e->tbnd.data();
    e->ta.tviol = &e->tviol;
    e->nph = 5; e->rack = 0; e->obj = kObjEntries;
    start(*e);
    return e.release();
}

int kao_emu_set_evaluator(void *h, int32_t mode)
{
    Emu &e = *static_cast<Emu *>(h);
    if (mode != 0 && !e.trans_ok) { g_err = "column-major evaluator: unsupported layout"; return -1; }
    if (mode < 0 || mode > 6) { g_err = "unknown evaluator form"; return -1; }
    e.trans = mode;
    return 0;
}

void kao_emu_destroy(void *h) { delete static_cast<Emu *>(h); }

// rows the column-major evaluator charged one by one (its slow, exact path) since the last call
long long kao_emu_rows_charged_one_by_one(void)
{
    const long long n = emu_rows_charged_one_by_one;
    emu_rows_charged_one_by_one = 0;
    return n;
}

// 5 ints: words per row, counter planes above the fours (NPH), rack form, objective planes, dense weight table
void kao_emu_config(void *h, int32_t *out)
{
    Emu &e = *static_cast<Emu *>(h);
    out[0] = e.hm.W; out[1] = e.nph; out[2] = e.rack; out[3] = e.obj; out[4] = e.prm.dense;
}

// the evaluator configurations dispatch instantiates, 4 ints each as kao_emu_config; returns their number
int kao_emu_dispatch_configs(int32_t *out, int32_t cap)
{
    int n = 0;
#define KAO_EMU_LIST(W_, NPH_, R_, O_)                                                        \
    if (n < cap) { out[4 * n] = W_; out[4 * n + 1] = NPH_; out[4 * n + 2] = R_; out[4 * n + 3] = O_; } \
    ++n;
    KAO_EMU_CFGS(KAO_EMU_LIST)
#undef KAO_EMU_LIST
    return n;
}

void kao_emu_set_base(void *h, const int32_t *replicas)
{
    Emu &e = *static_cast<Emu *>(h);
    std::vector<uint32_t> bitsT;
    std::vector<uint8_t> leader;
    encode_replicas(e.hm, replicas, bitsT, leader);
    set_base(e, bitsT, leader);
}

// replica lists of the base and its evaluation as the identity candidate of the search evaluator
void kao_emu_get_base(void *h, int32_t *replicas, int64_t *violation, int64_t *objective, int32_t *moves)
{
    Emu &e = *static_cast<Emu *>(h);
    std::vector<uint32_t> bitsT(e.bits.begin(), e.bits.begin() + (size_t)e.hm.W * e.hm.Ppad);
    decode_replicas(e.hm, bitsT, e.leader, replicas);
    if (moves) *moves = count_moves(e.hm, replicas);
    if (e.rf || e.topics) {                     // eval_large_base_kernel<W, kRF>: the raw violation (tviol added)
        with_w(e, [&](auto r) {
            const auto t = decltype(r)::base(e);
            if (violation) *violation = t.viol;
            if (objective) *objective = t.obj;
            return 0;
        });
        return;
    }
    // idx + 1 == round_size is the identity candidate (docs/MODEL.md §5)
    const unsigned long long k = dispatch(e, [&](auto r) { return decltype(r)::key(e, 0, 0, 1, 2); });
    if (violation) *violation = (int64_t)key_violation(k, e.prm.key_obj_bits);
    if (objective) *objective = (int64_t)key_objective(k, e.prm.key_obj_bits);
}

void kao_emu_candidate_keys(void *h, uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_begin,
                            uint32_t count, uint64_t *keys)
{
    Emu &e = *static_cast<Emu *>(h);
    dispatch(e, [&](auto r) {
        for (uint32_t i = 0; i < count; ++i) keys[i] = decltype(r)::key(e, seed, round, idx_begin + i, round_size);
        return 0;
    });
}

// whole rounds: argmin of the keys, the winner becomes the base (kao_search, one GPU, no early stop)
void kao_emu_search(void *h, uint64_t seed, uint32_t first_round, uint32_t rounds, uint32_t round_size, uint64_t *round_keys)
{
    Emu &e = *static_cast<Emu *>(h);
    if (e.rf || e.topics) {
        with_w(e, [&](auto r) { decltype(r)::search(e, seed, first_round, rounds, round_size, round_keys); return 0; });
        return;
    }
    dispatch(e, [&](auto r) {
        for (uint32_t t = 0; t < rounds; ++t) {
            unsigned long long best = kKeyNone;
            for (uint32_t idx = 0; idx < round_size; ++idx) best = std::min(best, decltype(r)::key(e, seed, first_round + t, idx, round_size));
            if (round_keys) round_keys[t] = best;
            if (best != kKeyNone) decltype(r)::apply(e, seed, first_round + t, (uint32_t)(best & kIdxMask), round_size);
        }
        return 0;
    });
}

// delta mode keys (rows of up to 64 slots): totals of the base as the kernel builds them per round
int kao_emu_candidate_keys_delta(void *h, uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_begin,
                                 uint32_t count, uint64_t *keys)
{
    Emu &e = *static_cast<Emu *>(h);
    if (e.rf || e.topics) {
        with_w(e, [&](auto r) { decltype(r)::keys(e, seed, round, round_size, idx_begin, count, keys); return 0; });
        return 0;
    }
    const HostModel &m = e.hm;
    std::vector<int> cnt(256, 0), lcnt(256, 0), rc(32 + 4, 0);
    for (int p = 0; p < m.P; ++p) {
        const int ld = e.leader[p];
        bool ok = false;
        for (int w = 0; w < m.W; ++w) {
            const uint32_t xw = e.bits[(size_t)w * m.Ppad + p];
            for (uint32_t b = xw; b; b &= b - 1) {
                const int sl = w * 32 + __ffs(b) - 1;
                ++cnt[sl];
                ++rc[sl >> m.log2S];
            }
            if ((ld >> 5) == w) ok = (xw >> (ld & 31)) & 1u;
        }
        if (ok) ++lcnt[ld];
    }
    // seeded with the base's raw evaluation, as the kernel's full pass of a first round: the base's packed key
    // would hand over the field's cap instead of a saturated violation
    dispatch(e, [&](auto r) {
        int bv, bo;
        decltype(r)::base_eval(e, bv, bo);
        for (uint32_t i = 0; i < count; ++i)
            keys[i] = decltype(r)::key_delta(e, seed, round, idx_begin + i, round_size, cnt.data(), lcnt.data(), rc.data(), bv, bo);
        return 0;
    });
    return 0;
}

// The state a search patches winner by winner (transposed and term planes with t_patch_row, the one-hot plane, the
// count of invalid leaders that decides t_leaders_valid, the displaced lists) against the same state rebuilt from the
// current bits / leader with the builders set_base uses.  0: equal; else the first array that differs (1 transposed
// planes, 2 term / rack-field planes, 3 one-hot plane, 4 count of invalid leaders, 5 list lengths, 6 D, 7 DL), its
// index in *at, a message in kao_emu_last_error.  The session keeps its patched state either way.
int kao_emu_check_state(void *h, int64_t *at)
{
    Emu &e = *static_cast<Emu *>(h);
    long long i = -1;
    int rc = 0;
    if (e.trans_ok && !e.rf) {
        std::vector<uint32_t> T = e.T, Z = e.Z;
        if (e.hm.W == 1) build_T<1>(e); else build_T<2>(e);
        const long long dt = first_diff(T, e.T), dz = first_diff(Z, e.Z);
        e.T.swap(T);
        e.Z.swap(Z);
        if (dt >= 0) rc = check_state_msg(1, "transposed planes", dt, &i, g_err);
        else if (dz >= 0) rc = check_state_msg(2, "term / rack-field planes", dz, &i, g_err);
    }
    if (rc == 0) rc = check_base_state(e, &i, g_err);
    *at = i;
    return rc;
}

// explicit candidates (kao_eval / eval_batch_kernel): replicas [n][P*RF]
void kao_emu_eval(void *h, const int32_t *replicas, int32_t n, int64_t *violation, int64_t *objective)
{
    Emu &e = *static_cast<Emu *>(h);
    const HostModel &m = e.hm;
    for (int i = 0; i < n; ++i) {
        std::vector<uint32_t> cb;
        std::vector<uint8_t> cl;
        encode_replicas(m, replicas + (size_t)i * m.P * m.RF, cb, cl);
        long long v = 0, o = 0;
        switch (m.W) {                      // counter depth 6: only one-word rows of 8192 padded rows get past kao_emu_create
        case 1: if (e.nph == 6) eval_explicit<1, 6>(e, cb.data(), cl.data(), v, o);
                else eval_explicit<1, 5>(e, cb.data(), cl.data(), v, o);
                break;
        case 2: eval_explicit<2, 5>(e, cb.data(), cl.data(), v, o); break;
        case 4: eval_explicit<4, 5>(e, cb.data(), cl.data(), v, o); break;
        default: eval_explicit<8, 5>(e, cb.data(), cl.data(), v, o); break;
        }
        violation[i] = v;
        objective[i] = o;
    }
}

}  // extern "C"

#include "tensor_core.cpp"
#include "reduce_fixed.cpp"
