// kao_engine.cu — kernels, device session and the C ABI (include/kao.h) of libkao.so.
//
// Replaces the reference's "emit the LP of README.md:139-185, run lp_solve, read the binaries
// back" step (/root/reference/README.md:135-136) with a GPU candidate search over the same model.
// There is no CPU fallback: every entry point fails with KAO_E_CUDA when no device is usable.
#include "kao_kernels.cuh"
#include "kao_host.hpp"
#include "kao_bound.hpp"
#include "kao_lagrange.hpp"
#include "kao_large.hpp"
#include "kao_leaders.hpp"
#include "../../include/kao.h"

#include <chrono>
#include <condition_variable>
#include <map>
#include <mutex>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

// The search kernels are instantiated in kao_inst.cu (one object per row width / counter depth /
// evaluation mode); here they are only declared.
#define KAO_DECL_FULL(W, NPH, R, O)                                             \
    extern template __global__ void KAO_ROUND_KERNEL(W, NPH, R, O);            \
    extern template __global__ void KAO_PERSISTENT_KERNEL(W, NPH, R, O, threads_for<W>(), false);
#define KAO_DECL_DELTA(W, NPH, R, O) extern template __global__ void KAO_PERSISTENT_KERNEL(W, NPH, R, O, KAO_THREADS_DELTA, true);
KAO_FOR_CFGS_NARROW(KAO_DECL_FULL, 1, 5) KAO_FOR_CFGS_NARROW(KAO_DECL_FULL, 2, 5)
KAO_FOR_CFGS_WIDE(KAO_DECL_FULL, 4, 5) KAO_FOR_CFGS_WIDE(KAO_DECL_FULL, 8, 5)
KAO_FOR_CFGS_NARROW(KAO_DECL_DELTA, 1, 5) KAO_FOR_CFGS_NARROW(KAO_DECL_DELTA, 2, 5)
KAO_FOR_CFGS_WIDE(KAO_DECL_DELTA, 4, 5) KAO_FOR_CFGS_WIDE(KAO_DECL_DELTA, 8, 5)
// the deeper column counters of 8192 padded rows (counter_nph): only one-word rows fit shared memory there
KAO_FOR_CFGS_NARROW(KAO_DECL_FULL, 1, 6) KAO_FOR_CFGS_NARROW(KAO_DECL_DELTA, 1, 6)
// column-major evaluator (kao_device_t.cuh), every built schedule
#define KAO_DECL_T(S, POP, T)                                                  \
    extern template __global__ void KAO_PERSISTENT_KERNEL_T(1, 0, S, POP, T);  \
    extern template __global__ void KAO_PERSISTENT_KERNEL_T(1, 32, S, POP, T); \
    extern template __global__ void KAO_PERSISTENT_KERNEL_T(2, 0, S, POP, T);  \
    extern template __global__ void KAO_PERSISTENT_KERNEL_T(2, 32, S, POP, T);
KAO_FOR_SCHEDULES(KAO_DECL_T)


// Winner of a round becomes the base: re-materialise its patches from (seed, round, index), write
// the patched rows to the base in HBM, then rebuild the displaced list D.  One block.
template <int W>
__global__ void __launch_bounds__(1024, 1)
apply_winner_kernel(Params d, uint64_t seed, uint32_t round, uint32_t round_size,
                    const unsigned long long *key, int regen_only)
{
    __shared__ uint32_t s_prow[kMaxOps * W];
    __shared__ int s_scan[72];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (warp == 0 && !regen_only) {
        const unsigned long long k = *key;
        if (k != kKeyNone) {
            Gen<W> gen;
            uint32_t no_rows[kMaxOps][W];
            gen.bitsT = d.bitsT; gen.leader = d.leader; gen.cs = d.consts; gen.d = &d;
            gen.prow = s_prow; gen.lane = lane;
            gen.D = d.D; gen.DL = d.DL; gen.nD = d.nD[0]; gen.nL = d.nD[1];
            PatchSet ps;
            gen.run(seed, round, (uint32_t)(k & kIdxMask), round_size, ps, no_rows);
            __syncwarp();
            if (lane == 0) {
#pragma unroll
                for (int i = 0; i < kMaxOps; ++i) {
                    if (i < ps.n) {
                        for (int t = 0; t < W; ++t) d.bitsT[(size_t)t * d.Ppad + ps.p[i]] = s_prow[i * W + t];
                        d.leader[ps.p[i]] = (uint8_t)ps.ld[i];
                    }
                }
            }
        }
    }
    __threadfence_block();
    __syncthreads();
    rebuild_lists<W, 1024>(d.bitsT, d.leader, d.homeT, d.P, d.Ppad, d.D, d.DL, d.nD, s_scan);
}

__global__ void fill_u64_kernel(unsigned long long *p, unsigned long long v, size_t n)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}

// Explicit population: one warp per candidate, rows read straight from HBM (coalesced 128-bit
// loads), same evaluator.  cand_bits [n][W][Ppad], cand_leader [n][Ppad].
template <int W, int NPH>
__global__ void __launch_bounds__(256)
eval_batch_kernel(Params d, const uint32_t *cand_bits, const uint8_t *cand_leader, int n,
                  long long *viol_out, long long *obj_out)
{
    const int lane = threadIdx.x & 31;
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= n) return;
    PatchSet ps;
    ps.n = 0;
#pragma unroll
    for (int i = 0; i < kMaxOps; ++i) { ps.p[i] = -1; ps.ld[i] = 0xFF; }
    int viol, obj;
    eval_candidate<EvalCfg<W, NPH, 0, kObjEntries>, false>(d, cand_bits + (size_t)w * W * d.Ppad,
                                                               cand_leader + (size_t)w * d.Ppad, d.swT, d.consts, ps,
                                                               nullptr, lane, viol, obj);
    if (lane == 0) { viol_out[w] = viol; obj_out[w] = obj; }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static int fail(int code, const std::string &msg) { g_err = msg; return code; }
static bool schedule_exists(int sync, int pop, int threads);
#define CUDA_TRY(expr)                                                                       \
    do {                                                                                     \
        cudaError_t e_ = (expr);                                                             \
        if (e_ != cudaSuccess)                                                               \
            return fail(KAO_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));     \
    } while (0)

// Nothing may cross the C ABI but a return code (include/kao.h: "never throw"): every extern "C" body
// runs inside this guard.
template <class F> static int guarded(F &&f) noexcept
{
    try {
        return f();
    } catch (const std::bad_alloc &) {
        return fail(KAO_E_ARG, "out of host memory (argument too large?)");
    } catch (const std::exception &e) {
        return fail(KAO_E_CUDA, std::string("internal error: ") + e.what());
    } catch (...) {
        return fail(KAO_E_CUDA, "internal error");
    }
}

// Device buffers are recycled across handles: kao_solve creates and destroys a session per call,
// and cudaMalloc / cudaFree (which synchronises the device) would dominate short solves.
namespace {
// Pinned host buffers (a search call's download staging) are recycled the same way: cudaMallocHost pins pages per call.
template <bool kHost> struct BufPool {
    std::mutex mu;
    std::multimap<std::pair<int, size_t>, void *> free_;
    size_t held = 0;
    cudaError_t get(int dev, void **p, size_t n)
    {
        n = (n + 255) & ~size_t(255);
        {
            std::lock_guard<std::mutex> g(mu);
            auto it = free_.find({dev, n});
            if (it != free_.end()) { *p = it->second; free_.erase(it); held -= n; return cudaSuccess; }
        }
        return kHost ? cudaMallocHost(p, n) : cudaMalloc(p, n);
    }
    void put(int dev, void *p, size_t n)
    {
        n = (n + 255) & ~size_t(255);
        std::lock_guard<std::mutex> g(mu);
        if (held + n > (size_t(1) << 30)) { kHost ? cudaFreeHost(p) : cudaFree(p); return; }
        free_.insert({{dev, n}, p});
        held += n;
    }
};
BufPool<false> g_pool;
BufPool<true> g_host_pool;

// a temporary device buffer that is freed on every path out of the scope that owns it
template <class T> struct DevTmp {
    T *p = nullptr;
    cudaError_t alloc(size_t count) { return cudaMalloc(&p, count * sizeof(T)); }
    ~DevTmp() { if (p) cudaFree(p); }
};

// every wait inside a kernel (grid barrier, peer GPUs) gives up after this much wall time and the call
// returns KAO_E_CUDA instead of hanging the GPU; KAO_WAIT_TIMEOUT_MS overrides the 20 s default
unsigned long long wait_budget_ns()
{
    static const unsigned long long ns = [] {
        double ms = 20000.0;
        if (const char *e = std::getenv("KAO_WAIT_TIMEOUT_MS")) { const double v = std::atof(e); if (v >= 1.0) ms = v; }
        return (unsigned long long)(ms * 1e6);
    }();
    return ns;
}
}  // namespace

constexpr size_t kBarBytes = 32;   // d_bar: [0] grid barrier, [1] release, [2] abort, [3] rounds run, [4..7] early-stop carry (2 x u64)

struct kao_handle {
    std::vector<std::pair<void *, size_t>> owned;   // device buffers to hand back to the pool
    std::vector<std::pair<void *, size_t>> owned_host;   // pinned host buffers to hand back to theirs
    HostModel hm;               // layout, tables, host copy of problem data
    int device = 0;
    int sms = 0;
    Params prm{};
    SmemPlan plan{};
    int threads = 0, grid = 0;
    // column-major full evaluator (kao_set_evaluator): layout supported, selected (the default wherever it
    // applies), its shared-memory plan
    bool trans_ok = false;
    int evaluator = KAO_EVAL_ROW_MAJOR;
    SmemPlan plan_t{};
    // schedule of the column-major evaluator (kao_set_schedule): column-loop form, tensor cores or popcount
    // compression per stream, threads per CTA.  Same results whatever the schedule.
    int sch_sync = KAO_SCHEDULE_DEFAULT_SYNC, sch_pop = KAO_SCHEDULE_DEFAULT_POP, sch_threads = KAO_SCHEDULE_DEFAULT_THREADS;
    // device buffers
    uint32_t *d_bits = nullptr; uint8_t *d_leader = nullptr; uint32_t *d_sw = nullptr;
    uint32_t *d_dense = nullptr; uint32_t *d_planes = nullptr; uint8_t *d_zslot = nullptr; uint32_t *d_home = nullptr; uint16_t *d_D = nullptr; uint16_t *d_DL = nullptr; int *d_nD = nullptr;
    Consts *d_consts = nullptr; unsigned long long *d_key = nullptr; unsigned long long *d_keys = nullptr;
    size_t keys_cap = 0;
    long long *d_vo = nullptr;
    unsigned int *d_bar = nullptr;          // kBarBytes, see above; the round keys d_keys follow it in the same buffer
    void *h_stage = nullptr;                // pinned host copy of d_bar and d_keys (kBarBytes + 8 * keys_cap bytes)
    // cross-GPU exchange (kao_p2p_*, kao_solve with n_gpus > 1)
    Mailbox *d_mail = nullptr;              // own mailbox (plain cudaMalloc: exported through CUDA IPC / used by peers directly)
    Mailbox *peer_mail[kMaxPeers] = {};
    Mailbox **d_mailptrs = nullptr;         // device copy of peer_mail for the kernel
    bool peer_opened[kMaxPeers] = {};       // mapped with cudaIpcOpenMemHandle (to be closed)
    bool mail_pooled = false;               // d_mail came from the buffer pool (kao_solve's gang), not from cudaMalloc
    int p2p_rank = 0, p2p_world = 1;
    uint64_t p2p_calls = 0;
    uint32_t patience = 0, last_rounds = 0;
    unsigned long long *d_lkeys = nullptr;   // kMailRounds keys, sharded search only
    // more than kSmemRowsMax partitions (kao_large.cu): the base stays in HBM, delta search only
    bool large = false;
    LargeArgs la{};
    // per-topic balance rows (kao_create_topics): always on the large path
    bool topics = false;
    TopicArgs ta{};
    // per-partition C1 / C7 rows (kao_create_replication): always on the large path, rf | ppr_lo << 8 | ppr_hi << 16
    bool rf = false;
    uint32_t *d_rftab = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    uint64_t launches = 0;
};


template <class T> static cudaError_t dalloc(kao_handle *h, T **p, size_t bytes)
{
    void *v = nullptr;
    cudaError_t e = g_pool.get(h->device, &v, bytes);
    if (e == cudaSuccess) { *p = static_cast<T *>(v); h->owned.emplace_back(v, bytes); }
    return e;
}

struct RoundArgs {
    uint64_t seed; uint32_t round, round_size, lo, hi; unsigned long long *d_key, *d_all; cudaStream_t st;
};
struct PersistArgs {
    uint64_t seed; uint32_t first_round, rounds, round_size; unsigned long long *d_keys; unsigned int *d_bar; cudaStream_t st;
    P2P pp;
    unsigned long long *all_keys;
};

static cudaError_t set_smem_attr(kao_handle *h, const void *kern, bool *done)
{
    if (!done[h->device & 63]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) return e;
        done[h->device & 63] = true;
    }
    return cudaSuccess;
}

struct LaunchRound {
    template <class Cfg> cudaError_t run(kao_handle *h, const RoundArgs &a) const
    {
        constexpr int T = threads_for<Cfg::W>();
        auto kern = search_round_kernel<Cfg, T>;
        static bool done[64] = {};
        cudaError_t e = set_smem_attr(h, reinterpret_cast<const void *>(kern), done);
        if (e != cudaSuccess) return e;
        const uint32_t n = a.hi - a.lo, warps = T / 32;
        uint32_t grid = (n + warps - 1) / warps;
        if (grid > (uint32_t)h->grid) grid = (uint32_t)h->grid;
        if (grid == 0) return cudaSuccess;
        kern<<<grid, T, h->plan.total, a.st>>>(h->prm, h->plan, a.seed, a.round, a.round_size, a.lo, a.hi, a.d_key, a.d_all);
        ++h->launches;
        return cudaGetLastError();
    }
};
template <bool kDelta> struct LaunchPersistent {
    template <class Cfg> cudaError_t run(kao_handle *h, const PersistArgs &a) const
    {
        constexpr int T = kDelta ? KAO_THREADS_DELTA : cfg_threads<Cfg>();
        auto kern = search_persistent_kernel<Cfg, T, kDelta>;
        static bool done[64] = {};
        cudaError_t e = set_smem_attr(h, reinterpret_cast<const void *>(kern), done);
        if (e != cudaSuccess) return e;
        Params prm = h->prm;
        // the column-major plan depends on the warps per CTA of the schedule (per-warp scratch) and, with sorted batches,
        // on the candidates of a CTA per round (the most any CTA takes: its warps' iterations)
        const uint32_t stride = (uint32_t)h->grid * (T / 32), share = a.pp.idx_hi - a.pp.idx_lo;
        const uint32_t cands = cfg_mma<Cfg>() ? (share + stride - 1) / stride * (T / 32) : 0;
        SmemPlan plan = Cfg::kTrans ? make_plan_t(Cfg::W, h->hm.Ppad, T, h->hm.P, h->hm.RF, cfg_mma<Cfg>(), cands)
                        : (kDelta && Cfg::W > 2) ? make_plan_delta_wide(Cfg::W, h->hm.Ppad, T, h->hm.P, h->hm.RF) : h->plan;
        if (plan.total > 227u * 1024u) return cudaErrorInvalidConfiguration;
        uint64_t seed = a.seed; uint32_t fr = a.first_round, rounds = a.rounds, rs = a.round_size;
        unsigned long long *keys = a.d_keys, *all = a.all_keys; unsigned int *bar = a.d_bar;
        P2P pp = a.pp;
        void *args[] = {&prm, &plan, &seed, &fr, &rounds, &rs, &keys, &bar, &pp, &all};
        ++h->launches;
        // cooperative launch: all CTAs are guaranteed co-resident, which the grid barrier needs
        return cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(kern), dim3(h->grid), dim3(T), args,
                                           plan.total, a.st);
    }
};

// f(std::integral_constant<int, W>{}) for the session's row width W (32-bit words per row): the one place a
// row width becomes a template argument
template <class F> static decltype(auto) with_row_width(int W, F &&f)
{
    switch (W) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    default: return f(std::integral_constant<int, 8>{});
    }
}

template <int W, int NPH, int kRack, class F, class A>
static cudaError_t dispatch_obj(kao_handle *h, const F &f, const A &a)
{
    if constexpr (W <= 2) {
        if (h->prm.nplanes == 3) return f.template run<EvalCfg<W, NPH, kRack, 3>>(h, a);
    }
    return f.template run<EvalCfg<W, NPH, kRack, kObjEntries>>(h, a);
}
// Rack form of the evaluator (kao_device.cuh, row_rack_terms): "at most one replica per rack" with
// the field width fixed at compile time (8 / 16 slots / whole words), or general bounds.
template <int W, int NPH, class F, class A>
static cudaError_t dispatch_w(kao_handle *h, const F &f, const A &a)
{
    if (!h->hm.hi1) return dispatch_obj<W, NPH, 0>(h, f, a);
    if (h->hm.log2S == 3) return dispatch_obj<W, NPH, 3>(h, f, a);
    if (h->hm.log2S == 4) return dispatch_obj<W, NPH, 4>(h, f, a);
    return dispatch_obj<W, NPH, 5>(h, f, a);
}
template <class F, class A> static cudaError_t dispatch(kao_handle *h, const F &f, const A &a)
{
    // counter depth (counter_nph): per-lane column counts up to 255, or up to 511 at 8192 padded rows
    return with_row_width(h->hm.W, [&](auto w) -> cudaError_t {
        constexpr int W = decltype(w)::value;
        if (counter_nph(h->hm.Ppad) == 5) return dispatch_w<W, 5>(h, f, a);
        if constexpr (W == 1) return dispatch_w<W, 6>(h, f, a);
        return cudaErrorInvalidConfiguration;     // wider rows of 8192 partitions do not fit shared memory (kao_create)
    });
}
// all rounds of a search in one cooperative launch, with the evaluator the session selected
static cudaError_t launch_persistent(kao_handle *h, const PersistArgs &pa, bool delta)
{
    if (h->large) {
        ++h->launches;
        return large_search(h->hm.W, h->grid, h->prm, h->la, pa.seed, pa.first_round, pa.rounds, pa.round_size, pa.d_keys,
                            pa.d_bar, pa.pp, pa.all_keys, pa.st, h->topics ? &h->ta : nullptr, h->d_rftab);
    }
    if (delta) return dispatch(h, LaunchPersistent<true>{}, pa);
    if (h->evaluator == KAO_EVAL_COLUMN_MAJOR) {
        const bool nw32 = h->hm.Ppad == 1024;                   // 32 partition words per slot: compile-time offsets
#define KAO_RUN_T(S, POP, T)                                                                                   \
    if (h->sch_sync == S && h->sch_pop == POP && h->sch_threads == T) {                                        \
        if (h->hm.W == 1) return nw32 ? LaunchPersistent<false>{}.template run<EvalCfgT<1, 32, S, POP, T>>(h, pa) \
                                      : LaunchPersistent<false>{}.template run<EvalCfgT<1, 0, S, POP, T>>(h, pa); \
        return nw32 ? LaunchPersistent<false>{}.template run<EvalCfgT<2, 32, S, POP, T>>(h, pa)                 \
                    : LaunchPersistent<false>{}.template run<EvalCfgT<2, 0, S, POP, T>>(h, pa);                 \
    }
        KAO_FOR_SCHEDULES(KAO_RUN_T)
#undef KAO_RUN_T
        return cudaErrorInvalidValue;                           // kao_set_schedule only accepts built schedules
    }
    return dispatch(h, LaunchPersistent<false>{}, pa);
}
static cudaError_t launch_round(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                                uint32_t lo, uint32_t hi, unsigned long long *d_key,
                                unsigned long long *d_all, cudaStream_t st)
{
    return dispatch(h, LaunchRound{}, RoundArgs{seed, round, round_size, lo, hi, d_key, d_all, st});
}
static cudaError_t launch_apply(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                                const unsigned long long *d_key, int regen_only, cudaStream_t st)
{
    with_row_width(h->hm.W, [&](auto w) {
        apply_winner_kernel<decltype(w)::value><<<1, 1024, 0, st>>>(h->prm, seed, round, round_size, d_key, regen_only);
    });
    ++h->launches;
    return cudaGetLastError();
}

static int upload_base(kao_handle *h, const std::vector<uint32_t> &bitsT, const std::vector<uint8_t> &leader)
{
    CUDA_TRY(cudaMemcpy(h->d_bits, bitsT.data(), bitsT.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(h->d_leader, leader.data(), leader.size(), cudaMemcpyHostToDevice));
    if (h->large) CUDA_TRY(large_prepare(h->hm.W, h->prm, h->la, 0));
    else CUDA_TRY(launch_apply(h, 0, 0, 2, h->d_key, /*regen_only=*/1, 0));
    if (h->topics) CUDA_TRY(topics_prepare(h->hm.W, h->prm, h->ta, 0));
    CUDA_TRY(cudaDeviceSynchronize());
    return KAO_OK;
}

static int destroy_impl(kao_handle *h)
{
    if (!h) return KAO_OK;
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();                   // nothing of this session may still be running on a recycled buffer
    for (auto &b : h->owned) g_pool.put(h->device, b.first, b.second);
    for (auto &b : h->owned_host) g_host_pool.put(h->device, b.first, b.second);
    for (int r = 0; r < kMaxPeers; ++r)
        if (h->peer_opened[r]) cudaIpcCloseMemHandle(h->peer_mail[r]);
    if (h->d_mail && !h->mail_pooled) cudaFree(h->d_mail);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    delete h;
    return KAO_OK;
}

// Owns a session; closing it keeps kao_last_error() on the failure that led there.
struct HandleOwner {
    kao_handle *h = nullptr;
    HandleOwner() = default;
    HandleOwner(const HandleOwner &) = delete;
    ~HandleOwner() { close(); }
    void close() { const std::string keep = g_err; destroy_impl(h); g_err = keep; h = nullptr; }
};

static int reserve_keys(kao_handle *h, uint32_t rounds);

static int reset_impl(kao_handle *h)
{
    if (!h) return fail(KAO_E_ARG, "null handle");
    CUDA_TRY(cudaSetDevice(h->device));
    std::vector<uint32_t> bitsT; std::vector<uint8_t> leader;
    initial_base(h->hm, bitsT, leader);
    return upload_base(h, bitsT, leader);
}

// the shared-memory plan of a session below kSmemRowsMax partitions: mask planes + one-hot plane next to the base when
// they fit, else packed entries / the dense table (m.nplanes = 0); false when even that exceeds an SM's 227 KB
static bool fit_smem_plan(HostModel &m, int threads, SmemPlan &plan)
{
    plan = make_plan(m.W, m.Ppad, threads / 32, m.nplanes > 0 ? m.nplanes * m.W : 4, m.P, m.RF, m.nplanes > 0);
    if (plan.total > 227u * 1024u && m.nplanes > 0) {
        m.nplanes = 0;
        plan = make_plan(m.W, m.Ppad, threads / 32, 4, m.P, m.RF, false);
    }
    return plan.total <= 227u * 1024u;
}

static int create_impl(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp, int32_t device,
                       kao_handle *h)
{
    std::string why;
    if (!build_host_model(*pb, h->hm, why)) return fail(KAO_E_ARG, why);
    if (rp && !build_host_replication(*rp, h->hm, why)) return fail(KAO_E_ARG, why);
    HostTopics ht;
    if (tp && !build_host_topics(*pb, *tp, h->hm.Ppad, ht, why, rp ? rp->rf : nullptr)) return fail(KAO_E_ARG, why);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
        return fail(KAO_E_CUDA, "no CUDA device: libkao has no CPU path");
    if (device < 0 || device >= ndev) return fail(KAO_E_ARG, "bad device ordinal");
    h->device = device;
    CUDA_TRY(cudaSetDevice(device));
    {   // cudaGetDeviceProperties costs tens of milliseconds per call; one attribute, cached per device
        static int sm_count[64] = {};
        if (!sm_count[device & 63])
            CUDA_TRY(cudaDeviceGetAttribute(&sm_count[device & 63], cudaDevAttrMultiProcessorCount, device));
        h->sms = sm_count[device & 63];
    }
    const HostModel &m = h->hm;
    const int W = m.W, Ppad = m.Ppad;
    h->topics = tp != nullptr;
    h->rf = rp != nullptr;
    h->large = m.P > kSmemRowsMax || h->topics || h->rf;
    if (h->large) {
        // the large path scores the objective from packed entries or the dense table (no shared-memory planes)
        h->hm.nplanes = 0;
        h->hm.z_ok = false;
    } else {
        h->threads = W <= 2 ? KAO_THREADS : KAO_THREADS_WIDE;
        if (!fit_smem_plan(h->hm, h->threads, h->plan))
            return fail(KAO_E_ARG, "problem too large for the shared-memory resident search kernel");
        // column-major evaluator: 8-slot rack fields, C7 = "at most one replica per rack", an objective that fits
        // eight term planes (kao_host.hpp); its two transposed planes (2 * W words per partition) and the term planes
        // take the place of the objective table.  It is the default full evaluator wherever it applies.
        h->plan_t = make_plan_t(W, Ppad, KAO_THREADS, m.P, m.RF);
        h->trans_ok = W <= 2 && m.hi1 && m.log2S == 3 && m.z_ok &&
                      column_major_fits(W, Ppad, 1024, m.P, m.RF);     // incl. the inverted lists of its per-thread generator
        if (h->trans_ok) h->evaluator = KAO_EVAL_COLUMN_MAJOR;
        if (const char *env = std::getenv("KAO_EVALUATOR"))       // "row" forces the row-major evaluator (measurements)
            if (std::strcmp(env, "row") == 0) h->evaluator = KAO_EVAL_ROW_MAJOR;
        if (const char *env = std::getenv("KAO_SCHEDULE")) {      // "sync,pop(hex),threads": measurements only, ignored if not built
            int a = 0, c = 0; unsigned b = 0;
            if (std::sscanf(env, "%d,%x,%d", &a, &b, &c) == 3 && schedule_exists(a, (int)b, c)) {
                h->sch_sync = a; h->sch_pop = (int)b; h->sch_threads = c;
            }
        }
    }
    h->grid = h->sms;
    CUDA_TRY(dalloc(h, &h->d_bits, (size_t)W * Ppad * 4));
    CUDA_TRY(dalloc(h, &h->d_leader, (size_t)Ppad));
    CUDA_TRY(dalloc(h, &h->d_sw, (size_t)4 * Ppad * 4));
    CUDA_TRY(dalloc(h, &h->d_home, m.homeT.size() * 4));
    // the large path keeps two buffers per displaced list (kao_large.hpp), its transposed planes and winner record
    const size_t nlists = h->large ? 2 : 1;
    CUDA_TRY(dalloc(h, &h->d_D, nlists * Ppad * 2));
    CUDA_TRY(dalloc(h, &h->d_DL, nlists * Ppad * 2));
    if (h->large) {
        h->la.tnW = t_words(Ppad);
        CUDA_TRY(dalloc(h, &h->la.T, (size_t)kTPlanes * 32 * W * h->la.tnW * 4));
        CUDA_TRY(dalloc(h, &h->la.rec, sizeof(LargeRecord)));
    }
    if (h->topics) {
        // topic of each partition, bounds per topic, replica and leader counts per (topic, slot), the base's violation
        TopicArgs &ta = h->ta;
        const size_t cells = (size_t)ht.T * 32 * W;
        uint16_t *topic_of = nullptr;
        int4 *bnd = nullptr;
        ta.T = ht.T;
        CUDA_TRY(dalloc(h, &topic_of, ht.topic_of.size() * 2));
        CUDA_TRY(dalloc(h, &bnd, (size_t)ht.T * sizeof(int4)));
        CUDA_TRY(dalloc(h, &ta.tcnt, cells * 2));
        CUDA_TRY(dalloc(h, &ta.tlcnt, cells * 2));
        CUDA_TRY(dalloc(h, &ta.tviol, 16));
        CUDA_TRY(cudaMemcpy(topic_of, ht.topic_of.data(), ht.topic_of.size() * 2, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(bnd, ht.bnd.data(), ht.bnd.size() * 4, cudaMemcpyHostToDevice));
        ta.topic_of = topic_of;
        ta.bnd = bnd;
    }
    if (h->rf) {
        const std::vector<uint32_t> tab = replication_table(m);
        CUDA_TRY(dalloc(h, &h->d_rftab, tab.size() * 4));
        CUDA_TRY(cudaMemcpy(h->d_rftab, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice));
    }
    CUDA_TRY(dalloc(h, &h->d_nD, 16));
    CUDA_TRY(dalloc(h, &h->d_consts, sizeof(Consts)));
    CUDA_TRY(dalloc(h, &h->d_key, 16));
    { const int rc = reserve_keys(h, 0); if (rc != KAO_OK) return rc; }
    CUDA_TRY(cudaMemset(h->d_nD, 0, 16));
    { const unsigned long long none[2] = {kKeyNone, kKeyNone}; CUDA_TRY(cudaMemcpy(h->d_key, none, 16, cudaMemcpyHostToDevice)); }
    if (m.dense) {
        CUDA_TRY(dalloc(h, &h->d_dense, m.dense_w.size() * 4));
        CUDA_TRY(cudaMemcpy(h->d_dense, m.dense_w.data(), m.dense_w.size() * 4, cudaMemcpyHostToDevice));
    }
    CUDA_TRY(cudaMemcpy(h->d_sw, m.swT.data(), m.swT.size() * 4, cudaMemcpyHostToDevice));
    if (m.nplanes > 0) {
        CUDA_TRY(dalloc(h, &h->d_planes, m.planesT.size() * 4));
        CUDA_TRY(cudaMemcpy(h->d_planes, m.planesT.data(), m.planesT.size() * 4, cudaMemcpyHostToDevice));
    }
    CUDA_TRY(cudaMemcpy(h->d_home, m.homeT.data(), m.homeT.size() * 4, cudaMemcpyHostToDevice));
    if (m.z_ok) {
        CUDA_TRY(dalloc(h, &h->d_zslot, m.zslot.size()));
        CUDA_TRY(cudaMemcpy(h->d_zslot, m.zslot.data(), m.zslot.size(), cudaMemcpyHostToDevice));
    }
    Consts cs;
    fill_consts(m, cs);
    CUDA_TRY(cudaMemcpy(h->d_consts, &cs, sizeof cs, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaEventCreate(&h->ev0));
    CUDA_TRY(cudaEventCreate(&h->ev1));
    Params &p = h->prm;
    p.P = m.P; p.Ppad = Ppad; p.B = m.B; p.R = m.R; p.RF = m.RF; p.NS = m.NS; p.log2S = m.log2S;
    set_rf_masks(p);
    p.ppr_lo = m.ppr_lo; p.ppr_hi = m.ppr_hi; p.dense = m.dense ? 1 : 0;
    p.key_obj_bits = m.key_obj_bits;
    p.nentries = m.nentries; p.nplanes = m.nplanes; p.plane_on_leader = m.plane_on_leader;
    for (int c = 0; c < 6; ++c) p.plane_value[c] = m.plane_value[c];
    p.planesT = h->d_planes;
    p.nz = m.z_ok ? m.nz : 0; p.z_on_leader = m.z_on_leader; p.zslot = h->d_zslot;
    for (int j = 0; j < 8; ++j) p.z_value[j] = m.z_value[j];
    p.bitsT = h->d_bits; p.leader = h->d_leader; p.swT = h->d_sw; p.dense_w = h->d_dense;
    p.homeT = h->d_home; p.D = h->d_D; p.DL = h->d_DL; p.nD = h->d_nD; p.consts = h->d_consts;
    return reset_impl(h);
}

static int create_handle(const kao_problem *pb, int32_t device, kao_handle **out, const kao_topics *tp = nullptr,
                         const kao_replication *rp = nullptr)
{
    if (!pb || !out) return fail(KAO_E_ARG, "null argument");
    *out = nullptr;
    HandleOwner s;
    s.h = new kao_handle();
    const int rc = create_impl(pb, tp, rp, device, s.h);
    if (rc == KAO_OK) { *out = s.h; s.h = nullptr; }
    return rc;
}

static int set_base_impl(kao_handle *h, const int32_t *replicas)
{
    if (!h || !replicas) return fail(KAO_E_ARG, "null argument");
    CUDA_TRY(cudaSetDevice(h->device));
    std::vector<uint32_t> bitsT; std::vector<uint8_t> leader;
    encode_replicas(h->hm, replicas, bitsT, leader);
    return upload_base(h, bitsT, leader);
}

static int eval_on_device(kao_handle *h, const uint32_t *d_bits, const uint8_t *d_leader, int n,
                          long long *d_viol, long long *d_obj)
{
    if (h->large) {
        CUDA_TRY(large_eval(h->hm.W, h->prm, d_bits, d_leader, n, d_viol, d_obj, 0));
        ++h->launches;
        return KAO_OK;
    }
    const int blocks = (n * 32 + 255) / 256;
    with_row_width(h->hm.W, [&](auto w) {
        constexpr int W = decltype(w)::value;
        if (counter_nph(h->hm.Ppad) == 5) eval_batch_kernel<W, 5><<<blocks, 256>>>(h->prm, d_bits, d_leader, n, d_viol, d_obj);
        else eval_batch_kernel<W, 6><<<blocks, 256>>>(h->prm, d_bits, d_leader, n, d_viol, d_obj);
    });
    ++h->launches;
    CUDA_TRY(cudaGetLastError());
    return KAO_OK;
}

static int get_base_impl(kao_handle *h, int32_t *replicas, int64_t *violation, int64_t *objective, int32_t *moves)
{
    if (!h) return fail(KAO_E_ARG, "null handle");
    CUDA_TRY(cudaSetDevice(h->device));
    const HostModel &m = h->hm;
    std::vector<uint32_t> bitsT((size_t)m.W * m.Ppad);
    std::vector<uint8_t> leader((size_t)m.Ppad);
    CUDA_TRY(cudaMemcpy(bitsT.data(), h->d_bits, bitsT.size() * 4, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(leader.data(), h->d_leader, leader.size(), cudaMemcpyDeviceToHost));
    std::vector<int32_t> reps((size_t)m.P * m.RF);
    decode_replicas(m, bitsT, leader, reps.data());
    if (replicas) std::memcpy(replicas, reps.data(), reps.size() * 4);
    if (moves) *moves = count_moves(m, reps.data());
    if (violation || objective) {
        if (!h->d_vo) CUDA_TRY(dalloc(h, &h->d_vo, 16));
        int rc = KAO_OK;
        if (h->rf || h->topics) {
            CUDA_TRY(large_eval_base(h->hm.W, h->prm, h->topics ? &h->ta : nullptr, h->d_rftab, h->d_vo, h->d_vo + 1, 0));
            ++h->launches;
        } else {
            rc = eval_on_device(h, h->d_bits, h->d_leader, 1, h->d_vo, h->d_vo + 1);
        }
        long long vo[2] = {0, 0};
        if (rc == KAO_OK && cudaMemcpy(vo, h->d_vo, 16, cudaMemcpyDeviceToHost) != cudaSuccess) rc = KAO_E_CUDA;
        if (rc != KAO_OK) return rc;
        if (violation) *violation = vo[0];
        if (objective) *objective = vo[1];
    }
    return KAO_OK;
}

// what a session of more than kSmemRowsMax partitions does not offer (kao.h): full per-candidate evaluation, the choice
// of full evaluator, and sharding one search over several GPUs
static int refuse_large(const char *what, bool topics = false, bool rf = false)
{
    if (rf)
        return fail(KAO_E_ARG, std::string(what) + ": not offered with per-partition replication factors "
                                                   "(kao_create_replication / kao_solve_replication keep the base and "
                                                   "the per-partition rows in HBM and search with delta evaluation on "
                                                   "one GPU per search, at every P)");
    if (topics)
        return fail(KAO_E_ARG, std::string(what) + ": not offered with topic rows (kao_create_topics / kao_solve_topics "
                                                   "keep the base and the per-topic counts in HBM and search with delta "
                                                   "evaluation on one GPU per search, at every P)");
    return fail(KAO_E_ARG, std::string(what) + ": not offered above 8,160 partitions (the base of those kernels is "
                                               "staged in shared memory); larger problems are searched with delta "
                                               "evaluation on one GPU per search");
}
// the build limits of the Lagrangian LP bound (docs/MODEL.md §9)
static bool lp_bound_fits(const kao_problem &pb) { return pb.P <= kSmemRowsMax && (int64_t)pb.P * pb.RF < 65536; }
static const char *kLpLimit = "the Lagrangian LP bound is built for P <= 8,160 and P * RF < 2^16 (docs/MODEL.md 9)";

static bool check_round_args(uint32_t round_size) { return round_size >= 2 && round_size <= KAO_MAX_ROUND_SIZE; }
// delta evaluation keeps the base and the per-round tables in shared memory (rows wider than 64 slots: without the objective table)
static bool delta_fits(const kao_handle *h)
{
    if (h->hm.W <= 2) return true;                              // the session's own plan (validated at kao_create)
    return make_plan_delta_wide(h->hm.W, h->hm.Ppad, KAO_THREADS_DELTA, h->hm.P, h->hm.RF).total <= 227u * 1024u;
}
// the arguments every search call checks (kao_search*, kao_candidate_keys*, kao_solve); kao_solve has no session
// yet (h == nullptr): each of its sessions checks delta evaluation again when it searches
static int check_search_args(const kao_handle *h, uint32_t rounds, uint32_t round_size, bool delta)
{
    if (h && h->large && !delta)
        return fail(KAO_E_ARG, std::string("full per-candidate evaluation is not offered ") +
                                   (h->rf ? "with per-partition replication factors"
                                          : h->topics ? "with topic rows" : "above 8,160 partitions") +
                                   ": use delta evaluation (kao_search_delta, kao_candidate_keys_delta)");
    if (rounds > KAO_MAX_ROUNDS) return fail(KAO_E_ARG, "rounds must not exceed KAO_MAX_ROUNDS (2^20) per call");
    if (!check_round_args(round_size)) return fail(KAO_E_ARG, "round_size must be 2..2^24");
    if (delta && h && !h->large && !delta_fits(h)) return fail(KAO_E_ARG, "delta evaluation: the base and its per-round tables do not fit in shared memory");
    return KAO_OK;
}

// d_bar and the round keys in one device buffer, mirrored by one pinned host buffer: a search call downloads both
// with one copy
static int reserve_keys(kao_handle *h, uint32_t rounds)
{
    if (h->keys_cap < rounds || !h->d_keys) {
        // the old buffers stay owned by the handle until destroy
        const size_t bytes = kBarBytes + (size_t)(rounds > 0 ? rounds : 1) * 8;
        CUDA_TRY(dalloc(h, &h->d_bar, bytes));
        h->d_keys = reinterpret_cast<unsigned long long *>(h->d_bar + kBarBytes / 4);
        void *v = nullptr;
        CUDA_TRY(g_host_pool.get(h->device, &v, bytes));
        h->owned_host.emplace_back(v, bytes);
        h->h_stage = v;
        h->keys_cap = rounds;
    }
    if (rounds) {
        fill_u64_kernel<<<64, 256>>>(h->d_keys, kKeyNone, (size_t)rounds);
        CUDA_TRY(cudaGetLastError());
    }
    return KAO_OK;
}

static P2P solo_p2p(kao_handle *h, uint32_t idx_lo, uint32_t idx_hi)
{
    P2P pp{};
    pp.rank = 0; pp.world = 1; pp.idx_lo = idx_lo; pp.idx_hi = idx_hi;
    pp.abort = reinterpret_cast<int *>(h->d_bar + 2);
    pp.patience = h->patience; pp.rounds_run = h->d_bar + 3;
    pp.best_in = kKeyNone; pp.stall_in = 0;
    pp.carry = reinterpret_cast<unsigned long long *>(h->d_bar + 4);
    pp.timeout_ns = wait_budget_ns();
    return pp;
}

// A search call on a session around launch_rounds(), which enqueues its (at least one) rounds into h->d_keys: event
// timing, the displaced lists in HBM rebuilt once at the end for the per-round entry points (unless the search kernel
// left them there), d_bar and the keys downloaded into h->h_stage with one copy and one synchronisation.
template <class F>
static int timed_search(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds, uint32_t round_size,
                        uint64_t *round_keys, double *device_ms, bool delta, F &&launch_rounds)
{
    CUDA_TRY(cudaSetDevice(h->device));
    h->last_rounds = 0;
    int rc = reserve_keys(h, rounds);
    if (rc != KAO_OK) return rc;
    CUDA_TRY(cudaEventRecord(h->ev0, 0));
    if (rounds) {
        if ((rc = launch_rounds()) != KAO_OK) return rc;
        // the large path and the column-major search kernels keep the displaced lists in HBM current themselves
        const bool lists_current = h->large || (!delta && h->evaluator == KAO_EVAL_COLUMN_MAJOR);
        if (!lists_current) CUDA_TRY(launch_apply(h, seed, first_round, round_size, h->d_keys, /*regen_only=*/1, 0));
        CUDA_TRY(cudaMemcpyAsync(h->h_stage, h->d_bar, kBarBytes + (round_keys ? (size_t)rounds * 8 : 0),
                                 cudaMemcpyDeviceToHost, 0));
    }
    CUDA_TRY(cudaEventRecord(h->ev1, 0));
    CUDA_TRY(cudaEventSynchronize(h->ev1));
    if (device_ms) {
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, h->ev0, h->ev1));
        *device_ms = ms;
    }
    if (round_keys && rounds)
        std::memcpy(round_keys, static_cast<const uint8_t *>(h->h_stage) + kBarBytes, (size_t)rounds * 8);
    return KAO_OK;
}

static int search_impl(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                       uint32_t round_size, uint64_t *round_keys, double *device_ms, bool delta)
{
    if (!h) return fail(KAO_E_ARG, "null handle");
    int rc = check_search_args(h, rounds, round_size, delta);
    if (rc != KAO_OK) return rc;
    rc = timed_search(h, seed, first_round, rounds, round_size, round_keys, device_ms, delta, [&]() -> int {
        // all rounds in one cooperative launch; the HBM base is kept current by CTA 0
        CUDA_TRY(cudaMemsetAsync(h->d_bar, 0, kBarBytes, 0));
        CUDA_TRY(launch_persistent(h, PersistArgs{seed, first_round, rounds, round_size, h->d_keys, h->d_bar, 0,
                                                  solo_p2p(h, 0, round_size), nullptr}, delta));
        return KAO_OK;
    });
    if (rc != KAO_OK || !rounds) return rc;
    unsigned int st[4];
    std::memcpy(st, h->h_stage, sizeof st);
    if (st[2]) return fail(KAO_E_CUDA, "search kernel timed out at a grid barrier");
    h->last_rounds = st[3];
    return KAO_OK;
}

static bool schedule_exists(int sync, int pop, int threads)
{
#define KAO_HAS_T(S, POP, T) if (sync == S && pop == POP && threads == T) return true;
    KAO_FOR_SCHEDULES(KAO_HAS_T)
#undef KAO_HAS_T
    return false;
}

static int candidate_keys_impl(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                               uint32_t idx_begin, uint32_t count, uint64_t *keys, bool delta)
{
    if (!h || !keys) return fail(KAO_E_ARG, "null argument");
    const int rc = check_search_args(h, 1, round_size, delta);
    if (rc != KAO_OK) return rc;
    if (idx_begin > round_size || count > round_size - idx_begin) return fail(KAO_E_ARG, "bad index range");
    if (count == 0) return KAO_OK;
    CUDA_TRY(cudaSetDevice(h->device));
    DevTmp<unsigned long long> all;
    CUDA_TRY(all.alloc(count));
    { const unsigned long long none = kKeyNone; CUDA_TRY(cudaMemcpy(h->d_key, &none, 8, cudaMemcpyHostToDevice)); }
    if (delta || h->evaluator == KAO_EVAL_COLUMN_MAJOR) {
        // these evaluators live in the persistent kernel only: one round, key dump, base untouched
        CUDA_TRY(cudaMemset(h->d_bar, 0, kBarBytes));
        P2P pp = solo_p2p(h, idx_begin, idx_begin + count);
        pp.patience = 0;
        CUDA_TRY(launch_persistent(h, PersistArgs{seed, round, 1, round_size, h->d_key, h->d_bar, 0, pp, all.p}, delta));
    } else {
        CUDA_TRY(launch_round(h, seed, round, round_size, idx_begin, idx_begin + count, h->d_key, all.p, 0));
    }
    CUDA_TRY(cudaMemcpy(keys, all.p, (size_t)count * 8, cudaMemcpyDeviceToHost));
    return KAO_OK;
}

// ---- cross-GPU sharded search: the 8-byte minimum of every round travels through peer-writable mailboxes
static int ensure_mailbox(kao_handle *h)
{
    if (h->d_mail) return KAO_OK;
    CUDA_TRY(cudaSetDevice(h->device));
    CUDA_TRY(cudaMalloc(&h->d_mail, sizeof(Mailbox)));
    CUDA_TRY(cudaMemset(h->d_mail, 0xFF, sizeof(Mailbox)));        // kMailEmpty everywhere
    CUDA_TRY(cudaDeviceSynchronize());
    return KAO_OK;
}
static int publish_mailboxes(kao_handle *h, int rank, int world)
{
    if (!h->d_mailptrs) CUDA_TRY(dalloc(h, &h->d_mailptrs, sizeof(Mailbox *) * kMaxPeers));
    if (!h->d_lkeys) CUDA_TRY(dalloc(h, &h->d_lkeys, (size_t)kMailRounds * 8));     // round keys of one launch
    CUDA_TRY(cudaMemcpy(h->d_mailptrs, h->peer_mail, sizeof(Mailbox *) * kMaxPeers, cudaMemcpyHostToDevice));
    h->p2p_rank = rank; h->p2p_world = world; h->p2p_calls = 0;
    return KAO_OK;
}

static int p2p_export_impl(kao_handle *h, uint8_t *handle_out)
{
    if (!h || !handle_out) return fail(KAO_E_ARG, "null argument");
    if (h->large) return refuse_large("kao_p2p_export", h->topics, h->rf);
    static_assert(sizeof(cudaIpcMemHandle_t) == KAO_IPC_HANDLE_BYTES, "ipc handle size");
    const int rc = ensure_mailbox(h);
    if (rc != KAO_OK) return rc;
    cudaIpcMemHandle_t ipc;
    CUDA_TRY(cudaIpcGetMemHandle(&ipc, h->d_mail));
    std::memcpy(handle_out, &ipc, sizeof ipc);
    return KAO_OK;
}

static int p2p_connect_impl(kao_handle *h, int32_t rank, int32_t world, const uint8_t *handles)
{
    if (!h || !handles) return fail(KAO_E_ARG, "null argument");
    if (h->large) return refuse_large("kao_p2p_connect", h->topics, h->rf);
    if (world < 1 || world > kMaxPeers || rank < 0 || rank >= world) return fail(KAO_E_ARG, "bad rank / world");
    if (!h->d_mail) return fail(KAO_E_STATE, "call kao_p2p_export first");
    CUDA_TRY(cudaSetDevice(h->device));
    for (int r = 0; r < world; ++r) {
        if (r == rank) { h->peer_mail[r] = h->d_mail; continue; }
        cudaIpcMemHandle_t ipc;
        std::memcpy(&ipc, handles + (size_t)r * KAO_IPC_HANDLE_BYTES, sizeof ipc);
        void *p = nullptr;
        CUDA_TRY(cudaIpcOpenMemHandle(&p, ipc, cudaIpcMemLazyEnablePeerAccess));
        h->peer_mail[r] = static_cast<Mailbox *>(p);
        h->peer_opened[r] = true;
    }
    return publish_mailboxes(h, rank, world);
}

static int sharded_impl(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                        uint32_t round_size, uint64_t *round_keys, double *device_ms, bool delta)
{
    if (!h) return fail(KAO_E_ARG, "null handle");
    if (h->large) return refuse_large("sharded search", h->topics, h->rf);
    const int rc = check_search_args(h, rounds, round_size, delta);
    if (rc != KAO_OK) return rc;
    if (h->p2p_world < 2 || !h->peer_mail[h->p2p_world - 1]) return fail(KAO_E_STATE, "kao_p2p_connect first");
    const int world = h->p2p_world, rank = h->p2p_rank;
    // contiguous slice of every round for this rank (same split on every rank)
    const uint32_t base = round_size / world, extra = round_size % world;
    const uint32_t lo = rank * base + ((uint32_t)rank < extra ? rank : extra);
    const uint32_t hi = lo + base + ((uint32_t)rank < extra ? 1 : 0);
    // one cooperative launch per kMailRounds rounds: the mailbox bank alternates from launch to launch
    return timed_search(h, seed, first_round, rounds, round_size, round_keys, device_ms, delta, [&]() -> int {
        unsigned long long best = kKeyNone;                         // early-stop state, carried from launch to launch
        uint32_t stall = 0;
        for (uint32_t done = 0; done < rounds; done += kMailRounds) {
            const uint32_t n = rounds - done < kMailRounds ? rounds - done : kMailRounds;
            const int bank = (int)(h->p2p_calls & 1);
            ++h->p2p_calls;
            // the OTHER bank is reset now: no peer can reach the next launch before this rank has taken
            // part in every round of this one (docs/MODEL.md §7), so the reset cannot race with a writer
            CUDA_TRY(cudaMemsetAsync(&h->d_mail->slot[bank ^ 1][0][0], 0xFF, sizeof(h->d_mail->slot[0]), 0));
            fill_u64_kernel<<<32, 256>>>(h->d_lkeys, kKeyNone, (size_t)n);
            CUDA_TRY(cudaMemsetAsync(h->d_bar, 0, kBarBytes, 0));
            h->launches += 1;
            P2P pp = solo_p2p(h, lo, hi);
            pp.rank = rank; pp.world = world; pp.bank = bank;
            pp.mail = h->d_mailptrs;
            pp.lkeys = h->d_lkeys; pp.release = h->d_bar + 1;
            pp.best_in = best; pp.stall_in = stall;
            const PersistArgs pa{seed, first_round + done, n, round_size, h->d_keys + done, h->d_bar, 0, pp, nullptr};
            CUDA_TRY(launch_persistent(h, pa, delta));
            unsigned int st[8] = {};
            CUDA_TRY(cudaMemcpy(st, h->d_bar, kBarBytes, cudaMemcpyDeviceToHost));
            if (st[2]) return fail(KAO_E_CUDA, "sharded search timed out waiting for a peer GPU");
            h->last_rounds = done + st[3];
            std::memcpy(&best, st + 4, 8);
            { unsigned long long s64; std::memcpy(&s64, st + 6, 8); stall = (uint32_t)s64; }
            if (st[3] < n) break;                                   // early stop (every rank stops at the same round)
        }
        return KAO_OK;
    });
}

static int profile_rounds_impl(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                               uint32_t round_size, double *search_ms, double *apply_ms)
{
    if (!h || !rounds || rounds > 4096) return fail(KAO_E_ARG, "bad argument (1..4096 rounds)");
    if (h->large) return refuse_large("kao_profile_rounds (full evaluation, one launch per round)", h->topics, h->rf);
    if (!check_round_args(round_size)) return fail(KAO_E_ARG, "bad round_size");
    CUDA_TRY(cudaSetDevice(h->device));
    struct Events {
        std::vector<cudaEvent_t> ev;
        ~Events() { for (auto &e : ev) if (e) cudaEventDestroy(e); }
    } evs;
    evs.ev.assign(3 * (size_t)rounds, nullptr);
    for (auto &e : evs.ev) CUDA_TRY(cudaEventCreate(&e));
    DevTmp<unsigned long long> k;
    CUDA_TRY(k.alloc(rounds));
    fill_u64_kernel<<<32, 256>>>(k.p, kKeyNone, (size_t)rounds);
    for (uint32_t t = 0; t < rounds; ++t) {
        CUDA_TRY(cudaEventRecord(evs.ev[3 * t], 0));
        CUDA_TRY(launch_round(h, seed, first_round + t, round_size, 0, round_size, k.p + t, nullptr, 0));
        CUDA_TRY(cudaEventRecord(evs.ev[3 * t + 1], 0));
        CUDA_TRY(launch_apply(h, seed, first_round + t, round_size, k.p + t, 0, 0));
        CUDA_TRY(cudaEventRecord(evs.ev[3 * t + 2], 0));
    }
    CUDA_TRY(cudaDeviceSynchronize());
    double s_ms = 0, a_ms = 0;
    for (uint32_t t = 0; t < rounds; ++t) {
        float a = 0, b = 0;
        CUDA_TRY(cudaEventElapsedTime(&a, evs.ev[3 * t], evs.ev[3 * t + 1]));
        CUDA_TRY(cudaEventElapsedTime(&b, evs.ev[3 * t + 1], evs.ev[3 * t + 2]));
        s_ms += a; a_ms += b;
    }
    if (search_ms) *search_ms = s_ms;
    if (apply_ms) *apply_ms = a_ms;
    return KAO_OK;
}

static int eval_impl(const kao_problem *pb, int32_t device, const int32_t *replicas, int32_t n,
                     int64_t *violation, int64_t *objective)
{
    if (!pb || !replicas || n < 0 || !violation || !objective) return fail(KAO_E_ARG, "bad argument");
    HandleOwner s;
    int rc = create_handle(pb, device, &s.h);
    if (rc != KAO_OK) return rc;
    kao_handle *h = s.h;
    const HostModel &m = h->hm;
    const size_t nb = (size_t)m.W * m.Ppad, nl = (size_t)m.Ppad;
    if (n == 0) return KAO_OK;
    std::vector<uint32_t> bits(nb * n), one;
    std::vector<uint8_t> lead(nl * n), onel;
    for (int i = 0; i < n; ++i) {
        encode_replicas(m, replicas + (size_t)i * m.P * m.RF, one, onel);
        std::memcpy(bits.data() + nb * i, one.data(), nb * 4);
        std::memcpy(lead.data() + nl * i, onel.data(), nl);
    }
    DevTmp<uint32_t> d_b; DevTmp<uint8_t> d_l; DevTmp<long long> d_v;
    CUDA_TRY(d_b.alloc(bits.size()));
    CUDA_TRY(d_l.alloc(lead.size()));
    CUDA_TRY(d_v.alloc((size_t)n * 2));
    CUDA_TRY(cudaMemcpy(d_b.p, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(d_l.p, lead.data(), lead.size(), cudaMemcpyHostToDevice));
    rc = eval_on_device(h, d_b.p, d_l.p, n, d_v.p, d_v.p + n);
    if (rc != KAO_OK) return rc;
    static_assert(sizeof(long long) == sizeof(int64_t), "abi");
    CUDA_TRY(cudaMemcpy(violation, d_v.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(objective, d_v.p + n, (size_t)n * 8, cudaMemcpyDeviceToHost));
    return KAO_OK;
}

// ---- kao_solve: one GPU, or the rounds sharded over several GPUs of this process
static int pick_devices(const kao_options *opt, std::vector<int> &devs)
{
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
        return fail(KAO_E_CUDA, "no CUDA device: libkao has no CPU path");
    devs.clear();
    if (opt->device_mask) {
        for (int i = 0; i < 32; ++i)
            if (opt->device_mask >> i & 1u) devs.push_back(i);
        if (opt->n_gpus > 1 && opt->n_gpus != (int)devs.size()) return fail(KAO_E_ARG, "n_gpus does not match device_mask");
    } else {
        const int n = opt->n_gpus > 1 ? opt->n_gpus : 1;
        for (int i = 0; i < n; ++i) devs.push_back(opt->device + i);
    }
    if (devs.empty() || (int)devs.size() > KAO_MAX_GPUS) return fail(KAO_E_ARG, "1..KAO_MAX_GPUS devices");
    for (int d : devs)
        if (d < 0 || d >= ndev) return fail(KAO_E_ARG, "bad device ordinal (n_gpus / device_mask exceed the visible devices)");
    return KAO_OK;
}

// ---- several GPUs of this process: one host thread per GPU does everything for its device (create, connect,
// search, destroy), so that the per-call set-up cost does not grow with the number of GPUs
namespace {
struct Rendezvous {                                   // a reusable barrier that also spreads "somebody failed"
    std::mutex mu;
    std::condition_variable cv;
    int n, waiting = 0, generation = 0;
    bool failed = false;
    explicit Rendezvous(int parties) : n(parties) {}
    bool arrive(bool ok)                              // -> false once any party has arrived with ok == false
    {
        std::unique_lock<std::mutex> lk(mu);
        failed |= !ok;
        const int gen = generation;
        if (++waiting == n) { waiting = 0; ++generation; cv.notify_all(); }
        else cv.wait(lk, [&] { return gen != generation; });
        return !failed;
    }
};
std::mutex g_peer_mu;
bool g_peer_enabled[64][64] = {};
}  // namespace

static int enable_peers(int dev, const std::vector<int> &devs)
{
    CUDA_TRY(cudaSetDevice(dev));
    for (int other : devs) {
        if (other == dev) continue;
        {
            std::lock_guard<std::mutex> g(g_peer_mu);
            if (g_peer_enabled[dev & 63][other & 63]) continue;
        }
        int can = 0;
        CUDA_TRY(cudaDeviceCanAccessPeer(&can, dev, other));
        if (!can) return fail(KAO_E_CUDA, "the selected GPUs cannot access each other's memory (no peer access)");
        const cudaError_t e = cudaDeviceEnablePeerAccess(other, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else if (e != cudaSuccess) return fail(KAO_E_CUDA, std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
        std::lock_guard<std::mutex> g(g_peer_mu);
        g_peer_enabled[dev & 63][other & 63] = true;
    }
    return KAO_OK;
}

// ---- what both kao_solve drivers (restarts, sharded rounds) share
// KAO_TRACE (stderr): where a kao_solve call spends its host time
static void stamp(std::chrono::steady_clock::time_point t0, const char *what)
{
    static const bool trace = std::getenv("KAO_TRACE") != nullptr;
    if (trace)
        std::fprintf(stderr, "[kao trace] kao_solve: %s at %.3f ms\n", what,
                     std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
}

// the kao_options flags that configure a session: KAO_FLAG_PATIENCE(n), and KAO_FLAG_ROW_MAJOR (the column-major
// evaluator is the default where the layout allows it; the flag selects the other full evaluator, same keys)
static void apply_options(kao_handle *h, const kao_options *opt)
{
    h->patience = opt->flags >> 16;
    if (opt->flags & KAO_FLAG_ROW_MAJOR) h->evaluator = KAO_EVAL_ROW_MAJOR;
}

struct Outcome {                                      // the final assignment of one restart
    int64_t viol = 0, obj = 0;
    int32_t moves = 0;
    uint32_t restart = 0;
    uint64_t key = kKeyNone;                          // its last round key
    std::vector<int32_t> reps;
};
// the restart kao_solve returns: lowest violation, then highest objective, then lowest restart index
static bool better(const Outcome &a, const Outcome &b)
{
    if (a.viol != b.viol) return a.viol < b.viol;
    if (a.obj != b.obj) return a.obj > b.obj;
    return a.restart < b.restart;
}
// the session's base after restart r, whose round keys the search wrote to keys
static int read_outcome(kao_handle *h, uint32_t r, const std::vector<uint64_t> &keys, Outcome &o)
{
    o.reps.resize((size_t)h->hm.P * h->hm.RF);
    o.restart = r;
    o.key = h->last_rounds ? keys[h->last_rounds - 1] : kKeyNone;
    return get_base_impl(h, o.reps.data(), &o.viol, &o.obj, &o.moves);
}
struct Solved {                                       // what a kao_solve driver hands back
    Outcome win;
    uint32_t rounds_run = 0;                          // summed over the restarts
    double dev_ms = 0;                                // summed over the restarts of a GPU, max over the GPUs
    HostModel hm;                                     // GPU 0's
};
// worker(i) for each GPU of the call, GPU 0 on the calling thread and one host thread for every other; a failure is
// reported with its GPU named when there are several
template <class F> static int on_each_gpu(const std::vector<int> &devs, F &&worker)
{
    const int world = (int)devs.size();
    std::vector<int> rcs(world, KAO_OK);
    std::vector<std::string> errs(world);
    auto run = [&](int i) {
        rcs[i] = guarded([&] { return worker(i); });
        if (rcs[i] != KAO_OK) errs[i] = g_err;
    };
    std::vector<std::thread> th;
    for (int i = 1; i < world; ++i) th.emplace_back(run, i);
    run(0);
    for (auto &t : th) t.join();
    for (int i = 0; i < world; ++i)
        if (rcs[i] != KAO_OK) return fail(rcs[i], world > 1 ? "GPU " + std::to_string(devs[i]) + ": " + errs[i] : errs[i]);
    return KAO_OK;
}

// The rounds of every restart sharded over the GPUs: every round's index range is split between them and its winner
// agreed through the mailboxes, so all GPUs hold the same base.
static int solve_gang(const kao_problem *pb, const kao_options *opt, const std::vector<int> &devs, uint32_t restarts,
                      bool delta, Solved &out)
{
    const int world = (int)devs.size();
    std::vector<kao_handle *> hs(world, nullptr);
    std::vector<double> ms(world, 0.0);
    std::vector<uint64_t> keys(opt->rounds ? opt->rounds : 1, kKeyNone);
    Rendezvous meet(world);
    static const bool trace = std::getenv("KAO_TRACE") != nullptr;       // stderr: where a multi-GPU solve spends its host time
    const auto t_start = std::chrono::steady_clock::now();
    return on_each_gpu(devs, [&](int i) {
        int phase = 0, first = KAO_OK;                // this rank's first failure
        std::string err;
        auto step = [&](int rc) {                     // record the first failure of this rank, then meet the others
            if (rc != KAO_OK && first == KAO_OK) { first = rc; err = g_err; }
            const auto t_a = std::chrono::steady_clock::now();
            const bool all_ok = meet.arrive(rc == KAO_OK);
            if (trace) {
                const auto t_b = std::chrono::steady_clock::now();
                std::fprintf(stderr, "[kao trace] gpu %d phase %d: reached at %.3f ms, waited %.3f ms for the others\n", devs[i], phase,
                             std::chrono::duration<double, std::milli>(t_a - t_start).count(),
                             std::chrono::duration<double, std::milli>(t_b - t_a).count());
            }
            ++phase;
            return all_ok;
        };
        HandleOwner s;
        bool ok = step(guarded([&] { return create_handle(pb, devs[i], &s.h); }));
        kao_handle *h = s.h;
        hs[i] = h;
        if (ok) ok = step(guarded([&] {
            int rc = enable_peers(devs[i], devs);
            if (rc != KAO_OK) return rc;
            CUDA_TRY(dalloc(h, &h->d_mail, sizeof(Mailbox)));          // recycled: no cudaMalloc / cudaFree per solve
            h->mail_pooled = true;
            CUDA_TRY(cudaMemsetAsync(h->d_mail, 0xFF, sizeof(Mailbox), 0));   // kMailEmpty everywhere, before any peer can write
            CUDA_TRY(cudaStreamSynchronize(0));
            apply_options(h, opt);
            return KAO_OK;
        }));
        if (ok) ok = step(guarded([&] {
            for (int j = 0; j < world; ++j) h->peer_mail[j] = hs[j]->d_mail;    // unified addressing: a peer's pointer is valid here
            return publish_mailboxes(h, i, world);
        }));
        Outcome cur;
        for (uint32_t r = 0; ok && r < restarts; ++r) {
            const uint64_t seed = opt->seed + 0x9E3779B97F4A7C15ull * r;
            ok = step(guarded([&] {
                int rc = r ? reset_impl(h) : KAO_OK;
                if (rc == KAO_OK) rc = sharded_impl(h, seed, 0, opt->rounds, opt->round_size, i == 0 ? keys.data() : nullptr, &ms[i], delta);
                return rc;
            }));
            if (ok && i == 0) {                       // all ranks hold the same base: rank 0 reports it
                const int rc = guarded([&] {
                    const int rc = read_outcome(h, r, keys, cur);
                    if (rc != KAO_OK) return rc;
                    double dev_ms = 0;
                    for (int j = 0; j < world; ++j) dev_ms = ms[j] > dev_ms ? ms[j] : dev_ms;
                    out.dev_ms += dev_ms;
                    out.rounds_run += h->last_rounds;
                    if (r == 0 || better(cur, out.win)) out.win = cur;
                    return KAO_OK;
                });
                if (rc != KAO_OK) { first = rc; err = g_err; }
            }
            if (ok) ok = meet.arrive(first == KAO_OK);   // nobody resets the base while rank 0 reads it
        }
        if (i == 0 && h) out.hm = h->hm;
        s.close();
        if (trace)
            std::fprintf(stderr, "[kao trace] gpu %d destroyed at %.3f ms\n", devs[i],
                         std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_start).count());
        return first == KAO_OK ? KAO_OK : fail(first, err);
    });
}

// The restarts side by side on the GPUs of the call: restart r runs on GPU r mod N as an ordinary single-GPU search
// (no exchange between the GPUs at all), one host thread per GPU and none for one GPU.  The winner is exactly what
// one GPU returns for the same call: this is kao_solve on one GPU, and with KAO_FLAG_SPREAD_RESTARTS on several.
static int solve_restarts(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp, const kao_options *opt,
                          const std::vector<int> &devs, uint32_t restarts, bool delta,
                          std::chrono::steady_clock::time_point t0, Solved &out)
{
    const int world = (int)devs.size();
    std::vector<Solved> per(world);
    const int rc = on_each_gpu(devs, [&](int i) {
        Solved &g = per[i];
        HandleOwner s;
        int rc = create_handle(pb, devs[i], &s.h, tp, rp);
        if (rc != KAO_OK) return rc;
        stamp(t0, "session created (model built, tables uploaded, initial base)");
        kao_handle *h = s.h;
        apply_options(h, opt);
        if (i == 0) g.hm = h->hm;
        std::vector<uint64_t> keys(opt->rounds ? opt->rounds : 1, kKeyNone);
        Outcome cur;
        for (uint32_t r = (uint32_t)i; r < restarts; r += (uint32_t)world) {
            double dev_ms = 0;
            if (r != (uint32_t)i && (rc = reset_impl(h)) != KAO_OK) return rc;
            rc = search_impl(h, opt->seed + 0x9E3779B97F4A7C15ull * r, 0, opt->rounds, opt->round_size, keys.data(), &dev_ms, delta);
            if (rc != KAO_OK) return rc;
            stamp(t0, "search done");
            if ((rc = read_outcome(h, r, keys, cur)) != KAO_OK) return rc;
            stamp(t0, "result downloaded and evaluated");
            g.dev_ms += dev_ms;
            g.rounds_run += h->last_rounds;
            if (r == (uint32_t)i || better(cur, g.win)) g.win = cur;
        }
        return KAO_OK;
    });
    if (rc != KAO_OK) return rc;
    out = std::move(per[0]);
    for (int i = 1; i < world && (uint32_t)i < restarts; ++i) {     // a GPU past the number of restarts ran none
        out.rounds_run += per[i].rounds_run;
        out.dev_ms = per[i].dev_ms > out.dev_ms ? per[i].dev_ms : out.dev_ms;
        if (better(per[i].win, out.win)) out.win = std::move(per[i].win);
    }
    return KAO_OK;
}

static int solve_impl(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp, const kao_options *opt,
                      kao_result *res)
{
    if (!pb || !opt || !res || !res->replicas) return fail(KAO_E_ARG, "null argument");
    int rc = check_search_args(nullptr, opt->rounds, opt->round_size, false);
    if (rc != KAO_OK) return rc;
    if (tp || rp) {
        // the topic and replication rows are checked before any CUDA call (each session builds them again)
        HostModel m;
        HostTopics ht;
        std::string why;
        if (!build_host_model(*pb, m, why) || (rp && !build_host_replication(*rp, m, why)) ||
            (tp && !build_host_topics(*pb, *tp, m.Ppad, ht, why, rp ? rp->rf : nullptr)))
            return fail(KAO_E_ARG, why);
    }
    if (rp && (opt->flags & KAO_FLAG_LP_BOUND))
        return fail(KAO_E_ARG, "KAO_FLAG_LP_BOUND: the Lagrangian LP bound is built for one RF and one C7 row for every "
                               "partition (docs/MODEL.md 9), not for per-partition replication factors");
    // more than kSmemRowsMax partitions, topic rows or replication rows: the large path, which searches with delta
    // evaluation (kao_solve returns the assignment, whatever evaluator found it) on one GPU per search; refused before
    // anything is searched
    const bool large = pb->P > kSmemRowsMax || tp || rp;
    const bool sharded = (opt->n_gpus > 1 || __builtin_popcount(opt->device_mask) > 1) && !(opt->flags & KAO_FLAG_SPREAD_RESTARTS);
    if (large && (opt->flags & KAO_FLAG_ROW_MAJOR)) return refuse_large("KAO_FLAG_ROW_MAJOR", tp, rp);
    if (large && sharded) return refuse_large("n_gpus > 1 without KAO_FLAG_SPREAD_RESTARTS (every round sharded over the GPUs)", tp, rp);
    if ((opt->flags & KAO_FLAG_LP_BOUND) && !lp_bound_fits(*pb)) return fail(KAO_E_ARG, std::string("KAO_FLAG_LP_BOUND: ") + kLpLimit);
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<int> devs;
    rc = pick_devices(opt, devs);
    if (rc != KAO_OK) return rc;
    const int world = (int)devs.size();
    // independent restarts (flags & 0xFF, 0 and 1 both mean a single search): each restarts from the
    // initial base with its own seed; the best final assignment wins (better())
    const uint32_t restarts = (opt->flags & 0xFFu) ? (opt->flags & 0xFFu) : 1u;
    const bool delta = (opt->flags & KAO_FLAG_DELTA) != 0 || large;
    Solved s;
    rc = world > 1 && !(opt->flags & KAO_FLAG_SPREAD_RESTARTS) ? solve_gang(pb, opt, devs, restarts, delta, s)
                                                                : solve_restarts(pb, tp, rp, opt, devs, restarts, delta, t0, s);
    if (rc != KAO_OK) return rc;
    stamp(t0, "session destroyed");
    std::memcpy(res->replicas, s.win.reps.data(), s.win.reps.size() * 4);
    res->violation = s.win.viol; res->objective = s.win.obj; res->moves = s.win.moves; res->key = s.win.key;
    res->feasible = res->violation == 0;
    res->n_candidates = (uint64_t)s.rounds_run * opt->round_size;
    res->rounds_run = s.rounds_run;
    res->restarts = restarts;
    res->device_ms = s.dev_ms;
    res->objective_bound = objective_upper_bound(s.hm, *pb);
    if ((opt->flags & KAO_FLAG_BOUND) && res->feasible)
        res->objective_bound = objective_flow_bound(s.hm, *pb, res->replicas, res->objective_bound);
    if ((opt->flags & KAO_FLAG_LP_BOUND) && res->feasible) {
        // the Lagrangian LP bound aimed at the returned objective (MODEL §9), on the first GPU of the call
        int64_t lp = 0;
        uint32_t its = 0;
        std::string why;
        rc = lagrange_bound_device(*pb, devs[0], res->objective, KAO_LP_ITERATIONS, wait_budget_ns(), &lp, &its, nullptr, nullptr, why);
        if (rc != KAO_OK) return fail(rc, why);
        res->objective_bound = std::min(res->objective_bound, lp);
        stamp(t0, "LP bound computed");
    }
    res->optimal = res->feasible && res->objective == res->objective_bound;
    res->key_obj_bits = s.hm.key_obj_bits;
    res->n_gpus = world;
    res->reserved = 0;
    stamp(t0, "bound computed");
    res->total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (!res->feasible) { g_err = "no candidate satisfying C1..C7 was found"; return KAO_INFEASIBLE; }
    return KAO_OK;
}

// fixed partitions (docs/MODEL.md §12): solve the reduced problem, then put the fixed rows and constants back.  A reduced
// problem of at most kSmemRowsMax plain rows whose tables do not fit the shared memory of an SM (at 33..64 slots above
// 7,680 rows) would be refused by the shared-memory path, although the cluster it came from runs on the HBM path: it
// runs there too, with uniform replication rows (rf[p] = RF, ppr = pb's C7: the same program), and keeps the LP
// certificate, computed here on the plain reduced problem.
static int solve_fixed_impl(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp, const uint8_t *fixed,
                            const kao_options *opt, kao_result *res)
{
    if (!fixed) return solve_impl(pb, tp, rp, opt, res);
    if (!pb || !opt || !res || !res->replicas) return fail(KAO_E_ARG, "null argument");
    const auto t0 = std::chrono::steady_clock::now();
    FixedReduction fr;
    std::string why;
    if (!reduce_fixed(*pb, tp, rp, fixed, fr, why)) return fail(KAO_E_ARG, why);
    kao_options o = *opt;
    const kao_replication *rrp = rp ? &fr.rp : nullptr;
    std::vector<int32_t> urf, ulo, uhi;
    kao_replication uniform{};
    bool lp_here = false;
    if (!tp && !rp && fr.pb.P <= kSmemRowsMax) {
        HostModel m;
        SmemPlan plan;
        if (!build_host_model(fr.pb, m, why)) return fail(KAO_E_ARG, why);
        if (!fit_smem_plan(m, m.W <= 2 ? KAO_THREADS : KAO_THREADS_WIDE, plan)) {
            const std::string on = "the reduced problem (" + std::to_string(fr.pb.P) +
                                   " rows) does not fit the shared memory of an SM and runs on the HBM path, which offers no ";
            if (o.flags & KAO_FLAG_ROW_MAJOR) return fail(KAO_E_ARG, "KAO_FLAG_ROW_MAJOR: " + on + "evaluator choice");
            if ((o.n_gpus > 1 || __builtin_popcount(o.device_mask) > 1) && !(o.flags & KAO_FLAG_SPREAD_RESTARTS))
                return fail(KAO_E_ARG, "n_gpus > 1 without KAO_FLAG_SPREAD_RESTARTS: " + on + "sharded rounds");
            urf.assign(fr.pb.P, pb->RF); ulo.assign(fr.pb.P, pb->ppr_lo); uhi.assign(fr.pb.P, pb->ppr_hi);
            uniform = kao_replication{urf.data(), ulo.data(), uhi.data()};
            rrp = &uniform;
            lp_here = (o.flags & KAO_FLAG_LP_BOUND) != 0;
            if (lp_here && !lp_bound_fits(fr.pb)) return fail(KAO_E_ARG, std::string("KAO_FLAG_LP_BOUND: ") + kLpLimit);
            o.flags &= ~KAO_FLAG_LP_BOUND;
        }
    }
    // solve_impl writes into a copy, so that the caller's result never points at the local buffer
    std::vector<int32_t> reduced((size_t)fr.pb.P * pb->RF, -1);
    kao_result r = *res;
    r.replicas = reduced.data();
    const int rc = solve_impl(&fr.pb, tp ? &fr.tp : nullptr, rrp, &o, &r);
    if (rc != KAO_OK && rc != KAO_INFEASIBLE) return rc;
    if (lp_here && r.feasible) {
        std::vector<int> devs;
        int64_t lp = 0;
        uint32_t its = 0;
        int lrc = pick_devices(opt, devs);
        if (lrc != KAO_OK) return lrc;
        lrc = lagrange_bound_device(fr.pb, devs[0], r.objective, KAO_LP_ITERATIONS, wait_budget_ns(), &lp, &its, nullptr,
                                    nullptr, why);
        if (lrc != KAO_OK) return fail(lrc, why);
        r.objective_bound = std::min(r.objective_bound, lp);
        r.optimal = r.feasible && r.objective == r.objective_bound;
    }
    int32_t *const out = res->replicas;
    *res = r;
    res->replicas = out;
    expand_fixed(*pb, fr, reduced.data(), out);
    res->violation += fr.V0;
    res->objective += fr.O0;
    res->objective_bound += fr.O0;
    res->feasible = res->violation == 0;
    res->optimal = res->feasible && res->objective == res->objective_bound;
    res->total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (!res->feasible) {
        g_err = fr.V0 ? "the fixed partitions alone violate C3, C4, C6 or a fixed topic's rows" : "no candidate satisfying C1..C7 was found";
        return KAO_INFEASIBLE;
    }
    return KAO_OK;
}

static int objective_bound_fixed_impl(const kao_problem *pb, const kao_replication *rp, const uint8_t *fixed,
                                      const int32_t *replicas, int64_t *bound)
{
    if (!pb || !bound) return fail(KAO_E_ARG, "null argument");
    FixedReduction fr;
    std::string why;
    const kao_problem *q = pb;
    const kao_replication *qr = rp;
    std::vector<int32_t> sub;
    if (fixed) {
        if (!reduce_fixed(*pb, nullptr, rp, fixed, fr, why)) return fail(KAO_E_ARG, why);
        q = &fr.pb;
        qr = rp ? &fr.rp : nullptr;
        if (replicas) {
            sub.resize((size_t)fr.pb.P * pb->RF);
            for (size_t k = 0; k < fr.searched.size(); ++k)
                std::memcpy(&sub[k * pb->RF], replicas + (size_t)fr.searched[k] * pb->RF, (size_t)pb->RF * 4);
            replicas = sub.data();
        }
    }
    HostModel m;
    if (!build_host_model(*q, m, why) || (qr && !build_host_replication(*qr, m, why))) return fail(KAO_E_ARG, why);
    *bound = objective_upper_bound(m, *q);
    if (replicas) *bound = objective_flow_bound(m, *q, replicas, *bound);
    *bound += fr.O0;
    return KAO_OK;
}

// ------------------------------------------------------------------------------------------
// the C ABI (include/kao.h): thin, guarded entry points
// ------------------------------------------------------------------------------------------
extern "C" int kao_version(void) { return KAO_VERSION; }
extern "C" const char *kao_last_error(void) { return g_err.c_str(); }
extern "C" int kao_key_obj_bits(const kao_problem *pb)
{
    return guarded([&] {
        if (!pb) return fail(KAO_E_ARG, "null argument");
        HostModel m;
        std::string why;
        if (!build_host_model(*pb, m, why)) return fail(KAO_E_ARG, why);
        return m.key_obj_bits;
    });
}
extern "C" int kao_objective_bound(const kao_problem *pb, const int32_t *replicas, int64_t *bound)
{
    return guarded([&] {
        if (!pb || !bound) return fail(KAO_E_ARG, "null argument");
        HostModel m;
        std::string why;
        if (!build_host_model(*pb, m, why)) return fail(KAO_E_ARG, why);
        *bound = objective_upper_bound(m, *pb);
        if (replicas) *bound = objective_flow_bound(m, *pb, replicas, *bound);
        return KAO_OK;
    });
}
extern "C" int kao_objective_bound_replication(const kao_problem *pb, const kao_replication *rp, const int32_t *replicas,
                                               int64_t *bound)
{
    return guarded([&] {
        if (!pb || !bound) return fail(KAO_E_ARG, "null argument");
        HostModel m;
        std::string why;
        if (!build_host_model(*pb, m, why) || (rp && !build_host_replication(*rp, m, why))) return fail(KAO_E_ARG, why);
        *bound = objective_upper_bound(m, *pb);
        if (replicas) *bound = objective_flow_bound(m, *pb, replicas, *bound);
        return KAO_OK;
    });
}
// leader-only rebalancing (docs/MODEL.md §13): host-side, exact, no GPU; the replica sets stay as cur lists them
extern "C" int kao_solve_leaders(const kao_problem *pb, const kao_topics *tp, const uint8_t *fixed, kao_result *res,
                                 int64_t *fixed_violation)
{
    return guarded([&] {
        if (!pb || !res || !res->replicas) return fail(KAO_E_ARG, "null argument");
        const auto t0 = std::chrono::steady_clock::now();
        LeaderPlan plan;
        std::string why;
        if (!solve_leaders(*pb, tp, fixed, plan, why)) return fail(KAO_E_ARG, why);
        std::memcpy(res->replicas, plan.replicas.data(), plan.replicas.size() * sizeof(int32_t));
        res->objective = res->objective_bound = plan.objective;
        res->violation = plan.violation;
        res->feasible = plan.violation == 0;
        res->optimal = res->feasible;
        res->moves = 0;
        res->key = 0;
        res->n_candidates = 0;
        res->rounds_run = 0;
        res->restarts = 0;
        res->device_ms = 0;
        res->key_obj_bits = kao_key_obj_bits(pb);
        res->n_gpus = 0;
        if (fixed_violation) *fixed_violation = plan.fixed_violation;
        res->total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        if (!res->feasible) return fail(KAO_INFEASIBLE, "leaders only: the best choice of leaders still violates the rows by " +
                                                        std::to_string(plan.violation) + " (" + std::to_string(plan.fixed_violation) +
                                                        " of it in the rows the replica sets fix)");
        return KAO_OK;
    });
}
extern "C" int kao_lp_bound(const kao_problem *pb, const int32_t *replicas, int32_t device, uint32_t max_iterations,
                            int64_t *bound, uint32_t *iterations_run, int64_t *multipliers)
{
    return guarded([&] {
        if (!pb || !replicas || !bound || !iterations_run) return fail(KAO_E_ARG, "null argument");
        if (max_iterations < 1 || max_iterations > KAO_MAX_LP_ITERATIONS)
            return fail(KAO_E_ARG, "max_iterations must be 1..KAO_MAX_LP_ITERATIONS (2^20)");
        HostModel m;
        std::string why;
        if (!build_host_model(*pb, m, why)) return fail(KAO_E_ARG, why);
        if (!lp_bound_fits(*pb)) return fail(KAO_E_ARG, std::string("kao_lp_bound: ") + kLpLimit);
        int64_t T = 0;
        if (!feasible_objective(*pb, replicas, T, why)) return fail(KAO_E_ARG, why);
        int ndev = 0;
        if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(KAO_E_CUDA, "no CUDA device: libkao has no CPU path");
        if (device < 0 || device >= ndev) return fail(KAO_E_ARG, "bad device ordinal");
        const int rc = lagrange_bound_device(*pb, device, T, max_iterations, wait_budget_ns(), bound, iterations_run, multipliers, nullptr, why);
        return rc == KAO_OK ? KAO_OK : fail(rc, why);
    });
}
extern "C" int kao_create(const kao_problem *pb, int32_t device, kao_handle **out) { return guarded([&] { return create_handle(pb, device, out); }); }
extern "C" int kao_create_topics(const kao_problem *pb, const kao_topics *tp, int32_t device, kao_handle **out)
{
    return guarded([&] { return create_handle(pb, device, out, tp); });
}
extern "C" int kao_create_replication(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp,
                                      int32_t device, kao_handle **out)
{
    return guarded([&] { return create_handle(pb, device, out, tp, rp); });
}
extern "C" int kao_destroy(kao_handle *h) { return guarded([&] { return destroy_impl(h); }); }
extern "C" int kao_reset(kao_handle *h) { return guarded([&] { return reset_impl(h); }); }
extern "C" int kao_set_base(kao_handle *h, const int32_t *replicas) { return guarded([&] { return set_base_impl(h, replicas); }); }
extern "C" int kao_get_base(kao_handle *h, int32_t *replicas, int64_t *violation, int64_t *objective, int32_t *moves)
{
    return guarded([&] { return get_base_impl(h, replicas, violation, objective, moves); });
}
extern "C" int kao_round_launch(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                                uint32_t idx_lo, uint32_t idx_hi, uint64_t *d_key, void *stream)
{
    return guarded([&] {
        if (!h || !d_key) return fail(KAO_E_ARG, "null argument");
        if (h->large) return refuse_large("kao_round_launch", h->topics, h->rf);
        if (!check_round_args(round_size) || idx_lo > idx_hi || idx_hi > round_size)
            return fail(KAO_E_ARG, "bad round_size / index range");
        CUDA_TRY(cudaSetDevice(h->device));
        CUDA_TRY(launch_round(h, seed, round, round_size, idx_lo, idx_hi,
                              reinterpret_cast<unsigned long long *>(d_key), nullptr, (cudaStream_t)stream));
        return KAO_OK;
    });
}
extern "C" int kao_round_apply(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                               const uint64_t *d_key, void *stream)
{
    return guarded([&] {
        if (!h || !d_key) return fail(KAO_E_ARG, "null argument");
        if (h->large) return refuse_large("kao_round_apply", h->topics, h->rf);
        if (!check_round_args(round_size)) return fail(KAO_E_ARG, "bad round_size");
        CUDA_TRY(cudaSetDevice(h->device));
        CUDA_TRY(launch_apply(h, seed, round, round_size, reinterpret_cast<const unsigned long long *>(d_key), 0,
                              (cudaStream_t)stream));
        return KAO_OK;
    });
}
extern "C" int kao_set_evaluator(kao_handle *h, int32_t evaluator)
{
    return guarded([&] {
        if (!h) return fail(KAO_E_ARG, "null handle");
        if (h->large) return refuse_large("kao_set_evaluator", h->topics, h->rf);
        if (evaluator != KAO_EVAL_ROW_MAJOR && evaluator != KAO_EVAL_COLUMN_MAJOR) return fail(KAO_E_ARG, "unknown evaluator");
        if (evaluator == KAO_EVAL_COLUMN_MAJOR && !h->trans_ok)
            return fail(KAO_E_ARG, "column-major evaluator: needs rows of up to 64 slots, racks of up to 8 brokers, at most one "
                                   "replica per rack (C7 0..1), three objective mask planes, and its planes in shared memory");
        h->evaluator = evaluator;
        return KAO_OK;
    });
}
extern "C" int kao_set_schedule(kao_handle *h, int32_t sync, int32_t pop, int32_t threads)
{
    return guarded([&] {
        if (!h) return fail(KAO_E_ARG, "null handle");
        if (h->large) return refuse_large("kao_set_schedule", h->topics, h->rf);
        if (!schedule_exists(sync, pop, threads)) return fail(KAO_E_ARG, "no such schedule (kao.h, kao_set_schedule)");
        h->sch_sync = sync; h->sch_pop = pop; h->sch_threads = threads;
        return KAO_OK;
    });
}
extern "C" int kao_get_evaluator(kao_handle *h, int32_t *evaluator, int32_t *sync, int32_t *pop, int32_t *threads)
{
    if (!h) return fail(KAO_E_ARG, "null handle");
    if (evaluator) *evaluator = h->evaluator;
    if (sync) *sync = h->sch_sync;
    if (pop) *pop = h->sch_pop;
    if (threads) *threads = h->sch_threads;
    return KAO_OK;
}
extern "C" int kao_set_patience(kao_handle *h, uint32_t rounds_without_improvement)
{
    if (!h) return fail(KAO_E_ARG, "null handle");
    h->patience = rounds_without_improvement;
    return KAO_OK;
}
extern "C" int kao_last_rounds(kao_handle *h, uint32_t *rounds_run)
{
    if (!h || !rounds_run) return fail(KAO_E_ARG, "null argument");
    *rounds_run = h->last_rounds;
    return KAO_OK;
}
extern "C" int kao_search(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                          uint32_t round_size, uint64_t *round_keys, double *device_ms)
{
    return guarded([&] { return search_impl(h, seed, first_round, rounds, round_size, round_keys, device_ms, false); });
}
// Same search, same keys, same trajectory — but every candidate is scored by DELTA evaluation
// (base totals + its <= 3 patched rows, one thread per candidate) instead of a full evaluation.
extern "C" int kao_search_delta(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                                uint32_t round_size, uint64_t *round_keys, double *device_ms)
{
    return guarded([&] { return search_impl(h, seed, first_round, rounds, round_size, round_keys, device_ms, true); });
}
extern "C" int kao_candidate_keys(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                                  uint32_t idx_begin, uint32_t count, uint64_t *keys)
{
    return guarded([&] { return candidate_keys_impl(h, seed, round, round_size, idx_begin, count, keys, false); });
}
extern "C" int kao_candidate_keys_delta(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                                        uint32_t idx_begin, uint32_t count, uint64_t *keys)
{
    return guarded([&] { return candidate_keys_impl(h, seed, round, round_size, idx_begin, count, keys, true); });
}
extern "C" int kao_p2p_export(kao_handle *h, uint8_t *handle_out) { return guarded([&] { return p2p_export_impl(h, handle_out); }); }
extern "C" int kao_p2p_connect(kao_handle *h, int32_t rank, int32_t world, const uint8_t *handles)
{
    return guarded([&] { return p2p_connect_impl(h, rank, world, handles); });
}
extern "C" int kao_search_sharded(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                                  uint32_t round_size, uint64_t *round_keys, double *device_ms)
{
    return guarded([&] { return sharded_impl(h, seed, first_round, rounds, round_size, round_keys, device_ms, false); });
}
extern "C" int kao_search_sharded_delta(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                                        uint32_t round_size, uint64_t *round_keys, double *device_ms)
{
    return guarded([&] { return sharded_impl(h, seed, first_round, rounds, round_size, round_keys, device_ms, true); });
}
extern "C" int kao_profile_rounds(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                                  uint32_t round_size, double *search_ms, double *apply_ms)
{
    return guarded([&] { return profile_rounds_impl(h, seed, first_round, rounds, round_size, search_ms, apply_ms); });
}
extern "C" int kao_stats(kao_handle *h, uint64_t *kernel_launches, int32_t *words_per_row,
                         int32_t *slots, int32_t *dense_weights)
{
    if (!h) return fail(KAO_E_ARG, "null handle");
    if (kernel_launches) *kernel_launches = h->launches;
    if (words_per_row) *words_per_row = h->hm.W;
    if (slots) *slots = h->hm.NS;
    if (dense_weights) *dense_weights = h->hm.dense ? 1 : 0;
    return KAO_OK;
}
extern "C" int kao_eval(const kao_problem *pb, int32_t device, const int32_t *replicas, int32_t n,
                        int64_t *violation, int64_t *objective)
{
    return guarded([&] { return eval_impl(pb, device, replicas, n, violation, objective); });
}
extern "C" int kao_solve(const kao_problem *pb, const kao_options *opt, kao_result *res)
{
    return guarded([&] { return solve_impl(pb, nullptr, nullptr, opt, res); });
}
extern "C" int kao_solve_topics(const kao_problem *pb, const kao_topics *tp, const kao_options *opt, kao_result *res)
{
    return guarded([&] { return solve_impl(pb, tp, nullptr, opt, res); });
}
extern "C" int kao_solve_replication(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp,
                                     const kao_options *opt, kao_result *res)
{
    return guarded([&] { return solve_impl(pb, tp, rp, opt, res); });
}
extern "C" int kao_solve_fixed(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp, const uint8_t *fixed,
                               const kao_options *opt, kao_result *res)
{
    return guarded([&] { return solve_fixed_impl(pb, tp, rp, fixed, opt, res); });
}
extern "C" int kao_objective_bound_fixed(const kao_problem *pb, const kao_replication *rp, const uint8_t *fixed,
                                         const int32_t *replicas, int64_t *bound)
{
    return guarded([&] { return objective_bound_fixed_impl(pb, rp, fixed, replicas, bound); });
}
