// kao_lagrange.cu — the Lagrangian LP bound on the GPU (docs/MODEL.md §9).  The coupling rows C3 (replicas per
// broker), C4 (leaders per broker) and C6 (replicas per rack) are dualised with int64 multipliers of
// KAO_LP_FRACTION_BITS fractional bits; what is left splits into one small network flow per partition, solved
// exactly by a dynamic program over the racks.  The subgradient iteration runs in ONE cooperative persistent
// launch: partitions are spread over the CTAs, every CTA sums its partitions' part of L and of the row counts in
// shared memory, adds them into a double-buffered HBM accumulator with integer atomics, meets the others at the
// search kernels' grid barrier (spin_until), and takes the same step from the same totals as every other CTA.
// Integer sums do not depend on the order of the atomics, so the trajectory is deterministic and bit-identical
// to the plain-C restatement (tests/lp_ref/lagrange_ref.c).
#include "kao_kernels.cuh"
#include "kao_lagrange.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <climits>

namespace kao {
namespace {

constexpr int kLpThreads = 128;
constexpr int kLpF = KAO_LP_FRACTION_BITS;
constexpr long long kLpBox = 1ll << 34;             // |u| <= U = 2^34 (MODEL §9: every sum fits in int64)
constexpr long long kLpNeg = LLONG_MIN;           // no admissible row (yet)
constexpr int kLpMaxRF = KAO_MAX_RF;

struct LpArgs {
    int P, B, R, RF, ppr_lo, ppr_hi, NR, chunk;
    const uint32_t *w;                 // [P][B] wF | wL << 16
    const int *tab;                    // rstart[R + 1], order[B] (brokers by rack, ascending index), rack[B]
    const long long *bnd;              // lo[NR], hi[NR] (upper bounds lowered to what an assignment can reach)
    long long T;
    uint32_t max_iterations;
    unsigned long long *acc;           // [2][1 + NR] running sums per parity of the iteration: L part, row counts
    unsigned int *bar;                 // [0] grid barrier arrivals, [1] abort
    unsigned long long timeout_ns;
    long long *out;                    // [0] bound, [1] iterations run, [2 ..] multipliers of the minimum
};

// best_p of one partition (MODEL §9): the best row satisfying C1, C2, C5 and C7 under the reduced weights
// (w << F) - a3[b] (follower) / (wL << F) - a4[b] (leader); the counts of the row it picks go to cnt3/cnt4/cnt6.
// The DP and its tie-breaks are those of the restatement, statement for statement.
__device__ long long best_row(const uint32_t *wrow, const long long *a3, const long long *a4, const int *rstart,
                              const int *order, int R, int RF, int plo, int phi, unsigned long long *cnt3,
                              unsigned long long *cnt4, unsigned long long *cnt6)
{
    long long dp[kLpMaxRF + 1][2], nd[kLpMaxRF + 1][2];
    uint8_t ch[KAO_MAX_RACKS][kLpMaxRF + 1][2];
    uint8_t topj[KAO_MAX_RACKS][kLpMaxRF], gpos[KAO_MAX_RACKS][kLpMaxRF + 1], kr[KAO_MAX_RACKS];
    int16_t restj[KAO_MAX_RACKS];
    for (int n = 0; n <= RF; ++n) dp[n][0] = dp[n][1] = kLpNeg;
    dp[0][0] = 0;
    auto fw = [&](int b) { return ((long long)(wrow[b] & 0xFFFFu) << kLpF) - a3[b]; };
    auto lw = [&](int b) { return ((long long)(wrow[b] >> 16) << kLpF) - a4[b]; };
    for (int r = 0; r < R; ++r) {
        const int j0 = rstart[r], j1 = rstart[r + 1], size = j1 - j0;
        int K = min(min(size, RF), phi);
        kr[r] = (uint8_t)K;
        // the K best followers: descending reduced follower weight, ties by ascending broker index
        long long tv[kLpMaxRF];
        int len = 0;
        for (int j = j0; j < j1; ++j) {
            const int b = order[j];
            const long long v = fw(b);
            int pos = len;
            while (pos > 0 && tv[pos - 1] < v) --pos;
            if (pos >= K) continue;
            for (int i = (len < K ? len : K - 1); i > pos; --i) { tv[i] = tv[i - 1]; topj[r][i] = topj[r][i - 1]; }
            tv[pos] = v; topj[r][pos] = (uint8_t)b;
            if (len < K) ++len;
        }
        long long S[kLpMaxRF + 1], G[kLpMaxRF + 1];
        S[0] = 0;
        for (int i = 0; i < K; ++i) S[i + 1] = S[i] + tv[i];
        // the best leader among the rack's other brokers: largest reduced leader weight, first by broker index
        restj[r] = -1;
        long long restv = 0;
        for (int j = j0; j < j1; ++j) {
            const int b = order[j];
            bool top = false;
            for (int i = 0; i < K; ++i) top |= topj[r][i] == b;
            if (top) continue;
            const long long v = lw(b);
            if (restj[r] < 0 || v > restv) { restj[r] = (int16_t)b; restv = v; }
        }
        // G[k]: a leader and k - 1 followers in this rack; candidates in follower rank order, then the rest
        for (int k = 1; k <= K; ++k) {
            long long best = 0;
            int bp = -1;
            for (int i = 0; i < K; ++i) {
                const long long v = (i < k ? S[k] - tv[i] : S[k - 1]) + lw(topj[r][i]);
                if (bp < 0 || v > best) { best = v; bp = i; }
            }
            if (restj[r] >= 0 && S[k - 1] + restv > best) { best = S[k - 1] + restv; bp = K; }
            G[k] = best; gpos[r][k] = (uint8_t)bp;
        }
        for (int n = 0; n <= RF; ++n) nd[n][0] = nd[n][1] = kLpNeg;
        for (int n = 0; n <= RF; ++n)
            for (int l = 0; l < 2; ++l) {
                if (dp[n][l] == kLpNeg) continue;
                for (int k = plo; k <= K && n + k <= RF; ++k) {
                    const long long v = dp[n][l] + S[k];
                    if (v > nd[n + k][l]) { nd[n + k][l] = v; ch[r][n + k][l] = (uint8_t)k; }
                    if (l == 0 && k >= 1) {
                        const long long g = dp[n][0] + G[k];
                        if (g > nd[n + k][1]) { nd[n + k][1] = g; ch[r][n + k][1] = (uint8_t)(k | 16); }
                    }
                }
            }
        for (int n = 0; n <= RF; ++n) { dp[n][0] = nd[n][0]; dp[n][1] = nd[n][1]; }
    }
    const long long best = dp[RF][1];
    if (best == kLpNeg) return kLpNeg;
    int n = RF, l = 1;
    for (int r = R - 1; r >= 0; --r) {
        const int c = ch[r][n][l], k = c & 15, lead = c >> 4;
        if (k) atomicAdd(cnt6 + r, (unsigned long long)k);
        if (!lead) {
            for (int i = 0; i < k; ++i) atomicAdd(cnt3 + topj[r][i], 1ull);
        } else {
            const int gp = gpos[r][k], leader = gp < kr[r] ? topj[r][gp] : restj[r];
            atomicAdd(cnt3 + leader, 1ull);
            atomicAdd(cnt4 + leader, 1ull);
            for (int i = 0, nf = 0; i < k && nf < k - 1; ++i)
                if (i != gp) { atomicAdd(cnt3 + topj[r][i], 1ull); ++nf; }
        }
        n -= k; l -= lead;
    }
    return best;
}

__device__ __forceinline__ long long block_sum(long long v, long long *s_red, int slot)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
    const int warp = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) s_red[slot * (kLpThreads / 32) + warp] = v;
    __syncthreads();
    long long t = 0;
    for (int i = 0; i < kLpThreads / 32; ++i) t += s_red[slot * (kLpThreads / 32) + i];
    return t;
}

__global__ void __launch_bounds__(kLpThreads, 1) lagrange_kernel(LpArgs a)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int NR = a.NR, B = a.B, tid = threadIdx.x;
    long long *s_u = reinterpret_cast<long long *>(smem);
    long long *s_ub = s_u + NR, *s_lo = s_ub + NR, *s_hi = s_lo + NR, *s_g = s_hi + NR;
    long long *s_a3 = s_g + NR, *s_a4 = s_a3 + B;
    unsigned long long *s_cnt = reinterpret_cast<unsigned long long *>(s_a4 + B);      // [1 + NR]
    unsigned long long *s_prev = s_cnt + (NR + 1);                                      // [2][1 + NR]
    long long *s_red = reinterpret_cast<long long *>(s_prev + 2 * (NR + 1));            // [2][warps]
    int *s_tab = reinterpret_cast<int *>(s_red + 2 * (kLpThreads / 32));               // rstart, order, rack
    int *s_flag = s_tab + (a.R + 1 + 2 * B);
    uint32_t *s_w = reinterpret_cast<uint32_t *>(s_flag + 4);
    const int *s_rstart = s_tab, *s_order = s_tab + a.R + 1, *s_rack = s_order + B;

    // stage once per call: this CTA's weight rows, the rack tables, the row bounds
    const int p0 = blockIdx.x * a.chunk, np = max(0, min(a.P - p0, a.chunk));
    for (int i = tid; i < np * B; i += kLpThreads) s_w[i] = a.w[(size_t)p0 * B + i];
    for (int i = tid; i < a.R + 1 + 2 * B; i += kLpThreads) s_tab[i] = a.tab[i];
    for (int i = tid; i < NR; i += kLpThreads) { s_u[i] = 0; s_lo[i] = a.bnd[i]; s_hi[i] = a.bnd[NR + i]; }
    for (int i = tid; i < 2 * (NR + 1); i += kLpThreads) s_prev[i] = 0;
    if (tid == 0) s_flag[0] = 0;
    __syncthreads();

    long long best = LLONG_MAX;
    uint32_t it = 0;
    for (;;) {
        ++it;
        for (int b = tid; b < B; b += kLpThreads) {
            s_a3[b] = s_u[b] + s_u[2 * B + s_rack[b]];
            s_a4[b] = s_a3[b] + s_u[B + b];
        }
        for (int i = tid; i <= NR; i += kLpThreads) s_cnt[i] = 0;
        __syncthreads();
        for (int q = tid; q < np; q += kLpThreads) {
            const long long v = best_row(s_w + (size_t)q * B, s_a3, s_a4, s_rstart, s_order, a.R, a.RF, a.ppr_lo,
                                         a.ppr_hi, s_cnt + 1, s_cnt + 1 + B, s_cnt + 1 + 2 * B);
            atomicAdd(s_cnt, (unsigned long long)v);
        }
        __syncthreads();
        unsigned long long *buf = a.acc + (size_t)(it & 1) * (NR + 1);
        for (int i = tid; i <= NR; i += kLpThreads)
            if (s_cnt[i]) atomicAdd(buf + i, s_cnt[i]);
        __syncthreads();
        // grid barrier: every CTA's sums are in `buf` before anyone reads it
        if (tid == 0) {
            __threadfence();
            atomicAdd(a.bar, 1u);
            if (!spin_until(a.bar, it * gridDim.x, reinterpret_cast<int *>(a.bar + 1), a.timeout_ns)) s_flag[0] = 1;
            __threadfence();
        }
        __syncthreads();
        if (s_flag[0]) return;
        // this iteration's totals: the running sum of this parity minus what it held two iterations ago (modulo
        // 2^64, exact).  `buf` is written again only after the next barrier, which every CTA passes after this.
        unsigned long long *prev = s_prev + (size_t)(it & 1) * (NR + 1);
        for (int i = tid; i <= NR; i += kLpThreads) {
            const unsigned long long cur = __ldcg(buf + i);
            s_cnt[i] = cur - prev[i];
            prev[i] = cur;
        }
        __syncthreads();
        long long phi = 0, n2 = 0;
        for (int i = tid; i < NR; i += kLpThreads) {
            const long long u = s_u[i], lo = s_lo[i], hi = s_hi[i], c = (long long)s_cnt[1 + i];
            phi += u > 0 ? u * hi : u * lo;
            const long long g = (u > 0 ? hi : u < 0 ? lo : (c < lo ? lo : c > hi ? hi : c)) - c;
            s_g[i] = g;
            n2 += g * g;
        }
        phi = block_sum(phi, s_red, 0);
        n2 = block_sum(n2, s_red, 1);
        const long long L = (long long)s_cnt[0] + phi;
        if (L < best) {
            best = L;
            if (blockIdx.x == 0)
                for (int i = tid; i < NR; i += kLpThreads) s_ub[i] = s_u[i];
        }
        if ((best >> kLpF) <= a.T || n2 == 0 || it >= a.max_iterations) break;
        long long s = (L - (a.T << kLpF)) / n2;
        if (s <= 0) break;
        if (s > 2 * kLpBox) s = 2 * kLpBox;          // any larger step clamps every moved multiplier to +-U as well
        for (int i = tid; i < NR; i += kLpThreads) {
            const long long v = s_u[i] - s * s_g[i];
            s_u[i] = v < -kLpBox ? -kLpBox : v > kLpBox ? kLpBox : v;
        }
        __syncthreads();
    }
    if (blockIdx.x == 0) {
        __syncthreads();
        if (tid == 0) { a.out[0] = best >> kLpF; a.out[1] = it; }
        for (int i = tid; i < NR; i += kLpThreads) a.out[2 + i] = s_ub[i];
    }
}

size_t lp_smem_bytes(int NR, int B, int R, int chunk)
{
    return (size_t)8 * (5 * NR + 2 * B) + 8 * (size_t)3 * (NR + 1) + 8 * 2 * (kLpThreads / 32) +
           4 * (size_t)(R + 1 + 2 * B + 4) + 4 * (size_t)chunk * B;
}

// device buffers of one call, freed on every path out
struct LpBuffers {
    void *p = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    ~LpBuffers()
    {
        if (p) cudaFree(p);
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    }
};

}  // namespace

int lagrange_bound_device(const kao_problem &pb, int device, int64_t T, uint32_t max_iterations,
                          unsigned long long timeout_ns, int64_t *bound, uint32_t *iterations_run,
                          int64_t *multipliers, double *device_ms, std::string &why)
{
    auto cuda_fail = [&](const char *what, cudaError_t e) { why = std::string(what) + ": " + cudaGetErrorString(e); return KAO_E_CUDA; };
    const int P = pb.P, B = pb.B, R = pb.R, NR = 2 * B + R;
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) return cuda_fail("cudaSetDevice", e);
    int sms = 0;
    e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (e != cudaSuccess) return cuda_fail("cudaDeviceGetAttribute", e);
    // one CTA per SM (at most one per partition), the partitions in contiguous chunks
    const int chunk = (P + std::min(sms, P) - 1) / std::min(sms, P), grid = (P + chunk - 1) / chunk;
    const size_t smem = lp_smem_bytes(NR, B, R, chunk);
    if (smem > 220u * 1024u) { why = "kao_lp_bound: the weight rows of a CTA's partitions do not fit in shared memory"; return KAO_E_ARG; }
    e = cudaFuncSetAttribute(lagrange_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_fail("cudaFuncSetAttribute", e);
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lagrange_kernel, kLpThreads, smem);
    if (e != cudaSuccess) return cuda_fail("cudaOccupancyMaxActiveBlocksPerMultiprocessor", e);
    if (per_sm < 1 || grid > per_sm * sms) { why = "kao_lp_bound: the grid cannot be co-resident"; return KAO_E_CUDA; }

    // host tables: packed weights, racks, row bounds (MODEL §9: an upper bound above what any assignment reaches
    // is lowered to that, which leaves the rows as they are and keeps every product in int64)
    std::vector<uint32_t> w((size_t)P * B);
    for (size_t i = 0; i < w.size(); ++i) w[i] = (uint32_t)pb.wF[i] | ((uint32_t)pb.wL[i] << 16);
    std::vector<int> tab(R + 1 + 2 * B, 0);
    for (int b = 0; b < B; ++b) ++tab[pb.rack_of[b] + 1];
    for (int r = 0; r < R; ++r) tab[r + 1] += tab[r];
    {
        std::vector<int> fill(R, 0);
        for (int b = 0; b < B; ++b) tab[R + 1 + tab[pb.rack_of[b]] + fill[pb.rack_of[b]]++] = b;
    }
    for (int b = 0; b < B; ++b) tab[R + 1 + B + b] = pb.rack_of[b];
    const long long tot = (long long)P * pb.RF;
    std::vector<long long> bnd(2 * NR);
    for (int b = 0; b < B; ++b) {
        bnd[b] = pb.rep_lo[b]; bnd[NR + b] = std::min<long long>(pb.rep_hi[b], tot);
        bnd[B + b] = pb.ldr_lo[b]; bnd[NR + B + b] = std::min<long long>(pb.ldr_hi[b], P);
    }
    for (int r = 0; r < R; ++r) { bnd[2 * B + r] = pb.rack_lo[r]; bnd[NR + 2 * B + r] = std::min<long long>(pb.rack_hi[r], tot); }

    // one device allocation: acc | bar | out | bnd | tab | w
    const size_t o_acc = 0, o_bar = o_acc + 8 * 2 * (size_t)(NR + 1), o_out = o_bar + 16, o_bnd = o_out + 8 * (size_t)(NR + 2),
                 o_tab = o_bnd + 8 * bnd.size(), o_w = (o_tab + 4 * tab.size() + 15) / 16 * 16, total = o_w + 4 * w.size();
    LpBuffers d;
    e = cudaMalloc(&d.p, total);
    if (e != cudaSuccess) return cuda_fail("cudaMalloc", e);
    char *base = static_cast<char *>(d.p);
    if ((e = cudaMemset(base, 0, o_out)) != cudaSuccess) return cuda_fail("cudaMemset", e);
    if ((e = cudaMemcpy(base + o_bnd, bnd.data(), 8 * bnd.size(), cudaMemcpyHostToDevice)) != cudaSuccess ||
        (e = cudaMemcpy(base + o_tab, tab.data(), 4 * tab.size(), cudaMemcpyHostToDevice)) != cudaSuccess ||
        (e = cudaMemcpy(base + o_w, w.data(), 4 * w.size(), cudaMemcpyHostToDevice)) != cudaSuccess)
        return cuda_fail("cudaMemcpy", e);
    LpArgs a;
    a.P = P; a.B = B; a.R = R; a.RF = pb.RF; a.ppr_lo = pb.ppr_lo; a.ppr_hi = pb.ppr_hi; a.NR = NR; a.chunk = chunk;
    a.w = reinterpret_cast<const uint32_t *>(base + o_w);
    a.tab = reinterpret_cast<const int *>(base + o_tab);
    a.bnd = reinterpret_cast<const long long *>(base + o_bnd);
    a.T = T; a.max_iterations = max_iterations;
    a.acc = reinterpret_cast<unsigned long long *>(base + o_acc);
    a.bar = reinterpret_cast<unsigned int *>(base + o_bar);
    a.timeout_ns = timeout_ns;
    a.out = reinterpret_cast<long long *>(base + o_out);
    if ((e = cudaEventCreate(&d.e0)) != cudaSuccess || (e = cudaEventCreate(&d.e1)) != cudaSuccess) return cuda_fail("cudaEventCreate", e);
    void *args[] = {&a};
    cudaEventRecord(d.e0);
    // cooperative launch: all CTAs are co-resident, which the grid barrier needs
    e = cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(lagrange_kernel), dim3(grid), dim3(kLpThreads), args, smem, 0);
    if (e != cudaSuccess) return cuda_fail("lagrange kernel launch", e);
    cudaEventRecord(d.e1);
    if ((e = cudaEventSynchronize(d.e1)) != cudaSuccess) return cuda_fail("lagrange kernel", e);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, d.e0, d.e1);
    if (device_ms) *device_ms = ms;
    unsigned int bar[2];
    std::vector<long long> out(NR + 2);
    if ((e = cudaMemcpy(bar, base + o_bar, 8, cudaMemcpyDeviceToHost)) != cudaSuccess ||
        (e = cudaMemcpy(out.data(), base + o_out, 8 * out.size(), cudaMemcpyDeviceToHost)) != cudaSuccess)
        return cuda_fail("cudaMemcpy", e);
    if (bar[1]) { why = "lagrange kernel timed out at a grid barrier"; return KAO_E_CUDA; }
    *bound = out[0];
    *iterations_run = (uint32_t)out[1];
    if (multipliers) for (int i = 0; i < NR; ++i) multipliers[i] = out[2 + i];
    return KAO_OK;
}

}  // namespace kao
