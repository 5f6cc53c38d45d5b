// kao_emu_sorted.cpp — TEST INFRASTRUCTURE.  The sorted-batch body of the tensor-core schedules (pop 0x300,
// csrc/kao_kernels.cuh: build_cand_list and the batch loop of search_persistent_kernel) restated for the host on top
// of the tensor-core emulation of tests/emu_mma: every CTA sorts its share of a round by cand_class
// (csrc/kao_device_mma.cuh) and its warps generate, park and evaluate batches of 32 neighbours of that order.
// tests/test_mma_sorted_batches.py checks it against the oracle restatement.  Never linked into libkao.so.
#include "../emu_mma/kao_emu_mma.cpp"

namespace {

// lane j generates candidate idx[j] (j < count), as one warp of the search kernel does; out[j]: its key
template <int W> void keys_lanes(MmaEmu &x, uint64_t seed, uint32_t round, const uint32_t *idx, uint32_t count, uint32_t round_size,
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
        if ((uint32_t)lane < count) make_gen<W>(x).run(seed, round, idx[lane], round_size, ps, rows);
        int pviol, pobj, pcount;
        patch_terms<W>(e.prm, ps, rows, pviol, pobj, pcount);
        mma_park_patch<W>(ps, rows, pviol, pobj, batch, lane);
        __syncwarp();
        int viol, obj;
        if (e.nW == 32) eval_batch_mma<EvalCfgT<W, 32, 1, 0x300>>(e.prm, &e.cs, x.T.data(), e.nW, x.Z.data(), batch, lane, viol, obj);
        else eval_batch_mma<EvalCfgT<W, 0, 1, 0x300>>(e.prm, &e.cs, x.T.data(), e.nW, x.Z.data(), batch, lane, viol, obj);
        const uint32_t j = (uint32_t)mma_lane_candidate(lane);
        if (j < count) out[j] = pack_key(viol, obj, idx[j], e.prm.key_obj_bits);
    });
}

// CTA c of `grid` CTAs of `warps` warps takes first = idx_lo + c * warps, + stride, ... below idx_hi.  If that share
// holds at most `cap` candidates it is sorted by cand_class (counting sort; the kernel's order within a class is
// arbitrary, this one keeps the positions' order) and cut into batches of 32; else every warp walks its own candidates
// in batches of 32 as the unsorted schedules do.  Returns the share in batch order; `bounds`: where each batch ends.
std::vector<uint32_t> cta_batches(uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_lo, uint32_t idx_hi,
                                  uint32_t grid, uint32_t warps, uint32_t cap, uint32_t cta, std::vector<uint32_t> &bounds)
{
    const uint32_t stride = grid * warps, first = idx_lo + cta * warps, n = cand_count(first, stride, warps, idx_hi);
    std::vector<uint32_t> list;
    bounds.assign(1, 0);
    if (n <= cap) {
        std::vector<uint32_t> cnt(kCandClasses + 1, 0), cls(n);
        for (uint32_t k = 0; k < n; ++k) ++cnt[1 + (cls[k] = cand_class(seed, round, cand_at(k, first, stride, warps), round_size))];
        for (uint32_t c = 0; c < kCandClasses; ++c) cnt[c + 1] += cnt[c];
        list.resize(n);
        for (uint32_t k = 0; k < n; ++k) list[cnt[cls[k]]++] = cand_at(k, first, stride, warps);
        for (uint32_t b = 0; 32 * b < n; ++b) bounds.push_back(std::min(n, 32 * b + 32));
    } else {
        const uint32_t iters = first < idx_hi ? (idx_hi - first + stride - 1) / stride : 0;
        for (uint32_t w = 0; w < warps; ++w)
            for (uint32_t it0 = 0; it0 < iters; it0 += 32) {
                for (uint32_t it = it0; it < std::min(iters, it0 + 32); ++it)
                    if (first + w + it * stride < idx_hi) list.push_back(first + w + it * stride);
                if (list.size() > bounds.back()) bounds.push_back((uint32_t)list.size());
            }
    }
    return list;
}

template <int W> void sorted_keys(MmaEmu &x, uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_lo, uint32_t idx_hi,
                                  uint32_t grid, uint32_t warps, uint32_t cap, unsigned long long *out)
{
    unsigned long long k32[32];
    std::vector<uint32_t> bounds;
    for (uint32_t c = 0; c < grid; ++c) {
        const std::vector<uint32_t> list = cta_batches(seed, round, round_size, idx_lo, idx_hi, grid, warps, cap, c, bounds);
        for (size_t b = 0; b + 1 < bounds.size(); ++b) {
            const uint32_t count = bounds[b + 1] - bounds[b];
            keys_lanes<W>(x, seed, round, list.data() + bounds[b], count, round_size, k32);
            for (uint32_t j = 0; j < count; ++j) out[list[bounds[b] + j] - idx_lo] = k32[j];
        }
    }
}

}  // namespace

extern "C" {

// keys of the candidates idx_lo .. idx_hi - 1 of a round as the sorted-batch body computes them (h: kao_emu_mma_create)
void kao_emu_sorted_keys(void *h, uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_lo, uint32_t idx_hi,
                         uint32_t grid, uint32_t warps, uint32_t cap, uint64_t *out)
{
    auto &x = *static_cast<MmaEmu *>(h);
    with_w(x, [&](auto w) {
        sorted_keys<decltype(w)::value>(x, seed, round, round_size, idx_lo, idx_hi, grid, warps, cap, reinterpret_cast<unsigned long long *>(out));
        return 0;
    });
}

// CTA cta's candidates in the order its warps generate them, their classes and where each batch ends; 1 if sorted
int kao_emu_sorted_cta_batches(uint64_t seed, uint32_t round, uint32_t round_size, uint32_t idx_lo, uint32_t idx_hi, uint32_t grid,
                               uint32_t warps, uint32_t cap, uint32_t cta, uint32_t *list, uint32_t *classes, uint32_t *bounds, uint32_t *nbounds)
{
    std::vector<uint32_t> b;
    const std::vector<uint32_t> l = cta_batches(seed, round, round_size, idx_lo, idx_hi, grid, warps, cap, cta, b);
    for (size_t i = 0; i < l.size(); ++i) { list[i] = l[i]; classes[i] = cand_class(seed, round, l[i], round_size); }
    for (size_t i = 0; i < b.size(); ++i) bounds[i] = b[i];
    *nbounds = (uint32_t)b.size();
    return cand_count(idx_lo + cta * warps, grid * warps, warps, idx_hi) <= cap ? 1 : 0;
}

}  // extern "C"
