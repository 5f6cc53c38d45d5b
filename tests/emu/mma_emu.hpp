// mma_emu.hpp — TEST INFRASTRUCTURE.  The two warp-wide PTX instructions of the tensor-core column-major evaluator
// (csrc/kao_device_mma.cuh) restated for the warp emulator of warp_emu.hpp, with their PTX fragment
// semantics.  Both are warp collectives: every lane publishes its operands, then reads what the others published.
#pragma once
#include "warp_emu.hpp"

#include <cstring>

namespace emu {
enum { OP_LDSM = 101, OP_MMA = 102 };

// every lane's 64-bit value, through one collective
inline void gather_lanes(int op, uint64_t mine, uint64_t (&all)[kLanes])
{
    collective(op, mine, [&all](const uint64_t *v, int) {
        std::memcpy(all, v, sizeof(all));
        return (uint64_t)0;
    });
}
}  // namespace emu

// ldmatrix.sync.aligned.m8n8.x4.shared.b16: lanes 8 m .. 8 m + 7 give the 16-byte rows of matrix m; register m of
// lane l is 32-bit word l % 4 of row l / 4 of matrix m
inline void emu_ldsm_x4(const uint32_t *row, uint32_t (&a)[4])
{
    if (reinterpret_cast<uintptr_t>(row) & 15u) { fprintf(stderr, "mma_emu: ldmatrix row not 16-byte aligned\n"); abort(); }
    uint64_t rows[emu::kLanes];
    emu::gather_lanes(emu::OP_LDSM, (uint64_t)reinterpret_cast<uintptr_t>(row), rows);
    const int me = emu::warp().cur;
    for (int m = 0; m < 4; ++m) a[m] = reinterpret_cast<const uint32_t *>((uintptr_t)rows[8 * m + me / 4])[me % 4];
}

// mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc: D = C + popc(A AND B) over k, with the PTX fragments
// (g = lane / 4, t = lane % 4): a0 / a1 = rows g / g + 8, k-word t; a2 / a3 = the same rows, k-word t + 4;
// b0 / b1 = column g, k-words t / t + 4; d0, d1 = row g, columns 2 t, 2 t + 1; d2, d3 = row g + 8
inline void emu_bmma_and_popc(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    uint64_t a01[emu::kLanes], a23[emu::kLanes], b[emu::kLanes];
    emu::gather_lanes(emu::OP_MMA, a[0] | (uint64_t)a[1] << 32, a01);
    emu::gather_lanes(emu::OP_MMA, a[2] | (uint64_t)a[3] << 32, a23);
    emu::gather_lanes(emu::OP_MMA, b0 | (uint64_t)b1 << 32, b);
    const int me = emu::warp().cur, g = me >> 2, t = me & 3;
    for (int i = 0; i < 4; ++i) {
        const int row = g + (i >= 2 ? 8 : 0), col = 2 * t + (i & 1), sh = row < 8 ? 0 : 32;
        int sum = 0;
        for (int kt = 0; kt < 4; ++kt) {
            const int la = (row & 7) * 4 + kt, lb = col * 4 + kt;
            sum += __builtin_popcount((uint32_t)(a01[la] >> sh) & (uint32_t)b[lb]) +
                   __builtin_popcount((uint32_t)(a23[la] >> sh) & (uint32_t)(b[lb] >> 32));
        }
        c[i] += sum;
    }
}
