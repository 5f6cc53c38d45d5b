// kao_lagrange.hpp — host interface of the Lagrangian LP bound (docs/MODEL.md §9, kernel in kao_lagrange.cu): an
// upper bound on the objective of every feasible assignment, as tight as the LP relaxation of the whole 0/1
// program, where the flow bound of kao_bound.hpp is not.
#pragma once
#include "../../include/kao.h"

#include <cstdint>
#include <string>
#include <vector>

namespace kao {

// The objective of `replicas` ([P*RF] dense broker indices, leader first) when it satisfies C1..C7; false with
// the reason otherwise.  The iteration of MODEL §9 aims at this value (its T).
inline bool feasible_objective(const kao_problem &pb, const int32_t *replicas, int64_t &objective, std::string &why)
{
    const int P = pb.P, B = pb.B, R = pb.R, RF = pb.RF;
    std::vector<int64_t> on_broker(B, 0), led(B, 0), on_rack(R, 0);
    std::vector<int> in_rack(R, 0);
    objective = 0;
    for (int p = 0; p < P; ++p) {
        const int32_t *row = replicas + (size_t)p * RF;
        std::fill(in_rack.begin(), in_rack.end(), 0);
        for (int i = 0; i < RF; ++i) {
            const int b = row[i];
            if (b < 0 || b >= B) { why = "replicas: partition " + std::to_string(p) + " has fewer than RF replicas on target brokers (C1)"; return false; }
            for (int k = 0; k < i; ++k)
                if (row[k] == b) { why = "replicas: partition " + std::to_string(p) + " holds broker " + std::to_string(b) + " twice (C5)"; return false; }
            ++on_broker[b]; ++on_rack[pb.rack_of[b]]; ++in_rack[pb.rack_of[b]];
            objective += i == 0 ? pb.wL[(size_t)p * B + b] : pb.wF[(size_t)p * B + b];
        }
        ++led[row[0]];
        for (int r = 0; r < R; ++r)
            if (in_rack[r] < pb.ppr_lo || in_rack[r] > pb.ppr_hi) { why = "replicas: partition " + std::to_string(p) + " violates C7"; return false; }
    }
    for (int b = 0; b < B; ++b) {
        if (on_broker[b] < pb.rep_lo[b] || on_broker[b] > pb.rep_hi[b]) { why = "replicas: broker " + std::to_string(b) + " violates C3"; return false; }
        if (led[b] < pb.ldr_lo[b] || led[b] > pb.ldr_hi[b]) { why = "replicas: broker " + std::to_string(b) + " violates C4"; return false; }
    }
    for (int r = 0; r < R; ++r)
        if (on_rack[r] < pb.rack_lo[r] || on_rack[r] > pb.rack_hi[r]) { why = "replicas: rack " + std::to_string(r) + " violates C6"; return false; }
    return true;
}

// Runs the integer iteration of MODEL §9 on `device` in one cooperative launch, aiming at T (the objective of a
// feasible assignment).  bound = floor(min L / 2^KAO_LP_FRACTION_BITS), iterations_run, multipliers (optional,
// [2B + R], the ones of the minimum), device_ms = CUDA-event time of the kernel.  pb must have passed
// build_host_model.  KAO_OK, or KAO_E_CUDA / KAO_E_ARG with `why`.
int lagrange_bound_device(const kao_problem &pb, int device, int64_t T, uint32_t max_iterations,
                          unsigned long long timeout_ns, int64_t *bound, uint32_t *iterations_run,
                          int64_t *multipliers, double *device_ms, std::string &why);

}  // namespace kao
