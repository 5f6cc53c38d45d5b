// kao_bound.hpp — a tight upper bound on the objective of the 0/1 program (README.md:144-185), computed on the
// host from the assignment the search returned.  It is what lets kao_solve say "proven optimal": the search
// is a heuristic and never claims more than a bound shows (kao_result.objective_bound / .optimal).
//
// With y[p,b] = x[b,p] + l[b,p] (a replica of p on b, leader or not) the objective is
//     sum wF[p,b] y[p,b]  +  sum (wL[p,b] - wF[p,b]) l[b,p],
// and every feasible assignment is feasible for the two relaxations below, which no longer see each other
// (the coupling l <= y is dropped):
//   Y  max sum wF y      s.t. C1 (row sums RF), C3 (broker totals), C6 (rack totals), C7 (per partition and rack), 0 <= y <= 1
//   L  max sum (wL-wF) l s.t. C2 (one leader per partition), C4 (leaders per broker),                           0 <= l <= 1
// Both are network flow problems (integral polytopes), so  Y* + L*  is an upper bound on the optimum of the
// 0/1 program — the one lp_solve returns (README.md:135-136).  On the BASELINE configs it equals the optimum
// for configs 1-3 and is 3 above it for config 4 (tests/test_gpu_configs.py).  Each relaxation is solved by
// cancelling negative cycles in the residual graph of the flow that the search's own (feasible) assignment
// induces: when the search is at the relaxation's optimum there is no such cycle and one Bellman-Ford pass
// proves it; otherwise every cancelled cycle raises the bound by at least 1.
#pragma once
#include "kao_host.hpp"

#include <cstdint>
#include <vector>

namespace kao {

class Circulation {
public:
    explicit Circulation(int nodes) : first_(nodes, -1) {}
    // arc u -> v carrying `flow` units, low <= flow <= cap, `cost` per unit (costs are minimised)
    void add(int u, int v, int low, int cap, int cost, int flow)
    {
        push(u, v, cap - flow, cost);       // even index: forward residual
        push(v, u, flow - low, -cost);      // odd index: backward residual (the pair is a ^ 1)
    }
    // cancels negative cycles until none is left; returns the total cost change (<= 0) or 1 if `max_cycles` ran out
    long long minimise(int max_cycles)
    {
        long long delta = 0;
        const int n = (int)first_.size();
        std::vector<long long> dist(n);
        std::vector<int> parent(n), mark(n);
        for (int cycles = 0;; ++cycles) {
            std::fill(dist.begin(), dist.end(), 0);             // a virtual source reaches every node at cost 0
            std::fill(parent.begin(), parent.end(), -1);
            int on_cycle = -1;
            for (int round = 0; round < n && on_cycle < 0; ++round) {
                bool relaxed = false;
                for (int u = 0; u < n; ++u)
                    for (int a = first_[u]; a >= 0; a = next_[a])
                        if (res_[a] > 0 && dist[u] + cost_[a] < dist[to_[a]]) {
                            dist[to_[a]] = dist[u] + cost_[a];
                            parent[to_[a]] = a;
                            relaxed = true;
                        }
                if (!relaxed) return delta;                     // potentials exist: the flow is optimal
                // a cycle in the predecessor graph is a negative cycle of the residual graph
                std::fill(mark.begin(), mark.end(), 0);
                for (int s = 0; s < n && on_cycle < 0; ++s) {
                    if (mark[s]) continue;
                    int v = s;
                    while (v >= 0 && !mark[v]) { mark[v] = s + 1; v = parent[v] >= 0 ? to_[parent[v] ^ 1] : -1; }
                    if (v >= 0 && mark[v] == s + 1) on_cycle = v;
                }
            }
            if (on_cycle < 0) return delta;                     // n rounds without a cycle cannot happen; be safe
            if (cycles >= max_cycles) return 1;
            int push_units = INT32_MAX;
            long long cyc_cost = 0;
            for (int v = on_cycle;;) {
                const int a = parent[v];
                push_units = res_[a] < push_units ? res_[a] : push_units;
                cyc_cost += cost_[a];
                v = to_[a ^ 1];
                if (v == on_cycle) break;
            }
            for (int v = on_cycle;;) {
                const int a = parent[v];
                res_[a] -= push_units;
                res_[a ^ 1] += push_units;
                v = to_[a ^ 1];
                if (v == on_cycle) break;
            }
            delta += cyc_cost * push_units;
        }
    }

private:
    void push(int u, int v, int res, int cost)
    {
        to_.push_back(v); res_.push_back(res); cost_.push_back(cost);
        next_.push_back(first_[u]);
        first_[u] = (int)to_.size() - 1;
    }
    std::vector<int> first_, next_, to_, res_, cost_;
};

// replicas: a FEASIBLE assignment (violation 0), [P*RF] dense broker indices, leader first.  Returns Y* + L*, or
// the cheap per-partition bound when the flow bound cannot be had (an infeasible start, a runaway).
inline int64_t objective_flow_bound(const HostModel &m, const kao_problem &pb, const int32_t *replicas, int64_t cheap_bound)
{
    // per-partition rows (docs/MODEL.md §11): row p holds rf(p) replicas, the rest of its RF entries are -1
    const int P = m.P, B = m.B, R = m.R, RF = m.RF;
    std::vector<char> y((size_t)P * B, 0);
    std::vector<int> on_broker(B, 0), on_rack(R, 0), led(B, 0), ppr((size_t)P * R, 0);
    int64_t y_value = 0, l_value = 0, total = 0;
    for (int p = 0; p < P; ++p) {
        total += m.rf(p);
        for (int i = m.rf(p); i < RF; ++i)
            if (replicas[(size_t)p * RF + i] != -1) return cheap_bound;
        for (int i = 0; i < m.rf(p); ++i) {
            const int b = replicas[(size_t)p * RF + i];
            if (b < 0 || b >= B || y[(size_t)p * B + b]) return cheap_bound;
            y[(size_t)p * B + b] = 1;
            ++on_broker[b]; ++on_rack[m.rack_of[b]]; ++ppr[(size_t)p * R + m.rack_of[b]];
            y_value += pb.wF[(size_t)p * B + b];
        }
        const int lb = replicas[(size_t)p * RF];
        ++led[lb];
        l_value += (int64_t)pb.wL[(size_t)p * B + lb] - pb.wF[(size_t)p * B + lb];
    }
    // ---- Y: S -> partition -> (partition, rack) -> broker -> rack -> T -> S
    {
        const int S = 0, T = 1, nP = 2, nPR = nP + P, nB = nPR + P * R, nR = nB + B;
        Circulation g(nR + R);
        g.add(T, S, (int)total, (int)total, 0, (int)total);
        for (int p = 0; p < P; ++p) {
            g.add(S, nP + p, m.rf(p), m.rf(p), 0, m.rf(p));
            for (int r = 0; r < R; ++r) g.add(nP + p, nPR + p * R + r, m.plo(p), m.phi(p), 0, ppr[(size_t)p * R + r]);
            for (int b = 0; b < B; ++b)
                g.add(nPR + p * R + m.rack_of[b], nB + b, 0, 1, -(int)pb.wF[(size_t)p * B + b], y[(size_t)p * B + b]);
        }
        for (int b = 0; b < B; ++b) g.add(nB + b, nR + m.rack_of[b], pb.rep_lo[b], pb.rep_hi[b], 0, on_broker[b]);
        for (int r = 0; r < R; ++r) g.add(nR + r, T, m.rack_lo[r], m.rack_hi[r], 0, on_rack[r]);
        const long long d = g.minimise(4096);
        if (d > 0) return cheap_bound;
        y_value -= d;
    }
    // ---- L: S -> partition -> broker -> T -> S
    {
        const int S = 0, T = 1, nP = 2, nB = nP + P;
        Circulation g(nB + B);
        g.add(T, S, P, P, 0, P);
        for (int p = 0; p < P; ++p) {
            g.add(S, nP + p, 1, 1, 0, 1);
            const int lb = replicas[(size_t)p * RF];
            for (int b = 0; b < B; ++b)
                g.add(nP + p, nB + b, 0, 1, (int)pb.wF[(size_t)p * B + b] - (int)pb.wL[(size_t)p * B + b], b == lb ? 1 : 0);
        }
        for (int b = 0; b < B; ++b) g.add(nB + b, T, pb.ldr_lo[b], pb.ldr_hi[b], 0, led[b]);
        const long long d = g.minimise(4096);
        if (d > 0) return cheap_bound;
        l_value -= d;
    }
    const int64_t bound = y_value + l_value;
    return bound < cheap_bound ? bound : cheap_bound;
}

}  // namespace kao
