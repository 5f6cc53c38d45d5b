// kao_leaders.hpp — leader-only rebalancing (docs/MODEL.md §13): every partition keeps its replica set, and only the
// choice of its leader among those replicas is free.  Host-side and exact, no GPU.
//
// With the replica sets fixed, C1, C3, C5, C6, C7 and C3t are constants (the "fixed violation"), C2 holds by
// construction, and what remains is a transportation problem on a laminar family: partition -> (topic, broker) cell
// -> broker -> sink, one unit per partition, the C4t band on every cell arc, the C4 band on every broker arc, and
// choice arcs of cost -(wL - wF)[p, b].  A band is convex in its count, so each band arc is a set of parallel arcs: lo
// of them at -M, hi - lo at 0, the rest at +M.  M exceeds the largest objective gain any change of leaders can make,
// so the min-cost flow is the lexicographic optimum: least violation of C4 / C4t first, then the largest objective.
//
// The flow is solved by cancelling negative cycles from the current leaders.  The residual graph is collapsed to
// cells, brokers and the sink: the partitions led from cell c that could be led from cell c' form one arc c -> c'
// whose cost is the cheapest of them (a set per pair keeps them, so a cancelled cycle names its partitions), and the
// parallel band arcs of a cell or broker become one arc up (the next unit's marginal cost) and one arc down (minus the
// last unit's).  Single-partition moves are cancelled first in sweeps over the partitions; then Bellman-Ford passes
// cancel every cycle of the predecessor graph at once.  A pass that relaxes nothing proves that no negative cycle is
// left: the flow, so the leader choice, is optimal.  Every order (partitions, choices, arcs, ties) is fixed by the
// input, so the same input gives the same lists.
#pragma once
#include "kao_host.hpp"

#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdlib>
#include <set>
#include <string>
#include <utility>
#include <vector>

namespace kao {

struct LeaderPlan {
    std::vector<int32_t> replicas;            // [P*RF]: the chosen leader, the row's other replicas in cur order, -1 padded
    int64_t violation = 0, fixed_violation = 0, objective = 0;
};

// Validates pb, the rows and tp (as kao_create_topics does) and solves; false with `why` on a refusal.
inline bool solve_leaders(const kao_problem &pb, const kao_topics *tp, const uint8_t *fixed, LeaderPlan &out,
                          std::string &why)
{
    HostModel hm;
    if (!build_host_model(pb, hm, why)) return false;
    const int P = pb.P, B = pb.B, R = pb.R, RF = pb.RF, RFc = pb.RFcur;
    // ---- the rows: each a non-empty list of distinct target brokers, at most RF of them, before any -1 padding
    std::vector<int> first((size_t)P + 1, 0);
    std::vector<int> rb;                                    // brokers of every row, in cur order
    rb.reserve((size_t)P * RF);
    for (int p = 0; p < P; ++p) {
        first[p] = (int)rb.size();
        const int32_t *row = pb.cur + (size_t)p * RFc;
        const std::string at = "leaders only: partition " + std::to_string(p);
        bool gap = false;
        for (int i = 0; i < RFc; ++i) {
            if (row[i] < 0) { gap = true; continue; }
            if (row[i] >= B) { why = at + " names broker " + std::to_string(row[i]) + ", not a dense index 0..B-1"; return false; }
            if (gap) {
                why = at + " has a replica on a broker outside the target list (entry " + std::to_string(i) +
                      " follows a -1): its data would have to move";
                return false;
            }
            for (int k = first[p]; k < (int)rb.size(); ++k)
                if (rb[k] == row[i]) { why = at + " names broker " + std::to_string(row[i]) + " twice"; return false; }
            rb.push_back(row[i]);
        }
        const int n = (int)rb.size() - first[p];
        if (n == 0) { why = at + " has no replica"; return false; }
        if (n > RF) { why = at + " has " + std::to_string(n) + " replicas, more than RF = " + std::to_string(RF); return false; }
    }
    first[P] = (int)rb.size();
    HostTopics ht;
    if (tp && !build_host_topics(pb, *tp, hm.Ppad, ht, why)) return false;
    const int T = tp ? tp->T : 1;
    auto topic = [&](int p) { return tp ? (int)tp->topic_of[p] : 0; };
    auto gain = [&](int p, int b) { return (int64_t)pb.wL[(size_t)p * B + b] - pb.wF[(size_t)p * B + b]; };
    auto is_fixed = [&](int p) { return fixed && fixed[p]; };

    // ---- the constant rows: C1 (row length against RF), C7, C3, C6 and C3t; C2 and C5 hold by construction
    out.fixed_violation = 0;
    int64_t base_objective = 0;                             // the follower weight of every replica
    {
        std::vector<int64_t> on_broker(B, 0), on_rack(R, 0), in_rack(R, 0);
        std::vector<std::pair<int, int>> tb;                // (topic, broker) of every replica
        tb.reserve(rb.size());
        for (int p = 0; p < P; ++p) {
            std::fill(in_rack.begin(), in_rack.end(), 0);
            out.fixed_violation += std::abs(first[p + 1] - first[p] - RF);
            for (int k = first[p]; k < first[p + 1]; ++k) {
                ++on_broker[rb[k]]; ++on_rack[pb.rack_of[rb[k]]]; ++in_rack[pb.rack_of[rb[k]]];
                base_objective += pb.wF[(size_t)p * B + rb[k]];
                if (tp) tb.emplace_back(topic(p), rb[k]);
            }
            for (int r = 0; r < R; ++r) out.fixed_violation += band(in_rack[r], pb.ppr_lo, pb.ppr_hi);
        }
        for (int b = 0; b < B; ++b) out.fixed_violation += band(on_broker[b], pb.rep_lo[b], pb.rep_hi[b]);
        for (int r = 0; r < R; ++r) out.fixed_violation += band(on_rack[r], pb.rack_lo[r], pb.rack_hi[r]);
        if (tp) {
            std::sort(tb.begin(), tb.end());
            std::vector<int> cells(T, 0);                   // (topic, broker) cells holding a replica, per topic
            for (size_t i = 0; i < tb.size();) {
                size_t j = i;
                while (j < tb.size() && tb[j] == tb[i]) ++j;
                out.fixed_violation += band((int64_t)(j - i), tp->rep_lo[tb[i].first], tp->rep_hi[tb[i].first]);
                ++cells[tb[i].first];
                i = j;
            }
            for (int t = 0; t < T; ++t) out.fixed_violation += (int64_t)(B - cells[t]) * tp->rep_lo[t];
        }
    }

    // ---- cells: (topic, broker) pairs some row can be led from; choice k of row p leads it from cell cell_of[k]
    std::vector<int64_t> keys(rb.size());
    for (int p = 0; p < P; ++p)
        for (int k = first[p]; k < first[p + 1]; ++k) keys[k] = (int64_t)topic(p) * B + rb[k];
    std::vector<int64_t> cell_key(keys);
    std::sort(cell_key.begin(), cell_key.end());
    cell_key.erase(std::unique(cell_key.begin(), cell_key.end()), cell_key.end());
    const int C = (int)cell_key.size();
    std::vector<int> cell_of(rb.size());
    for (size_t k = 0; k < rb.size(); ++k)
        cell_of[k] = (int)(std::lower_bound(cell_key.begin(), cell_key.end(), keys[k]) - cell_key.begin());
    auto cell_broker = [&](int c) { return (int)(cell_key[c] % B); };
    auto cell_topic = [&](int c) { return (int)(cell_key[c] / B); };
    // the cells of every broker (the broker's down arcs), ascending
    std::vector<int> bc_first(B + 1, 0), bc(C);
    for (int c = 0; c < C; ++c) ++bc_first[cell_broker(c) + 1];
    for (int b = 0; b < B; ++b) bc_first[b + 1] += bc_first[b];
    {
        std::vector<int> fill(bc_first.begin(), bc_first.end() - 1);
        for (int c = 0; c < C; ++c) bc[fill[cell_broker(c)]++] = c;
    }

    // ---- the current leaders, and M: one more than the largest gain a change of leaders can make
    std::vector<int> choice(P, 0);                          // index into the row: 0 = the current leader
    std::vector<int64_t> cnt(C, 0), lcnt(B, 0);
    int64_t M = 1;
    for (int p = 0; p < P; ++p) {
        ++cnt[cell_of[first[p]]];
        ++lcnt[rb[first[p]]];
        if (is_fixed(p)) continue;
        int64_t lo = INT64_MAX, hi = INT64_MIN;
        for (int k = first[p]; k < first[p + 1]; ++k) { lo = std::min(lo, gain(p, rb[k])); hi = std::max(hi, gain(p, rb[k])); }
        M += hi - lo;
    }
    const int64_t NOHI = INT64_MAX / 4;
    auto cell_lo = [&](int c) { return tp ? (int64_t)tp->ldr_lo[cell_topic(c)] : 0; };
    auto cell_hi = [&](int c) { return tp ? (int64_t)tp->ldr_hi[cell_topic(c)] : NOHI; };
    // marginal cost of the unit k -> k + 1 of a band [lo, hi]
    auto marg = [&](int64_t k, int64_t lo, int64_t hi) { return k < lo ? -M : k < hi ? 0 : M; };
    auto cell_up = [&](int c) { return marg(cnt[c], cell_lo(c), cell_hi(c)); };
    auto cell_down = [&](int c) { return -marg(cnt[c] - 1, cell_lo(c), cell_hi(c)); };
    auto brk_up = [&](int b) { return marg(lcnt[b], pb.ldr_lo[b], pb.ldr_hi[b]); };
    auto brk_down = [&](int b) { return -marg(lcnt[b] - 1, pb.ldr_lo[b], pb.ldr_hi[b]); };
    // units an arc takes before its cost changes (up: to the next breakpoint; down: back to the previous one)
    auto room_up = [&](int64_t k, int64_t lo, int64_t hi) { return k < lo ? lo - k : k < hi ? hi - k : NOHI; };
    auto room_down = [&](int64_t k, int64_t lo, int64_t hi) { return k > hi ? k - hi : k > lo ? k - lo : k; };

    // ---- sweeps of single-partition moves: a row moves to the choice of lowest cost change when that is negative
    auto move_cost = [&](int p, int from, int to) {
        const int c0 = cell_of[from], c1 = cell_of[to], b0 = rb[from], b1 = rb[to];
        return cell_down(c0) + cell_up(c1) + brk_down(b0) + brk_up(b1) + gain(p, b0) - gain(p, b1);
    };
    auto lead = [&](int p, int to) {                        // row p is led from its choice `to` (an index into rb)
        const int from = first[p] + choice[p];
        --cnt[cell_of[from]]; --lcnt[rb[from]];
        ++cnt[cell_of[to]]; ++lcnt[rb[to]];
        choice[p] = to - first[p];
    };
    for (bool changed = true; changed;) {
        changed = false;
        for (int p = 0; p < P; ++p) {
            if (is_fixed(p) || first[p + 1] - first[p] < 2) continue;
            const int from = first[p] + choice[p];
            int best = -1;
            int64_t best_cost = 0;
            for (int k = first[p]; k < first[p + 1]; ++k) {
                if (k == from) continue;
                const int64_t d = move_cost(p, from, k);
                if (d < best_cost) { best_cost = d; best = k; }
            }
            if (best >= 0) { lead(p, best); changed = true; }
        }
    }

    // ---- the collapsed partition arcs: pair (c, c') holds (cost, row) for every row led from c that can be led from c'
    std::vector<std::pair<int, int>> pk;                    // (c, c') of every pair
    for (int p = 0; p < P; ++p) {
        if (is_fixed(p)) continue;
        for (int i = first[p]; i < first[p + 1]; ++i)
            for (int j = first[p]; j < first[p + 1]; ++j)
                if (i != j) pk.emplace_back(cell_of[i], cell_of[j]);
    }
    std::sort(pk.begin(), pk.end());
    pk.erase(std::unique(pk.begin(), pk.end()), pk.end());
    std::vector<int> pair_first(C + 1, 0);                  // pairs out of cell c: pair_first[c] .. pair_first[c + 1]
    for (const auto &e : pk) ++pair_first[e.first + 1];
    for (int c = 0; c < C; ++c) pair_first[c + 1] += pair_first[c];
    auto pair_id = [&](int c, int c2) {
        return (int)(std::lower_bound(pk.begin() + pair_first[c], pk.begin() + pair_first[c + 1], std::make_pair(c, c2)) - pk.begin());
    };
    std::vector<std::set<std::pair<int64_t, int>>> in_pair(pk.size());
    auto enter = [&](int p, bool add) {                     // row p joins / leaves the pairs out of its leader's cell
        const int from = first[p] + choice[p];
        for (int k = first[p]; k < first[p + 1]; ++k) {
            if (k == from) continue;
            const std::pair<int64_t, int> e(gain(p, rb[from]) - gain(p, rb[k]), p);
            auto &s = in_pair[pair_id(cell_of[from], cell_of[k])];
            if (add) s.insert(e); else s.erase(e);
        }
    };
    for (int p = 0; p < P; ++p)
        if (!is_fixed(p) && first[p + 1] - first[p] > 1) enter(p, true);
    auto target = [&](int p, int c2) {                      // the choice of row p in cell c2
        for (int k = first[p]; k < first[p + 1]; ++k) if (cell_of[k] == c2) return k;
        return -1;
    };

    // ---- Bellman-Ford passes over nodes 0..C-1 (cells), C..C+B-1 (brokers), C+B (sink); parent arc of node v:
    // kind 0 = pair (id in pa), 1 = up (cell -> broker, broker -> sink), 2 = down (broker -> cell, sink -> broker)
    const int N = C + B + 1, SINK = C + B;
    std::vector<int64_t> dist(N);
    std::vector<int> par(N), pkind(N), pa(N), mark(N);
    auto arc_cost = [&](int u, int v, int kind, int id) -> int64_t {
        if (kind == 0) return in_pair[id].begin()->first;
        if (kind == 1) return u < C ? cell_up(u) : brk_up(u - C);
        return v < C ? cell_down(v) : brk_down(v - C);
    };
    for (;;) {
        std::fill(dist.begin(), dist.end(), 0);
        std::fill(par.begin(), par.end(), -1);
        bool relaxed = true;
        std::vector<int> cyc;                               // a node on each cycle of the predecessor graph
        for (int pass = 0; pass <= N && relaxed && cyc.empty(); ++pass) {
            relaxed = false;
            auto relax = [&](int u, int v, int64_t w, int kind, int id) {
                if (dist[u] + w < dist[v]) { dist[v] = dist[u] + w; par[v] = u; pkind[v] = kind; pa[v] = id; relaxed = true; }
            };
            for (int c = 0; c < C; ++c) {
                for (int id = pair_first[c]; id < pair_first[c + 1]; ++id)
                    if (!in_pair[id].empty()) relax(c, pk[id].second, in_pair[id].begin()->first, 0, id);
                relax(c, C + cell_broker(c), cell_up(c), 1, -1);
            }
            for (int b = 0; b < B; ++b) {
                relax(C + b, SINK, brk_up(b), 1, -1);
                for (int i = bc_first[b]; i < bc_first[b + 1]; ++i)
                    if (cnt[bc[i]] > 0) relax(C + b, bc[i], cell_down(bc[i]), 2, -1);
                if (lcnt[b] > 0) relax(SINK, C + b, brk_down(b), 2, -1);
            }
            std::fill(mark.begin(), mark.end(), 0);
            for (int s = 0; s < N; ++s) {
                int v = s;
                while (v >= 0 && !mark[v]) { mark[v] = s + 1; v = par[v]; }
                if (v >= 0 && mark[v] == s + 1) cyc.push_back(v);
            }
        }
        if (cyc.empty()) break;                             // no negative cycle: the leader choice is optimal
        // cancel every cycle of the predecessor graph: they share no node, so no arc or pair
        for (int s : cyc) {
            std::vector<int> nodes;
            int64_t cost = 0, units = NOHI;
            for (int v = s;;) {
                nodes.push_back(v);
                const int u = par[v], kind = pkind[v];
                cost += arc_cost(u, v, kind, pa[v]);
                if (kind == 0) {
                    const auto &st = in_pair[pa[v]];
                    int64_t same = 0;
                    for (auto it = st.begin(); it != st.end() && it->first == st.begin()->first && same < units; ++it) ++same;
                    units = std::min(units, same);
                } else if (kind == 1) {
                    units = std::min(units, u < C ? room_up(cnt[u], cell_lo(u), cell_hi(u))
                                                  : room_up(lcnt[u - C], pb.ldr_lo[u - C], pb.ldr_hi[u - C]));
                } else {
                    units = std::min(units, v < C ? room_down(cnt[v], cell_lo(v), cell_hi(v))
                                                  : room_down(lcnt[v - C], pb.ldr_lo[v - C], pb.ldr_hi[v - C]));
                }
                v = u;
                if (v == s) break;
            }
            if (cost >= 0) continue;
            // the rows each pair arc moves, chosen before any of them moves
            std::vector<std::pair<int, int>> moves;         // (row, choice it is led from next)
            for (int v : nodes) {
                if (pkind[v] != 0) continue;
                auto it = in_pair[pa[v]].begin();
                for (int64_t k = 0; k < units; ++k, ++it) moves.emplace_back(it->second, target(it->second, v));
            }
            for (const auto &mv : moves) { enter(mv.first, false); lead(mv.first, mv.second); enter(mv.first, true); }
        }
    }

    // ---- the plan: leader first, the other replicas in cur order
    out.replicas.assign((size_t)P * RF, -1);
    out.objective = base_objective;
    int64_t free_violation = 0;
    for (int p = 0; p < P; ++p) {
        int32_t *row = &out.replicas[(size_t)p * RF];
        const int lk = first[p] + choice[p];
        int n = 0;
        row[n++] = rb[lk];
        for (int k = first[p]; k < first[p + 1]; ++k) if (k != lk) row[n++] = rb[k];
        out.objective += gain(p, rb[lk]);
    }
    for (int b = 0; b < B; ++b) free_violation += band(lcnt[b], pb.ldr_lo[b], pb.ldr_hi[b]);
    if (tp) {
        std::vector<int> cells(T, 0);
        for (int c = 0; c < C; ++c) { free_violation += band(cnt[c], cell_lo(c), cell_hi(c)); ++cells[cell_topic(c)]; }
        for (int t = 0; t < T; ++t) free_violation += (int64_t)(B - cells[t]) * tp->ldr_lo[t];
    }
    out.violation = out.fixed_violation + free_violation;
    return true;
}

}  // namespace kao
