// kao_host.hpp — host-side preparation of a kao_problem for the device engine: validation,
// rack-aligned slot layout (docs/MODEL.md §2), weight-table compaction, bounds in slot space,
// the initial base (docs/MODEL.md §4) and replica-list <-> bit-plane conversion.
// Model citations: /root/reference/README.md:139-185.
#pragma once
#include "../../include/kao.h"

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

namespace kao {

struct HostModel {
    int P = 0, B = 0, R = 0, RF = 0, RFcur = 0;
    int S = 0, log2S = 0, NS = 0, W = 0, Ppad = 0;
    int ppr_lo = 0, ppr_hi = 0;
    bool dense = false;
    std::vector<int> slot_of_broker, broker_of_slot, slot_of_order, order_of_slot;
    std::vector<uint8_t> rack_of;
    std::vector<int32_t> cur;                 // [P*RFcur]
    std::vector<int32_t> rack_lo, rack_hi;
    std::vector<uint32_t> bnd_rep, bnd_ldr;   // [256] lo | hi << 16 in slot space
    std::vector<uint32_t> swT;                // [4][Ppad]
    int nentries = 0;                         // entries per partition in use
    // weighted mask planes (docs/MODEL.md §3.2): objective = sum_c value_c * popc(part_c & M_c[p])
    int nplanes = 0, plane_on_leader = 0;
    int plane_value[6] = {0, 0, 0, 0, 0, 0};
    std::vector<uint32_t> planesT;            // [nplanes][W][Ppad]
    // sparse objective of the column-major evaluator (docs/MODEL.md §3.3): the non-zero terms of the objective
    // row (README.md:145-146 lists exactly these) grouped into nz <= 8 TERM PLANES — all terms of a plane share
    // one value and one kind (follower weight on the replica bit / leader bonus wL - wF on the leader bit) and a
    // partition has at most one term per plane: objective = sum_j z_value[j] * |{p : term j of p holds}|
    bool z_ok = false;                        // the term planes below describe the whole objective
    int nz = 0, z_on_leader = 0;
    int z_value[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    std::vector<uint8_t> zslot;               // [Ppad][8] slot of partition p's term in plane j, 0xFF = none
    bool hi1 = false;                         // C7 is exactly "at most one replica per rack"
    int key_obj_bits = 24;                    // width of the cost field of a packed key (docs/MODEL.md 3)
    std::vector<uint32_t> dense_w;            // [P][NS] when dense
    struct Cell { int p, b; uint32_t f, l; }; // a non-zero cell of the weight tables: follower / leader weight of (p, broker)
    std::vector<Cell> cells;                  // all of them, by partition then broker
    std::vector<int> cell_first;              // [P + 1] cells of partition p: cell_first[p] .. cell_first[p + 1]
    std::vector<uint32_t> homeT;              // [Ppad]
    // per-partition C1 / C7 rows (kao_replication, docs/MODEL.md §11); empty: RF and ppr_lo .. ppr_hi for every row
    std::vector<uint8_t> rf_p, ppr_lo_p, ppr_hi_p;
    int rf(int p) const { return rf_p.empty() ? RF : rf_p[p]; }
    int plo(int p) const { return ppr_lo_p.empty() ? ppr_lo : ppr_lo_p[p]; }
    int phi(int p) const { return ppr_hi_p.empty() ? ppr_hi : ppr_hi_p[p]; }
};

inline bool build_host_model(const kao_problem &pb, HostModel &m, std::string &why)
{
    auto bad = [&](const char *s) { why = s; return false; };
    // 65,280: the largest multiple of 256 below 2^16 (u16 partition ids and their 0xFFFF sentinel); above 8,160
    // partitions the engine searches with the base in HBM (kao_large.cu)
    if (pb.P < 1 || pb.P > 65280) return bad("P must be 1..65280");
    if (pb.B < 2 || pb.B > KAO_MAX_SLOTS) return bad("B must be 2..256");
    if (pb.R < 1 || pb.R > KAO_MAX_RACKS) return bad("R must be 1..32");
    if (pb.RF < 1 || pb.RF > KAO_MAX_RF || pb.RF >= pb.B) return bad("RF must be 1..8 and < B");
    if (pb.RFcur < 1 || pb.RFcur > 64) return bad("RFcur must be 1..64");
    if (!pb.rack_of || !pb.wF || !pb.wL || !pb.rep_lo || !pb.rep_hi || !pb.ldr_lo || !pb.ldr_hi ||
        !pb.rack_lo || !pb.rack_hi || !pb.cur)
        return bad("null table pointer");
    if (pb.ppr_lo < 0 || pb.ppr_lo > pb.ppr_hi || pb.ppr_hi > 127) return bad("bad per-partition-per-rack bounds");
    m.P = pb.P; m.B = pb.B; m.R = pb.R; m.RF = pb.RF; m.RFcur = pb.RFcur;
    m.ppr_lo = pb.ppr_lo; m.ppr_hi = pb.ppr_hi;
    m.rack_of.assign(pb.rack_of, pb.rack_of + pb.B);
    std::vector<int> size(pb.R, 0);
    for (int b = 0; b < pb.B; ++b) {
        if (m.rack_of[b] >= pb.R) return bad("rack_of entry out of range");
        ++size[m.rack_of[b]];
    }
    // rack-aligned slots: slot = rack * S + rank in rack, S = pow2 >= max(8, largest rack)
    int S = 8, lg = 3;
    const int largest = *std::max_element(size.begin(), size.end());
    while (S < largest) { S <<= 1; ++lg; }
    m.S = S; m.log2S = lg; m.NS = pb.R * S;
    if (m.NS > KAO_MAX_SLOTS) return bad("racks * pow2ceil(max(8, largest rack)) exceeds 256 slots");
    int W = 1;
    while (W * 32 < m.NS) W <<= 1;
    m.W = W;
    m.Ppad = (pb.P + 255) / 256 * 256;
    m.slot_of_broker.assign(pb.B, -1);
    m.broker_of_slot.assign(256, -1);
    m.slot_of_order.assign(256, 0);
    m.order_of_slot.assign(256, -1);
    {
        std::vector<int> rank(pb.R, 0);
        for (int b = 0; b < pb.B; ++b) {
            const int s = m.rack_of[b] * S + rank[m.rack_of[b]]++;
            m.slot_of_broker[b] = s;
            m.broker_of_slot[s] = b;
        }
        int o = 0;
        for (int s = 0; s < m.NS; ++s)
            if (m.broker_of_slot[s] >= 0) { m.slot_of_order[o] = s; m.order_of_slot[s] = o; ++o; }
    }
    // bounds, slot space; padding slots keep [0,0] so a replica there violates C3
    m.bnd_rep.assign(256, 0);
    m.bnd_ldr.assign(256, 0);
    for (int b = 0; b < pb.B; ++b) {
        if (pb.rep_lo[b] < 0 || pb.rep_lo[b] > pb.rep_hi[b] || pb.rep_hi[b] > 65535 ||
            pb.ldr_lo[b] < 0 || pb.ldr_lo[b] > pb.ldr_hi[b] || pb.ldr_hi[b] > 65535)
            return bad("per-broker bounds must satisfy 0 <= lo <= hi <= 65535");
        m.bnd_rep[m.slot_of_broker[b]] = (uint32_t)pb.rep_lo[b] | ((uint32_t)pb.rep_hi[b] << 16);
        m.bnd_ldr[m.slot_of_broker[b]] = (uint32_t)pb.ldr_lo[b] | ((uint32_t)pb.ldr_hi[b] << 16);
    }
    m.rack_lo.assign(pb.rack_lo, pb.rack_lo + pb.R);
    m.rack_hi.assign(pb.rack_hi, pb.rack_hi + pb.R);
    for (int r = 0; r < pb.R; ++r)
        if (m.rack_lo[r] < 0 || m.rack_lo[r] > m.rack_hi[r]) return bad("rack bounds must satisfy 0 <= lo <= hi");
    m.cur.assign(pb.cur, pb.cur + (size_t)pb.P * pb.RFcur);
    for (int32_t &b : m.cur) if (b < 0 || b >= pb.B) b = -1;
    // weights.  The tables are P x B cells of which only the current placements are non-zero (README.md:145-146 lists
    // just those): ONE scan collects the non-zero cells, everything below works on that short list (kao_solve builds
    // the model once per call: at 1000 x 64 the scan is what its host-side set-up costs)
    m.cell_first.assign((size_t)pb.P + 1, 0);
    m.cells.clear();
    for (int p = 0; p < pb.P; ++p) {
        m.cell_first[p] = (int)m.cells.size();
        const uint16_t *f = pb.wF + (size_t)p * pb.B, *l = pb.wL + (size_t)p * pb.B;
        int b = 0;
        for (; b + 4 <= pb.B; b += 4) {
            uint64_t f4, l4;
            std::memcpy(&f4, f + b, 8);
            std::memcpy(&l4, l + b, 8);
            if ((f4 | l4) == 0) continue;
            for (int k = b; k < b + 4; ++k)
                if (f[k] | l[k]) m.cells.push_back({p, k, f[k], l[k]});
        }
        for (; b < pb.B; ++b)
            if (f[b] | l[b]) m.cells.push_back({p, b, f[b], l[b]});
    }
    m.cell_first[pb.P] = (int)m.cells.size();
    // at most 4 non-zero cells per partition and 12-bit values -> packed entries staged in shared memory; anything
    // else -> dense table in HBM
    uint32_t maxw = 0;
    bool sparse_ok = true;
    for (const HostModel::Cell &c : m.cells) {
        maxw = std::max<uint32_t>(maxw, std::max(c.f, c.l));
        if (c.f > 4095 || c.l > 4095) sparse_ok = false;
    }
    for (int p = 0; p < pb.P; ++p)
        if (m.cell_first[p + 1] - m.cell_first[p] > 4) sparse_ok = false;
    if ((uint64_t)pb.P * pb.RF * maxw > 0xFFFFFFull) return bad("objective range exceeds 24 bits");
    // cost field of the packed key: just wide enough for the largest objective the model can reach, so
    // that the violation field gets the rest of the 63 bits (ADVICE r1: 15 bits saturate at P = 8000)
    m.key_obj_bits = 1;
    while (((uint64_t)pb.P * pb.RF * maxw) >> m.key_obj_bits) ++m.key_obj_bits;
    m.dense = !sparse_ok;
    m.swT.assign((size_t)4 * m.Ppad, 0);
    m.nentries = 0;
    if (m.dense) {
        m.dense_w.assign((size_t)pb.P * m.NS, 0);
        for (const HostModel::Cell &c : m.cells)
            m.dense_w[(size_t)c.p * m.NS + m.slot_of_broker[c.b]] = c.f | (c.l << 16);
    } else {
        for (int p = 0; p < pb.P; ++p) {
            int k = 0;
            for (int i = m.cell_first[p]; i < m.cell_first[p + 1]; ++i, ++k) {
                const HostModel::Cell &c = m.cells[i];
                m.swT[(size_t)k * m.Ppad + p] = (uint32_t)m.slot_of_broker[c.b] | (c.f << 8) | (c.l << 20);
            }
            m.nentries = std::max(m.nentries, k);
        }
    }
    // mask planes: one per distinct follower weight (applied to the row) and one per distinct
    // leader bonus wL - wF (applied to the leader one-hot); needs wL >= wF everywhere, at most two
    // follower weights and one bonus value, and only pays off for narrow rows
    {
        std::vector<uint32_t> vf, vd;
        bool ok = (m.W <= 2);
        for (const HostModel::Cell &c : m.cells) {
            if (!ok) break;
            if (c.l < c.f) { ok = false; break; }
            if (c.f && std::find(vf.begin(), vf.end(), c.f) == vf.end()) vf.push_back(c.f);
            if (c.l - c.f && std::find(vd.begin(), vd.end(), c.l - c.f) == vd.end()) vd.push_back(c.l - c.f);
            if (vf.size() + vd.size() > 6) ok = false;
        }
        // kernels exist for 3 planes (2 row planes + 1 leader plane); empty planes pad; other weight
        // tables are scored from packed entries / the dense table
        if (ok && vf.size() + vd.size() > 0 && vf.size() <= 2 && vd.size() <= 1) {
            std::sort(vf.begin(), vf.end());
            std::sort(vd.begin(), vd.end());
            m.nplanes = 3;
            const int nrow = 2 * m.nplanes / 3;
            m.planesT.assign((size_t)m.nplanes * m.W * m.Ppad, 0);
            for (int c = 0; c < m.nplanes; ++c) {
                const bool on_leader = c >= nrow;
                const size_t k = on_leader ? (size_t)(c - nrow) : (size_t)c;
                if (k >= (on_leader ? vd.size() : vf.size())) continue;        // padding plane
                const uint32_t val = on_leader ? vd[k] : vf[k];
                m.plane_value[c] = (int)val;
                if (on_leader) m.plane_on_leader |= 1 << c;
                for (const HostModel::Cell &cl : m.cells)
                    if ((on_leader ? cl.l - cl.f : cl.f) == val) {
                        const int s = m.slot_of_broker[cl.b];
                        m.planesT[((size_t)c * m.W + (s >> 5)) * m.Ppad + cl.p] |= 1u << (s & 31);
                    }
            }
        }
    }
    // term planes: classes (kind, value) in ascending order, followers first; a class takes as many planes as
    // its largest number of terms in one partition (terms of a partition in ascending slot order)
    {
        struct Term { int kind; uint32_t val; int slot; };
        std::vector<std::pair<int, uint32_t>> classes;
        bool ok = true;
        for (const HostModel::Cell &c : m.cells) {
            if (c.l < c.f) { ok = false; break; }
            for (int kind = 0; kind < 2; ++kind) {
                const uint32_t v = kind ? c.l - c.f : c.f;
                if (!v) continue;
                const std::pair<int, uint32_t> cls(kind, v);
                if (std::find(classes.begin(), classes.end(), cls) == classes.end()) classes.push_back(cls);
            }
            if (classes.size() > 8) { ok = false; break; }
        }
        if (ok) {
            std::sort(classes.begin(), classes.end());
            const size_t nc = classes.size();
            auto class_of = [&](int kind, uint32_t v) { return (size_t)(std::find(classes.begin(), classes.end(), std::pair<int, uint32_t>(kind, v)) - classes.begin()); };
            std::vector<int> mult(nc, 0), first(nc, 0), n(nc);
            std::vector<Term> ts;
            auto terms_of = [&](int p) {                // terms of partition p in ascending slot order
                ts.clear();
                for (int i = m.cell_first[p]; i < m.cell_first[p + 1]; ++i) {
                    const HostModel::Cell &c = m.cells[i];
                    if (c.f) ts.push_back({0, c.f, m.slot_of_broker[c.b]});
                    if (c.l - c.f) ts.push_back({1, c.l - c.f, m.slot_of_broker[c.b]});
                }
                std::sort(ts.begin(), ts.end(), [](const Term &a, const Term &b) { return a.slot < b.slot; });
            };
            for (int p = 0; p < pb.P; ++p) {
                std::fill(n.begin(), n.end(), 0);
                for (int i = m.cell_first[p]; i < m.cell_first[p + 1]; ++i) {
                    const HostModel::Cell &c = m.cells[i];
                    if (c.f) { const size_t k = class_of(0, c.f); mult[k] = std::max(mult[k], ++n[k]); }
                    if (c.l - c.f) { const size_t k = class_of(1, c.l - c.f); mult[k] = std::max(mult[k], ++n[k]); }
                }
            }
            int J = 0;
            for (size_t c = 0; c < nc; ++c) { first[c] = J; J += mult[c]; }
            if (J <= 8) {
                m.z_ok = true;
                m.nz = J;
                m.zslot.assign((size_t)m.Ppad * 8, 0xFF);
                for (size_t c = 0; c < nc; ++c)
                    for (int k = 0; k < mult[c]; ++k) {
                        m.z_value[first[c] + k] = (int)classes[c].second;
                        if (classes[c].first) m.z_on_leader |= 1 << (first[c] + k);
                    }
                for (int p = 0; p < pb.P; ++p) {
                    terms_of(p);
                    std::fill(n.begin(), n.end(), 0);
                    for (const Term &t : ts) {
                        const size_t c = class_of(t.kind, t.val);
                        m.zslot[(size_t)p * 8 + first[c] + n[c]++] = (uint8_t)t.slot;
                    }
                }
            }
        }
    }
    m.hi1 = (pb.ppr_lo == 0 && pb.ppr_hi == 1);
    // home slots: the first four surviving entries of cur[p]
    m.homeT.assign((size_t)m.Ppad, 0xFFFFFFFFu);
    for (int p = 0; p < pb.P; ++p) {
        uint32_t h = 0xFFFFFFFFu;
        for (int i = 0; i < pb.RFcur && i < 4; ++i) {
            const int b = m.cur[(size_t)p * pb.RFcur + i];
            if (b >= 0) h = (h & ~(0xFFu << (8 * i))) | ((uint32_t)m.slot_of_broker[b] << (8 * i));
        }
        m.homeT[p] = h;
    }
    return true;
}

// word-major bit-plane helpers
struct Plane {
    const HostModel &m;
    std::vector<uint32_t> &bitsT;
    bool has(int p, int s) const { return (bitsT[(size_t)(s >> 5) * m.Ppad + p] >> (s & 31)) & 1u; }
    void set(int p, int s) { bitsT[(size_t)(s >> 5) * m.Ppad + p] |= 1u << (s & 31); }
};

// docs/MODEL.md §4: keep what survives of cur (order kept, leader = first survivor, tail dropped
// beyond RF), then complete short rows greedily: fewest replicas of p in the rack, then least
// loaded broker, then lowest dense index.  With per-partition rows (§11) row p is kept / completed to rf[p].
inline void initial_base(const HostModel &m, std::vector<uint32_t> &bitsT, std::vector<uint8_t> &leader)
{
    bitsT.assign((size_t)m.W * m.Ppad, 0);
    leader.assign((size_t)m.Ppad, 0xFF);
    Plane pl{m, bitsT};
    std::vector<int> load(m.B, 0), count(m.P, 0);
    for (int p = 0; p < m.P; ++p) {
        for (int i = 0; i < m.RFcur && count[p] < m.rf(p); ++i) {
            const int b = m.cur[(size_t)p * m.RFcur + i];
            if (b < 0 || pl.has(p, m.slot_of_broker[b])) continue;
            pl.set(p, m.slot_of_broker[b]);
            ++load[b];
            if (count[p]++ == 0) leader[p] = (uint8_t)m.slot_of_broker[b];
        }
    }
    std::vector<int> in_rack(m.R);
    for (int p = 0; p < m.P; ++p) {
        while (count[p] < m.rf(p)) {
            std::fill(in_rack.begin(), in_rack.end(), 0);
            for (int b = 0; b < m.B; ++b) if (pl.has(p, m.slot_of_broker[b])) ++in_rack[m.rack_of[b]];
            int best = -1;
            for (int b = 0; b < m.B; ++b) {
                if (pl.has(p, m.slot_of_broker[b])) continue;
                if (best < 0 ||
                    std::make_pair(in_rack[m.rack_of[b]], load[b]) < std::make_pair(in_rack[m.rack_of[best]], load[best]))
                    best = b;
            }
            pl.set(p, m.slot_of_broker[best]);
            ++load[best];
            ++count[p];
            if (leader[p] == 0xFF) leader[p] = (uint8_t)m.slot_of_broker[best];
        }
    }
}

// replica lists (dense indices, leader first, -1 padded; README.md:52-63) -> bit-plane
inline void encode_replicas(const HostModel &m, const int32_t *replicas, std::vector<uint32_t> &bitsT,
                            std::vector<uint8_t> &leader)
{
    bitsT.assign((size_t)m.W * m.Ppad, 0);
    leader.assign((size_t)m.Ppad, 0xFF);
    Plane pl{m, bitsT};
    for (int p = 0; p < m.P; ++p) {
        bool have = false;
        for (int i = 0; i < m.RF; ++i) {
            const int b = replicas[(size_t)p * m.RF + i];
            if (b < 0 || b >= m.B) continue;
            pl.set(p, m.slot_of_broker[b]);
            if (!have) { leader[p] = (uint8_t)m.slot_of_broker[b]; have = true; }
        }
    }
}

// bit-plane -> replica lists: leader first, followers by ascending dense index (README.md:65-78, :88)
inline void decode_replicas(const HostModel &m, std::vector<uint32_t> &bitsT, const std::vector<uint8_t> &leader,
                            int32_t *replicas)
{
    Plane pl{m, bitsT};
    for (int p = 0; p < m.P; ++p) {
        int32_t *out = replicas + (size_t)p * m.RF;
        std::fill(out, out + m.RF, -1);
        int n = 0, lb = -1;
        const int ld = leader[p];
        if (ld < m.W * 32 && pl.has(p, ld) && m.broker_of_slot[ld] >= 0) out[n++] = lb = m.broker_of_slot[ld];
        for (int b = 0; b < m.B && n < m.RF; ++b)
            if (b != lb && pl.has(p, m.slot_of_broker[b])) out[n++] = b;
    }
}

// replicas placed on a broker that did not hold the partition (data that must be copied)
inline int count_moves(const HostModel &m, const int32_t *replicas)
{
    int moves = 0;
    for (int p = 0; p < m.P; ++p)
        for (int i = 0; i < m.RF; ++i) {
            const int b = replicas[(size_t)p * m.RF + i];
            if (b < 0) continue;
            bool had = false;
            for (int k = 0; k < m.RFcur; ++k) had |= (m.cur[(size_t)p * m.RFcur + k] == b);
            moves += had ? 0 : 1;
        }
    return moves;
}

// An upper bound on the objective of every feasible assignment: per partition the best choice of a
// leader plus RF - 1 (rf[p] - 1) followers on distinct brokers, with the balance and rack constraints C3..C7
// dropped.  A search result that reaches it is proven optimal (kao_result.optimal); otherwise the
// optimum lp_solve would return (README.md:135-136) lies between the two.
inline int64_t objective_upper_bound(const HostModel &m, const kao_problem &)
{
    // per partition: the best leader plus the best RF - 1 followers among the other brokers, constraints C3..C7
    // ignored.  Only the non-zero cells matter: every other broker weighs 0 as a follower and as a leader.
    int64_t total = 0;
    std::vector<std::pair<uint32_t, int>> top;           // follower weights of the row, largest first
    for (int p = 0; p < m.P; ++p) {
        const int nf = m.rf(p) - 1;
        const int lo = m.cell_first[p], hi = m.cell_first[p + 1];
        top.clear();
        for (int i = lo; i < hi; ++i)
            if (m.cells[i].f) top.emplace_back(m.cells[i].f, m.cells[i].b);
        std::sort(top.begin(), top.end(), [](const auto &x, const auto &y) { return x.first > y.first; });
        int64_t sum_nf = 0, sum_rf = 0;                  // sums of the nf / nf + 1 largest follower weights
        for (int i = 0; i < (int)top.size() && i <= nf; ++i) { if (i < nf) sum_nf += top[i].first; sum_rf += top[i].first; }
        int64_t best = hi - lo < m.B ? sum_nf : 0;       // led from a broker that weighs nothing
        for (int i = lo; i < hi; ++i) {
            const HostModel::Cell &c = m.cells[i];
            bool in_top = false;
            for (int k = 0; k < nf && k < (int)top.size(); ++k) in_top |= top[k].second == c.b;
            const int64_t followers = in_top ? sum_rf - c.f : sum_nf;       // the leader's broker cannot follow too
            best = std::max(best, (int64_t)c.l + followers);
        }
        total += best;
    }
    return total;
}

// The per-topic rows of a kao_topics (docs/MODEL.md §10), checked against the problem (P, RF): 1 <= T <= P, topic_of
// in range, 0 <= lo <= hi, and lo no more than the topic can reach.  topic_of as u16 (T <= P <= 65,280), bounds as
// (C3t lo, C3t hi, C4t lo, C4t hi) per topic.
struct HostTopics {
    int T = 0;
    std::vector<uint16_t> topic_of;           // [Ppad]
    std::vector<int32_t> bnd;                 // [T][4]
};

// rf: the per-partition replication factors of a valid kao_replication (nullptr: RF for every partition)
inline bool build_host_topics(const kao_problem &pb, const kao_topics &tp, int Ppad, HostTopics &ht, std::string &why,
                              const int32_t *rf = nullptr)
{
    auto bad = [&](const std::string &s) { why = "topic rows: " + s; return false; };
    if (tp.T < 1 || tp.T > pb.P) return bad("T must be 1..P");
    if (!tp.topic_of || !tp.rep_lo || !tp.rep_hi || !tp.ldr_lo || !tp.ldr_hi) return bad("null table pointer");
    std::vector<int64_t> n(tp.T, 0), reps(tp.T, 0);
    ht.T = tp.T;
    ht.topic_of.assign((size_t)Ppad, 0);
    for (int p = 0; p < pb.P; ++p) {
        const int t = tp.topic_of[p];
        if (t < 0 || t >= tp.T) return bad("topic_of[" + std::to_string(p) + "] = " + std::to_string(t) + " is not in 0..T-1");
        ht.topic_of[p] = (uint16_t)t;
        ++n[t];
        reps[t] += rf ? rf[p] : pb.RF;
    }
    ht.bnd.assign((size_t)tp.T * 4, 0);
    for (int t = 0; t < tp.T; ++t) {
        const int32_t rl = tp.rep_lo[t], rh = tp.rep_hi[t], ll = tp.ldr_lo[t], lh = tp.ldr_hi[t];
        if (rl < 0 || rl > rh || ll < 0 || ll > lh)
            return bad("topic " + std::to_string(t) + ": bounds must satisfy 0 <= lo <= hi");
        if (rl > reps[t] || ll > n[t])
            return bad("topic " + std::to_string(t) + ": lo exceeds what its " + std::to_string(n[t]) +
                       (rf ? " partitions can reach (replicas: the sum of their replication factors, leaders: partitions)"
                           : " partitions can reach (replicas: partitions * RF, leaders: partitions)"));
        ht.bnd[4 * t] = rl; ht.bnd[4 * t + 1] = rh; ht.bnd[4 * t + 2] = ll; ht.bnd[4 * t + 3] = lh;
    }
    return true;
}

// The per-partition C1 / C7 rows of a kao_replication (docs/MODEL.md §11) into m (built by build_host_model):
// 1 <= rf[p] <= min(RF, B - 1), 0 <= ppr_lo[p] <= ppr_hi[p] <= 127.
inline bool build_host_replication(const kao_replication &rp, HostModel &m, std::string &why)
{
    auto bad = [&](const std::string &s) { why = "per-partition replication factors: " + s; return false; };
    if (!rp.rf || !rp.ppr_lo || !rp.ppr_hi) return bad("null table pointer");
    const int top = std::min(m.RF, m.B - 1);
    m.rf_p.assign((size_t)m.P, 0);
    m.ppr_lo_p.assign((size_t)m.P, 0);
    m.ppr_hi_p.assign((size_t)m.P, 0);
    for (int p = 0; p < m.P; ++p) {
        const int32_t f = rp.rf[p], lo = rp.ppr_lo[p], hi = rp.ppr_hi[p];
        if (f < 1 || f > top)
            return bad("rf[" + std::to_string(p) + "] = " + std::to_string(f) + " is not in 1.." + std::to_string(top) +
                       " (the row width RF, and fewer than the brokers)");
        if (lo < 0 || lo > hi || hi > 127)
            return bad("partition " + std::to_string(p) + ": per-rack bounds must satisfy 0 <= ppr_lo <= ppr_hi <= 127");
        m.rf_p[p] = (uint8_t)f; m.ppr_lo_p[p] = (uint8_t)lo; m.ppr_hi_p[p] = (uint8_t)hi;
    }
    return true;
}

// the table the HBM-base kernels read a row's C1 / C7 operands from: rf | ppr_lo << 8 | ppr_hi << 16 per partition
inline std::vector<uint32_t> replication_table(const HostModel &m)
{
    std::vector<uint32_t> t((size_t)m.Ppad, 0);
    for (int p = 0; p < m.P; ++p) t[p] = (uint32_t)m.rf(p) | ((uint32_t)m.plo(p) << 8) | ((uint32_t)m.phi(p) << 16);
    return t;
}

inline void fill_consts(const HostModel &m, Consts &cs)
{
    for (int s = 0; s < 256; ++s) {
        cs.bnd_rep[s] = m.bnd_rep[s];
        cs.bnd_ldr[s] = m.bnd_ldr[s];
        cs.slot_of_order[s] = (uint8_t)m.slot_of_order[s];
        cs.order_of_slot[s] = m.order_of_slot[s] < 0 ? 0xFF : (uint8_t)m.order_of_slot[s];
    }
    for (int r = 0; r < 32; ++r) {
        cs.rack_lo[r] = r < m.R ? m.rack_lo[r] : 0;
        cs.rack_hi[r] = r < m.R ? m.rack_hi[r] : 0;
    }
}

}  // namespace kao
