// kao-cli — compiled host side above the C ABI (include/kao.h): the reference's operator surface.
//
//   in : `kafka-reassign-partitions --generate` "Current partition replica assignment" JSON
//        (/root/reference/README.md:52-63), target broker list (README.md:48), broker -> rack map
//        (README.md:27-29; wire format `id:rack,...` is ours, the snapshot has none), RF
//   out: `--reassignment-json-file` JSON (README.md:67-78, :88), leader first
//        or, with --emit-lp, the lp_solve LP-format model text the reference generates
//        (README.md:139-185) so that anyone with lp_solve can solve the same instance.
//
// The reference's host language is Java; no JDK is available in this image, so the host side is
// C++ here and the Java/JNI sources under java/ ship uncompiled (INTEGRATION.md).
#include "../../include/kao.h"

#include <algorithm>
#include <cctype>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <map>
#include <set>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

namespace {

// ---------------------------------------------------------------- minimal JSON reader
struct Json {
    enum Kind { Null, Bool, Num, Str, Arr, Obj } kind = Null;
    double num = 0;
    bool b = false;
    std::string str;
    std::vector<Json> arr;
    std::vector<std::pair<std::string, Json>> obj;
    const Json &at(const std::string &k) const
    {
        for (auto &kv : obj) if (kv.first == k) return kv.second;
        throw std::runtime_error("missing JSON key: " + k);
    }
};
struct Parser {
    const std::string &s;
    size_t i = 0;
    explicit Parser(const std::string &t) : s(t) {}
    void ws() { while (i < s.size() && std::isspace((unsigned char)s[i])) ++i; }
    [[noreturn]] void fail(const char *m) { throw std::runtime_error(std::string("JSON: ") + m + " at offset " + std::to_string(i)); }
    Json value()
    {
        ws();
        if (i >= s.size()) fail("unexpected end");
        Json v;
        const char c = s[i];
        if (c == '{') {
            v.kind = Json::Obj; ++i; ws();
            if (s[i] == '}') { ++i; return v; }
            for (;;) {
                ws(); Json k = value();
                if (k.kind != Json::Str) fail("object key must be a string");
                ws(); if (s[i] != ':') fail("expected ':'"); ++i;
                v.obj.emplace_back(k.str, value());
                ws();
                if (s[i] == ',') { ++i; continue; }
                if (s[i] == '}') { ++i; return v; }
                fail("expected ',' or '}'");
            }
        }
        if (c == '[') {
            v.kind = Json::Arr; ++i; ws();
            if (s[i] == ']') { ++i; return v; }
            for (;;) {
                v.arr.push_back(value());
                ws();
                if (s[i] == ',') { ++i; continue; }
                if (s[i] == ']') { ++i; return v; }
                fail("expected ',' or ']'");
            }
        }
        if (c == '"') {
            v.kind = Json::Str; ++i;
            while (i < s.size() && s[i] != '"') {
                if (s[i] == '\\' && i + 1 < s.size()) { ++i; v.str += s[i] == 'n' ? '\n' : s[i] == 't' ? '\t' : s[i]; }
                else v.str += s[i];
                ++i;
            }
            if (i >= s.size()) fail("unterminated string");
            ++i;
            return v;
        }
        if (!s.compare(i, 4, "true")) { v.kind = Json::Bool; v.b = true; i += 4; return v; }
        if (!s.compare(i, 5, "false")) { v.kind = Json::Bool; i += 5; return v; }
        if (!s.compare(i, 4, "null")) { i += 4; return v; }
        char *end = nullptr;
        v.num = std::strtod(s.c_str() + i, &end);
        if (end == s.c_str() + i) fail("bad token");
        v.kind = Json::Num;
        i = (size_t)(end - s.c_str());
        return v;
    }
};

// ---------------------------------------------------------------- host-side model (docs/MODEL.md §1)
struct Row { std::string topic; int partition; std::vector<int> replicas; };

struct Model {
    int P = 0, B = 0, R = 0, RF = 0, RFcur = 0;
    std::vector<int> broker_ids;                // dense index -> Kafka broker id
    std::vector<std::string> rack_names;
    std::vector<uint8_t> rack_of;
    std::vector<uint16_t> wF, wL;
    std::vector<int32_t> rep_lo, rep_hi, ldr_lo, ldr_hi, rack_lo, rack_hi, cur;
    int ppr_lo = 0, ppr_hi = 0;
    std::vector<Row> rows;
    // per-topic rows (docs/MODEL.md §10, --topic-balance): topics in name order, floor / ceil of n_t * RF / B and n_t / B
    std::vector<std::string> topic_names;
    std::vector<int32_t> topic_of, trep_lo, trep_hi, tldr_lo, tldr_hi;
    // per-partition C1 / C7 rows (docs/MODEL.md §11, --keep-rf / --topic-rf): empty when every partition has RF
    std::vector<int32_t> prf, pprlo, pprhi;
};

static int ceil_div(long a, long b) { return (int)((a + b - 1) / b); }

Model build_model(std::vector<Row> rows, std::vector<int> brokers, const std::map<int, std::string> &racks, int rf)
{
    Model m;
    std::sort(rows.begin(), rows.end(), [](const Row &a, const Row &b) {
        return a.topic != b.topic ? a.topic < b.topic : a.partition < b.partition; });
    std::sort(brokers.begin(), brokers.end());
    brokers.erase(std::unique(brokers.begin(), brokers.end()), brokers.end());
    m.rows = rows; m.broker_ids = brokers;
    m.P = (int)rows.size(); m.B = (int)brokers.size(); m.RF = rf;
    std::map<int, int> dense;
    for (int i = 0; i < m.B; ++i) dense[brokers[i]] = i;
    std::set<std::string> names;
    for (int b : brokers) {
        auto it = racks.find(b);
        if (it == racks.end()) throw std::runtime_error("no rack given for broker " + std::to_string(b));
        names.insert(it->second);
    }
    m.rack_names.assign(names.begin(), names.end());
    m.R = (int)m.rack_names.size();
    std::vector<long> size(m.R, 0);
    for (int b : brokers) {
        const int r = (int)(std::find(m.rack_names.begin(), m.rack_names.end(), racks.at(b)) - m.rack_names.begin());
        m.rack_of.push_back((uint8_t)r);
        ++size[r];
    }
    for (auto &r : rows) m.RFcur = std::max(m.RFcur, (int)r.replicas.size());
    m.RFcur = std::max(m.RFcur, 1);
    m.cur.assign((size_t)m.P * m.RFcur, -1);
    m.wF.assign((size_t)m.P * m.B, 0);
    m.wL.assign((size_t)m.P * m.B, 0);
    static const int WL[3] = {4, 2, 1}, WF[3] = {2, 2, 1};   // README.md:146 coefficients {1,2,4}; :131-133
    for (int p = 0; p < m.P; ++p)
        for (size_t i = 0; i < rows[p].replicas.size(); ++i) {
            auto it = dense.find(rows[p].replicas[i]);
            if (it == dense.end()) continue;               // broker not in the target list (e.g. 19, README.md:48)
            m.cur[(size_t)p * m.RFcur + i] = it->second;
            m.wF[(size_t)p * m.B + it->second] = (uint16_t)(i < 3 ? WF[i] : 1);
            m.wL[(size_t)p * m.B + it->second] = (uint16_t)(i < 3 ? WL[i] : 1);
        }
    const long tot = (long)m.P * rf;
    m.rep_lo.assign(m.B, (int)(tot / m.B)); m.rep_hi.assign(m.B, ceil_div(tot, m.B));        // README.md:158-161
    m.ldr_lo.assign(m.B, m.P / m.B);        m.ldr_hi.assign(m.B, ceil_div(m.P, m.B));         // README.md:163-166
    for (int r = 0; r < m.R; ++r) {                                                           // README.md:173-176
        m.rack_lo.push_back((int)(tot * size[r] / m.B));
        m.rack_hi.push_back(ceil_div(tot * size[r], m.B));
    }
    m.ppr_lo = rf / m.R; m.ppr_hi = ceil_div(rf, m.R);                                        // README.md:178-180
    std::vector<long> n;
    for (const Row &r : m.rows) {                               // rows are sorted by topic: a new name starts a topic
        if (m.topic_names.empty() || m.topic_names.back() != r.topic) { m.topic_names.push_back(r.topic); n.push_back(0); }
        m.topic_of.push_back((int32_t)m.topic_names.size() - 1);
        ++n.back();
    }
    for (long nt : n) {
        m.trep_lo.push_back((int)(nt * rf / m.B)); m.trep_hi.push_back(ceil_div(nt * rf, m.B));
        m.tldr_lo.push_back((int)(nt / m.B));      m.tldr_hi.push_back(ceil_div(nt, m.B));
    }
    return m;
}

// --keep-rf / --topic-rf (docs/MODEL.md §11): every topic keeps the length of its longest replica list (keep_rf, or no
// --rf given), else takes rf; the topics named in topic_rf take theirs.  When the partitions then differ, RF becomes the
// largest factor (the width of the replica lists), C3 / C6 and the topic rows follow the sum of the factors and every
// partition gets its own C1 = rf[p] and C7 = floor / ceil of rf[p] / R; when they agree the model is the plain one.
Model build_model_rf(const std::vector<Row> &rows, const std::vector<int> &brokers,
                     const std::map<int, std::string> &racks, bool keep_rf, int rf,
                     const std::map<std::string, int> &topic_rf)
{
    Model m = build_model(rows, brokers, racks, 1);                 // the sorted rows and their topics
    std::vector<int> longest(m.topic_names.size(), 1);
    for (int p = 0; p < m.P; ++p) longest[m.topic_of[p]] = std::max(longest[m.topic_of[p]], (int)m.rows[p].replicas.size());
    for (const auto &kv : topic_rf)
        if (std::find(m.topic_names.begin(), m.topic_names.end(), kv.first) == m.topic_names.end())
            throw std::runtime_error("--topic-rf: no topic named " + kv.first + " in the assignment");
    std::vector<int32_t> prf(m.P);
    for (int p = 0; p < m.P; ++p) {
        const std::string &name = m.topic_names[m.topic_of[p]];
        const auto it = topic_rf.find(name);
        prf[p] = it != topic_rf.end() ? it->second : (keep_rf || rf <= 0) ? longest[m.topic_of[p]] : rf;
    }
    const int top = *std::max_element(prf.begin(), prf.end());
    m = build_model(rows, brokers, racks, top);
    if (std::all_of(prf.begin(), prf.end(), [&](int32_t f) { return f == top; })) return m;
    long tot = 0;
    std::vector<long> reps(m.topic_names.size(), 0);
    for (int p = 0; p < m.P; ++p) { tot += prf[p]; reps[m.topic_of[p]] += prf[p]; }
    std::vector<long> size(m.R, 0);
    for (int b = 0; b < m.B; ++b) ++size[m.rack_of[b]];
    m.rep_lo.assign(m.B, (int)(tot / m.B)); m.rep_hi.assign(m.B, ceil_div(tot, m.B));
    for (int r = 0; r < m.R; ++r) { m.rack_lo[r] = (int)(tot * size[r] / m.B); m.rack_hi[r] = ceil_div(tot * size[r], m.B); }
    for (size_t t = 0; t < reps.size(); ++t) { m.trep_lo[t] = (int)(reps[t] / m.B); m.trep_hi[t] = ceil_div(reps[t], m.B); }
    m.prf = prf;
    for (int32_t f : prf) { m.pprlo.push_back(f / m.R); m.pprhi.push_back(ceil_div(f, m.R)); }
    return m;
}

// lp_solve LP-format text, same families and naming as README.md:144-185
void emit_lp(const Model &m, std::ostream &o, bool topics)
{
    auto var = [&](int b, int p, bool l) {
        return "t1b" + std::to_string(m.broker_ids[b]) + "p" + std::to_string(p) + (l ? "_l" : "");
    };
    o << "// Optimization function, based on current assignment\nmax: ";
    bool first = true;
    for (int p = 0; p < m.P; ++p)
        for (int b = 0; b < m.B; ++b) {
            const int f = m.wF[(size_t)p * m.B + b], l = m.wL[(size_t)p * m.B + b];
            if (f) { o << (first ? "" : " + ") << f << " " << var(b, p, false); first = false; }
            if (l) { o << (first ? "" : " + ") << l << " " << var(b, p, true); first = false; }
        }
    o << ";\n\n// Constrain on replication factor for every partition\n";
    for (int p = 0; p < m.P; ++p) {
        for (int b = 0; b < m.B; ++b) o << (b ? " + " : "") << var(b, p, false) << " + " << var(b, p, true);
        o << " = " << (m.prf.empty() ? m.RF : m.prf[p]) << ";\n";
    }
    o << "\n// Constraint on having one and only one leader per partition\n";
    for (int p = 0; p < m.P; ++p) {
        for (int b = 0; b < m.B; ++b) o << (b ? " + " : "") << var(b, p, true);
        o << " = 1;\n";
    }
    o << "\n// Constraint on min/max replicas per broker\n";
    for (int b = 0; b < m.B; ++b)
        for (int pass = 0; pass < 2; ++pass) {
            for (int p = 0; p < m.P; ++p) o << (p ? " + " : "") << var(b, p, false) << " + " << var(b, p, true);
            o << (pass ? " >= " : " <= ") << (pass ? m.rep_lo[b] : m.rep_hi[b]) << ";\n";
        }
    o << "\n// Constraint on min/max leaders per broker\n";
    for (int b = 0; b < m.B; ++b)
        for (int pass = 0; pass < 2; ++pass) {
            for (int p = 0; p < m.P; ++p) o << (p ? " + " : "") << var(b, p, true);
            o << (pass ? " >= " : " <= ") << (pass ? m.ldr_lo[b] : m.ldr_hi[b]) << ";\n";
        }
    o << "\n// Constraint on no leader and replicas on the same broker\n";
    for (int b = 0; b < m.B; ++b)
        for (int p = 0; p < m.P; ++p) o << var(b, p, false) << " + " << var(b, p, true) << " <= 1;\n";
    for (int r = 0; r < m.R; ++r) {
        o << "\n// Constrain on min/max total replicas per racks. " << m.rack_names[r] << " here\n";
        for (int pass = 0; pass < 2; ++pass) {
            bool f2 = true;
            for (int b = 0; b < m.B; ++b) {
                if (m.rack_of[b] != r) continue;
                for (int p = 0; p < m.P; ++p) { o << (f2 ? "" : " + ") << var(b, p, false) << " + " << var(b, p, true); f2 = false; }
            }
            o << (pass ? " >= " : " <= ") << (pass ? m.rack_lo[r] : m.rack_hi[r]) << ";\n";
        }
    }
    o << "\n// Constrain on min/max replicas per partitions per racks.\n";
    for (int p = 0; p < m.P; ++p) {
        const int plo = m.prf.empty() ? m.ppr_lo : m.pprlo[p], phi = m.prf.empty() ? m.ppr_hi : m.pprhi[p];
        for (int r = 0; r < m.R; ++r)
            for (int pass = 0; pass < (plo > 0 ? 2 : 1); ++pass) {
                bool f2 = true;
                for (int b = 0; b < m.B; ++b) {
                    if (m.rack_of[b] != r) continue;
                    o << (f2 ? "" : " + ") << var(b, p, false) << " + " << var(b, p, true); f2 = false;
                }
                o << (pass ? " >= " : " <= ") << (pass ? plo : phi) << ";\n";
            }
    }
    for (int t = 0; topics && t < (int)m.topic_names.size(); ++t)
        for (int kind = 0; kind < 2; ++kind) {
            o << "\n// Constraint on min/max " << (kind ? "leaders" : "replicas") << " of topic " << m.topic_names[t]
              << " per broker\n";
            for (int b = 0; b < m.B; ++b)
                for (int pass = 0; pass < 2; ++pass) {
                    bool f2 = true;
                    for (int p = 0; p < m.P; ++p) {
                        if (m.topic_of[p] != t) continue;
                        if (!kind) o << (f2 ? "" : " + ") << var(b, p, false) << " + " << var(b, p, true);
                        else o << (f2 ? "" : " + ") << var(b, p, true);
                        f2 = false;
                    }
                    const int lo = kind ? m.tldr_lo[t] : m.trep_lo[t], hi = kind ? m.tldr_hi[t] : m.trep_hi[t];
                    o << (pass ? " >= " : " <= ") << (pass ? lo : hi) << ";\n";
                }
        }
    o << "\n// All variables are binary\nbin\n";
    for (int p = 0; p < m.P; ++p)
        for (int b = 0; b < m.B; ++b)
            o << (p || b ? ", " : "") << var(b, p, false) << ", " << var(b, p, true);
    o << ";\n";
}

std::string slurp(const std::string &path)
{
    if (path == "-") { std::stringstream ss; ss << std::cin.rdbuf(); return ss.str(); }
    std::ifstream f(path);
    if (!f) throw std::runtime_error("cannot open " + path);
    std::stringstream ss; ss << f.rdbuf();
    return ss.str();
}

std::vector<std::string> split(const std::string &s, char sep)
{
    std::vector<std::string> out; std::string cur;
    for (char c : s) { if (c == sep) { out.push_back(cur); cur.clear(); } else if (!std::isspace((unsigned char)c)) cur += c; }
    out.push_back(cur);
    out.erase(std::remove(out.begin(), out.end(), std::string()), out.end());
    return out;
}

int usage()
{
    std::fprintf(stderr,
                 "usage: kao-cli --assignment FILE|- --brokers 0,1,2 --racks 0:a,1:b,2:a [--rf N]\n"
                 "               [--rounds 256] [--round-size 32768] [--restarts 1] [--seed 24301] [--device 0] [--delta] [--row-major] [--gpus N] [--spread-restarts] [--patience N] [--certificate] [--lp-certificate] [--topic-balance] [--emit-lp] [--stats]\n"
                 "               [--keep-rf] [--topic-rf name:N,...]\n");
    return 2;
}

}  // namespace

int main(int argc, char **argv)
{
    std::map<std::string, std::string> a;
    bool emit = false, stats = false, delta = false, rowmajor = false, spread = false, certificate = false, lp_certificate = false,
         topic_balance = false, keep_rf = false;
    for (int i = 1; i < argc; ++i) {
        std::string k = argv[i];
        if (k == "--emit-lp") { emit = true; continue; }
        if (k == "--stats") { stats = true; continue; }
        if (k == "--delta") { delta = true; continue; }
        if (k == "--row-major") { rowmajor = true; continue; }
        if (k == "--spread-restarts") { spread = true; continue; }   // --gpus N: the restarts side by side, one per GPU at a time
        if (k == "--certificate") { certificate = true; continue; }  // flow bound: --stats can then say "proven optimal"
        if (k == "--lp-certificate") { lp_certificate = true; continue; }  // Lagrangian LP bound (GPU): proves what the flow bound cannot
        if (k == "--topic-balance") { topic_balance = true; continue; }   // every topic spread over the brokers too
        if (k == "--keep-rf") { keep_rf = true; continue; }   // every topic keeps its own RF (docs/MODEL.md §11)
        if (k == "--column-major") continue;                  // accepted for old scripts: it is the default now
        if (k.rfind("--", 0) != 0 || i + 1 >= argc) return usage();
        a[k.substr(2)] = argv[++i];
    }
    if (!a.count("assignment") || !a.count("brokers") || !a.count("racks")) return usage();
    try {
        const std::string text = slurp(a["assignment"]);
        Parser ps(text);
        const Json doc = ps.value();
        std::vector<Row> rows;
        for (const Json &e : doc.at("partitions").arr) {
            Row r;
            r.topic = e.at("topic").str;
            r.partition = (int)e.at("partition").num;
            for (const Json &b : e.at("replicas").arr) r.replicas.push_back((int)b.num);
            rows.push_back(r);
        }
        if (rows.empty()) throw std::runtime_error("no partitions in the assignment");
        std::vector<int> brokers;
        for (auto &t : split(a["brokers"], ',')) brokers.push_back(std::atoi(t.c_str()));
        std::map<int, std::string> racks;
        for (auto &t : split(a["racks"], ',')) {
            const size_t c = t.find(':');
            if (c == std::string::npos) throw std::runtime_error("rack map entries look like id:rack");
            racks[std::atoi(t.substr(0, c).c_str())] = t.substr(c + 1);
        }
        int rf = 0;
        for (auto &r : rows) rf = std::max(rf, (int)r.replicas.size());
        if (a.count("rf")) rf = std::atoi(a["rf"].c_str());
        std::map<std::string, int> topic_rf;                  // --topic-rf name:N,...
        for (auto &t : split(a.count("topic-rf") ? a["topic-rf"] : "", ',')) {
            const size_t c = t.rfind(':');
            if (c == std::string::npos || c == 0) throw std::runtime_error("--topic-rf entries look like topic:N");
            topic_rf[t.substr(0, c)] = std::atoi(t.substr(c + 1).c_str());
        }
        Model m = keep_rf || !topic_rf.empty()
                      ? build_model_rf(rows, brokers, racks, keep_rf, a.count("rf") ? rf : 0, topic_rf)
                      : build_model(rows, brokers, racks, rf);
        if (emit) { emit_lp(m, std::cout, topic_balance); return 0; }

        kao_problem pb{};
        pb.P = m.P; pb.B = m.B; pb.R = m.R; pb.RF = m.RF; pb.RFcur = m.RFcur;
        pb.rack_of = m.rack_of.data(); pb.wF = m.wF.data(); pb.wL = m.wL.data();
        pb.rep_lo = m.rep_lo.data(); pb.rep_hi = m.rep_hi.data(); pb.ldr_lo = m.ldr_lo.data(); pb.ldr_hi = m.ldr_hi.data();
        pb.rack_lo = m.rack_lo.data(); pb.rack_hi = m.rack_hi.data(); pb.ppr_lo = m.ppr_lo; pb.ppr_hi = m.ppr_hi;
        pb.cur = m.cur.data();
        kao_options opt{};
        opt.seed = a.count("seed") ? std::strtoull(a["seed"].c_str(), nullptr, 0) : 0x5EED;
        opt.rounds = a.count("rounds") ? (uint32_t)std::atoi(a["rounds"].c_str()) : 256;
        opt.round_size = a.count("round-size") ? (uint32_t)std::atoi(a["round-size"].c_str()) : 32768;
        opt.device = a.count("device") ? std::atoi(a["device"].c_str()) : 0;
        opt.n_gpus = a.count("gpus") ? std::atoi(a["gpus"].c_str()) : 1;     // rounds sharded over N GPUs, same result
        opt.flags = a.count("restarts") ? (uint32_t)std::min(255, std::max(1, std::atoi(a["restarts"].c_str()))) : 1u;
        if (delta) opt.flags |= KAO_FLAG_DELTA;
        if (rowmajor) opt.flags |= KAO_FLAG_ROW_MAJOR;        // measurements: the other full evaluator, same result
        if (spread) opt.flags |= KAO_FLAG_SPREAD_RESTARTS;
        if (certificate) opt.flags |= KAO_FLAG_BOUND;
        if (lp_certificate) opt.flags |= KAO_FLAG_LP_BOUND;
        if (a.count("patience")) opt.flags |= KAO_FLAG_PATIENCE(std::min(65535, std::max(0, std::atoi(a["patience"].c_str()))));
        std::vector<int32_t> reps((size_t)m.P * m.RF, -1);
        kao_result res{};
        res.replicas = reps.data();
        kao_topics tp{(int32_t)m.topic_names.size(), m.topic_of.data(), m.trep_lo.data(), m.trep_hi.data(),
                      m.tldr_lo.data(), m.tldr_hi.data()};
        kao_replication rp{m.prf.data(), m.pprlo.data(), m.pprhi.data()};
        const int rc = !m.prf.empty() ? kao_solve_replication(&pb, topic_balance ? &tp : nullptr, &rp, &opt, &res)
                       : topic_balance ? kao_solve_topics(&pb, &tp, &opt, &res) : kao_solve(&pb, &opt, &res);
        if (rc < 0) { std::fprintf(stderr, "kao-cli: %s\n", kao_last_error()); return 1; }
        if (rc == KAO_INFEASIBLE)
            std::fprintf(stderr, "kao-cli: warning: no assignment satisfying every constraint was found (violation %lld)\n",
                         (long long)res.violation);
        std::cout << "{\"version\":1,\"partitions\":[\n";
        for (int p = 0; p < m.P; ++p) {
            std::cout << "    {\"topic\":\"" << m.rows[p].topic << "\",\"partition\":" << m.rows[p].partition << ",\"replicas\":[";
            bool first = true;
            for (int i = 0; i < m.RF; ++i) {
                const int b = reps[(size_t)p * m.RF + i];
                if (b < 0) continue;
                std::cout << (first ? "" : ",") << m.broker_ids[b];
                first = false;
            }
            std::cout << "]}" << (p + 1 < m.P ? "," : "") << "\n";
        }
        std::cout << "]}\n";
        if (stats)
            std::fprintf(stderr, "kao-cli: objective %lld (upper bound %lld%s), violation %lld, replica moves %d, %llu candidates, "
                                 "%d GPU(s), %.2f ms on device, %.2f ms total\n",
                         (long long)res.objective, (long long)res.objective_bound, res.optimal ? ": proven optimal" : "",
                         (long long)res.violation, res.moves, (unsigned long long)res.n_candidates, res.n_gpus, res.device_ms,
                         res.total_ms);
        return rc == KAO_INFEASIBLE ? 3 : 0;
    } catch (const std::exception &e) {
        std::fprintf(stderr, "kao-cli: %s\n", e.what());
        return 1;
    }
}
