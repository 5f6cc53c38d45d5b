// reduce_fixed.cpp — TEST INFRASTRUCTURE, part of kao_emu.cpp's translation unit.  The host reduction of
// kao_solve_fixed (reduce_fixed / expand_fixed in csrc/kao_host.hpp, docs/MODEL.md §12) behind a C interface, so that
// the CPU suite can score the reduced problem with the emulated sessions and compare it with the restricted program of
// tests/fixed_ref.py.
namespace {
template <class T> void put(const std::vector<T> &v, T *dst) { if (dst && !v.empty()) std::memcpy(dst, v.data(), v.size() * sizeof(T)); }
}  // namespace

extern "C" {

// nullptr when reduce_fixed refuses the input (kao_emu_last_error says why)
void *kao_fx_reduce(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp, const uint8_t *fixed)
{
    auto *fr = new FixedReduction;
    if (!reduce_fixed(*pb, tp, rp, fixed, *fr, g_err)) { delete fr; return nullptr; }
    return fr;
}
void kao_fx_free(void *h) { delete static_cast<FixedReduction *>(h); }

// sizes = {P', T'}, consts = {V0, O0}
void kao_fx_sizes(void *h, int32_t *sizes, int64_t *consts)
{
    const FixedReduction &fr = *static_cast<FixedReduction *>(h);
    sizes[0] = fr.pb.P; sizes[1] = (int32_t)fr.trep_lo.size();
    consts[0] = fr.V0; consts[1] = fr.O0;
}
void kao_fx_rows(void *h, int32_t *searched, uint16_t *wF, uint16_t *wL, int32_t *cur)
{
    const FixedReduction &fr = *static_cast<FixedReduction *>(h);
    put(fr.searched, searched); put(fr.wF, wF); put(fr.wL, wL); put(fr.cur, cur);
}
void kao_fx_bounds(void *h, int32_t *rep_lo, int32_t *rep_hi, int32_t *ldr_lo, int32_t *ldr_hi, int32_t *rack_lo, int32_t *rack_hi)
{
    const FixedReduction &fr = *static_cast<FixedReduction *>(h);
    put(fr.rep_lo, rep_lo); put(fr.rep_hi, rep_hi); put(fr.ldr_lo, ldr_lo); put(fr.ldr_hi, ldr_hi);
    put(fr.rack_lo, rack_lo); put(fr.rack_hi, rack_hi);
}
void kao_fx_replication(void *h, int32_t *rf, int32_t *ppr_lo, int32_t *ppr_hi)
{
    const FixedReduction &fr = *static_cast<FixedReduction *>(h);
    put(fr.rf, rf); put(fr.ppr_lo, ppr_lo); put(fr.ppr_hi, ppr_hi);
}
void kao_fx_topics(void *h, int32_t *topic_of, int32_t *rep_lo, int32_t *rep_hi, int32_t *ldr_lo, int32_t *ldr_hi)
{
    const FixedReduction &fr = *static_cast<FixedReduction *>(h);
    put(fr.topic_of, topic_of); put(fr.trep_lo, rep_lo); put(fr.trep_hi, rep_hi); put(fr.tldr_lo, ldr_lo); put(fr.tldr_hi, ldr_hi);
}
// [P'*RF] -> [P*RF] (pb: the problem the reduction was made from)
void kao_fx_expand(void *h, const kao_problem *pb, const int32_t *reduced, int32_t *replicas)
{
    expand_fixed(*pb, *static_cast<FixedReduction *>(h), reduced, replicas);
}

}  // extern "C"
