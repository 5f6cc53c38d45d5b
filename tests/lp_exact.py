"""TEST INFRASTRUCTURE — L(u) of the Lagrangian LP bound (docs/MODEL.md §9), evaluated exactly from its definition:
the φ terms of the dualised rows C3, C4, C6 plus, for every partition, the best row that satisfies C1, C2, C5 and C7
under the reduced weights.  It shares nothing with the rack DP of the kernel and of its restatement (tests/lp_ref):
the best row is a maximum over every choice of leader broker, and for each leader over every split of the RF replicas
into per-rack counts, where a rack of k replicas holds its k best followers (sorting), or the leader plus the k - 1
best of the rack's other brokers.  The racks without the leader are combined by prefix / suffix max-plus products.

Every value of a partition stays in int64 (a reduced weight is below 2^38 at the build limits of MODEL §9, a row of
at most 8 of them below 2^41); the sums over partitions and rows are Python ints."""
import numpy as np

F = 20                      # fractional bits of the multipliers (KAO_LP_FRACTION_BITS)
U = 1 << 34                 # |u| <= U
_NONE = np.int64(-(1 << 62))     # "no admissible choice": below every value, and twice it still fits in int64


def _maxplus(a, b, RF):
    """(P, RF + 1) tables of the best value with n replicas -> the best value with n replicas over both parts"""
    out = np.full_like(a, _NONE)
    for i in range(RF + 1):
        for j in range(RF + 1 - i):
            ok = (a[:, i] > _NONE) & (b[:, j] > _NONE)
            out[:, i + j] = np.maximum(out[:, i + j], np.where(ok, a[:, i] + b[:, j], _NONE))
    return out


def lagrangian_fixed(pb, u):
    """2^F · L(u) as a Python int; u = int64[2B + R] (C3 per broker, C4 per broker, C6 per rack) with F fractional
    bits.  Raises ValueError when a partition has no row that satisfies C1, C2, C5 and C7."""
    P, B, R, RF = pb.P, pb.B, pb.R, pb.RF
    u = np.asarray(u, np.int64)
    assert u.shape == (2 * B + R,) and int(np.abs(u).max(initial=0)) <= U
    u3, u4, u6 = u[:B], u[B:2 * B], u[2 * B:]
    rack = pb.rack_of.astype(np.int64)
    # φ: the row bounds, an upper bound above what an assignment reaches lowered to it
    tot = P * RF
    lo = [int(x) for x in pb.rep_lo] + [int(x) for x in pb.ldr_lo] + [int(x) for x in pb.rack_lo]
    hi = [min(int(x), tot) for x in pb.rep_hi] + [min(int(x), P) for x in pb.ldr_hi] + [min(int(x), tot) for x in pb.rack_hi]
    phi = sum(int(x) * (h if x > 0 else l) for x, l, h in zip(u, lo, hi))
    # reduced weights [P, B]
    f = (pb.wF.astype(np.int64) << F) - (u3 + u6[rack])[None, :]
    ld = (pb.wL.astype(np.int64) << F) - (u3 + u4 + u6[rack])[None, :]
    members = [np.flatnonzero(rack == r) for r in range(R)]
    plo, phi_hi = int(pb.ppr_lo), int(pb.ppr_hi)
    top = [min(len(mb), phi_hi) for mb in members]          # admissible counts of rack r: plo .. top[r]

    # per rack: prefix sums of the followers sorted by descending reduced weight, each broker's place in that order
    csum, place = [], []
    for mb in members:
        srt = -np.sort(-f[:, mb], axis=1)
        c = np.zeros((P, len(mb) + 1), np.int64)
        c[:, 1:] = np.cumsum(srt, axis=1)
        csum.append(c)
        # place of broker j among the rack's followers (ties in any order: a tie changes no sum below)
        order = np.argsort(-f[:, mb], axis=1, kind="stable")
        pl = np.empty_like(order)
        np.put_along_axis(pl, order, np.broadcast_to(np.arange(len(mb)), order.shape), axis=1)
        place.append(pl)

    # followers only: table [P, RF + 1] of rack r
    def followers(r):
        t = np.full((P, RF + 1), _NONE, np.int64)
        for k in range(plo, min(top[r], RF) + 1):
            t[:, k] = csum[r][:, k]
        return t

    tabs = [followers(r) for r in range(R)]
    unit = np.full((P, RF + 1), _NONE, np.int64)
    unit[:, 0] = 0
    pre = [unit]
    for r in range(R):
        pre.append(_maxplus(pre[-1], tabs[r], RF))
    suf = [unit]
    for r in reversed(range(R)):
        suf.append(_maxplus(suf[-1], tabs[r], RF))
    suf = suf[::-1]                                         # suf[r]: racks r .. R-1

    best = np.full(P, _NONE, np.int64)
    for r, mb in enumerate(members):
        rest = _maxplus(pre[r], suf[r + 1], RF)             # every rack but r, followers only
        for k in range(max(plo, 1), min(top[r], RF) + 1):
            others = rest[:, RF - k]
            ok = others > _NONE
            if not ok.any():
                continue
            # leader j of rack r with the k - 1 best other brokers of the rack as followers: the first k - 1 of
            # the sorted list, or the first k without j when j is among them
            fol = np.where(place[r] < k - 1, csum[r][:, k, None] - f[:, mb], csum[r][:, k - 1, None])
            v = (ld[:, mb] + fol).max(axis=1) + others
            best = np.maximum(best, np.where(ok, v, _NONE))
    if (best == _NONE).any():
        raise ValueError("a partition has no row that satisfies C1, C2, C5 and C7")
    return phi + sum(int(x) for x in best)
