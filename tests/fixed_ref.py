"""TEST INFRASTRUCTURE — fixed partitions (docs/MODEL.md §12) restated in Python, independent of the engine.

* :func:`evaluate` and :func:`solve_exact` state the restricted program directly: a fixed row keeps its current
  replicas, its own rows (C1, C2/C5, C7, per-partition replication rows) are not part of the program, and its replicas
  and leader still count in C3, C4, C6 and the topic rows.  No reduction is involved.
* :func:`reduce` restates the host reduction of ``kao_solve_fixed`` (``reduce_fixed`` in csrc/kao_host.hpp): the
  problem over the searched rows with the fixed load moved into the bounds, and the constants V0 / O0.  The GPU tests
  build the reduced problem with it, so they need neither the engine's reduction nor the reference.
"""
import dataclasses

import numpy as np

from oracle import model


def fixed_row(pb, p):
    """The replicas a fixed row keeps: the non-negative entries of cur[p], in order, the first one leading."""
    return [int(b) for b in pb.cur[p] if b >= 0]


def _band(c, lo, hi):
    return int(np.maximum(np.asarray(lo) - c, 0).sum() + np.maximum(c - np.asarray(hi), 0).sum())


def fixed_load(pb, fixed, tr=None):
    """(replicas per broker, leaders per broker, replicas per rack, objective, [T, B] topic replicas, [T, B] topic
    leaders) of the fixed rows."""
    f, fl, fr = np.zeros(pb.B, np.int64), np.zeros(pb.B, np.int64), np.zeros(pb.R, np.int64)
    T = 0 if tr is None else len(tr.rep_lo)
    ft, flt = np.zeros((T, pb.B), np.int64), np.zeros((T, pb.B), np.int64)
    o0 = 0
    for p in np.flatnonzero(fixed):
        row = fixed_row(pb, p)
        for i, b in enumerate(row):
            f[b] += 1
            fr[pb.rack_of[b]] += 1
            o0 += int(pb.wL[p, b] if i == 0 else pb.wF[p, b])
            if tr is not None:
                ft[tr.topic_of[p], b] += 1
        fl[row[0]] += 1
        if tr is not None:
            flt[tr.topic_of[p], row[0]] += 1
    return f, fl, fr, o0, ft, flt


def evaluate(pb, fixed, replicas, tr=None, rr=None):
    """(violation, objective) of `replicas` ([P, RF], leader first) in the restricted program: the rows of every
    partition count in C3 / C4 / C6 / topic rows and in the objective, only the searched ones in C1, C2/C5 and C7."""
    P, B, R = pb.P, pb.B, pb.R
    cnt, lcnt = np.zeros(B, np.int64), np.zeros(B, np.int64)
    T = 0 if tr is None else len(tr.rep_lo)
    tcnt, tlcnt = np.zeros((T, B), np.int64), np.zeros((T, B), np.int64)
    viol = obj = 0
    for p in range(P):
        row = [int(b) for b in replicas[p] if b >= 0]
        uniq = set(row)
        ld = row[0] if row else -1
        if ld >= 0:
            lcnt[ld] += 1
            obj += int(pb.wL[p, ld])
            if tr is not None:
                tlcnt[tr.topic_of[p], ld] += 1
        pr = np.zeros(R, np.int64)
        for b in uniq:
            cnt[b] += 1
            pr[pb.rack_of[b]] += 1
            if tr is not None:
                tcnt[tr.topic_of[p], b] += 1
            if b != ld:
                obj += int(pb.wF[p, b])
        if fixed[p]:
            continue
        n, lo, hi = (pb.RF, pb.ppr_lo, pb.ppr_hi) if rr is None else (int(rr.rf[p]), int(rr.ppr_lo[p]), int(rr.ppr_hi[p]))
        viol += abs(len(uniq) - n) + (ld < 0)
        viol += _band(pr, lo, hi)
    viol += _band(cnt, pb.rep_lo, pb.rep_hi) + _band(lcnt, pb.ldr_lo, pb.ldr_hi)
    viol += _band(np.bincount(pb.rack_of, weights=cnt, minlength=R).astype(np.int64), pb.rack_lo, pb.rack_hi)
    if tr is not None:
        viol += _band(tcnt, np.asarray(tr.rep_lo)[:, None], np.asarray(tr.rep_hi)[:, None])
        viol += _band(tlcnt, np.asarray(tr.ldr_lo)[:, None], np.asarray(tr.ldr_hi)[:, None])
    return viol, obj


def solve_exact(pb, fixed, tr=None, rr=None, time_limit=None):
    """HiGHS optimum of the restricted program: the variables of fixed rows fixed to cur, their C1 / C2 / C5 / C7 rows
    dropped (with `rr` the searched rows' C1 / C7 are rf[p] / ppr_lo[p]..ppr_hi[p]).  The objective includes O0."""
    import scipy.sparse as sp
    from scipy.optimize import Bounds, LinearConstraint, milp

    P, B, R = pb.P, pb.B, pb.R
    A, lo, hi = model._constraints(pb)
    if rr is not None:
        lo[:P] = hi[:P] = np.asarray(rr.rf, np.float64)
        lo[-P * R:] = np.repeat(np.asarray(rr.ppr_lo, np.float64), R)
        hi[-P * R:] = np.repeat(np.asarray(rr.ppr_hi, np.float64), R)
    fx = np.asarray(fixed, bool)
    # rows of model._constraints: C1 [P], C2 [P], C3 [B], C4 [B], C5 [P*B], C6 [R], C7 [P*R]
    keep = np.concatenate([~fx, ~fx, np.ones(2 * B, bool), np.repeat(~fx, B), np.ones(R, bool), np.repeat(~fx, R)])
    A, lo, hi = A[np.flatnonzero(keep)], lo[keep], hi[keep]
    if tr is not None:
        from topics_ref import topic_program_rows

        At, lt, ht = topic_program_rows(pb, tr)
        A, lo, hi = sp.vstack([A, At], format="csr"), np.concatenate([lo, lt]), np.concatenate([hi, ht])
    vlo, vhi = np.zeros(2 * P * B), np.ones(2 * P * B)
    for p in np.flatnonzero(fx):
        vhi[p * B:(p + 1) * B] = vhi[P * B + p * B:P * B + (p + 1) * B] = 0
        row = fixed_row(pb, p)
        vlo[P * B + p * B + row[0]] = vhi[P * B + p * B + row[0]] = 1
        for b in row[1:]:
            vlo[p * B + b] = vhi[p * B + b] = 1
    c = -np.concatenate([pb.wF.reshape(-1), pb.wL.reshape(-1)]).astype(np.float64)
    opts = {"mip_rel_gap": 0.0}
    if time_limit:
        opts["time_limit"] = time_limit
    res = milp(c, constraints=LinearConstraint(A, lo, hi), integrality=np.ones(c.size), bounds=Bounds(vlo, vhi),
               options=opts)
    if res.status == 0 and res.x is not None:
        reps = model.decode(pb, res.x)
        return model.Solution("optimal", int(round(-res.fun)), reps, None, 0.0, 0.0)
    return model.Solution({2: "infeasible", 1: "limit"}.get(res.status, "other"), None, None, None, 0.0, 0.0)


@dataclasses.dataclass
class Reduced:
    pb: object                # the problem over the searched rows (same class as the input)
    topics: object            # TopicRows over the searched topics, renumbered, or None
    replication: object       # ReplicationRows of the searched rows, or None
    V0: int
    O0: int
    searched: np.ndarray      # int [P'] original row of each searched row


def reduce(pb, fixed, tr=None, rr=None):
    """The reduction of kao_solve_fixed (docs/MODEL.md §12), for masks the engine accepts."""
    from kafka_assignment_optimizer_b200.problem import ReplicationRows, TopicRows

    fx = np.asarray(fixed, bool)
    s = np.flatnonzero(~fx)
    f, fl, fr, o0, ft, flt = fixed_load(pb, fx, tr)
    shift = lambda lo, hi, load: (np.maximum(np.asarray(lo, np.int64) - load, 0).astype(np.int32),
                                  np.maximum(np.asarray(hi, np.int64) - load, 0).astype(np.int32),
                                  int(np.maximum(load - np.asarray(hi, np.int64), 0).sum()))
    rl, rh, v1 = shift(pb.rep_lo, pb.rep_hi, f)
    ll, lh, v2 = shift(pb.ldr_lo, pb.ldr_hi, fl)
    kl, kh, v3 = shift(pb.rack_lo, pb.rack_hi, fr)
    v0 = v1 + v2 + v3
    red = dataclasses.replace(pb, P=len(s), wF=pb.wF[s], wL=pb.wL[s], cur=pb.cur[s], rep_lo=rl, rep_hi=rh, ldr_lo=ll,
                              ldr_hi=lh, rack_lo=kl, rack_hi=kh,
                              topics=[pb.topics[p] for p in s] if pb.topics else None)
    if hasattr(red, "fixed"):
        red.fixed = None
    if hasattr(red, "replication"):
        red.replication = None
    rr2 = None if rr is None else ReplicationRows(*(np.asarray(x, np.int32)[s] for x in (rr.rf, rr.ppr_lo, rr.ppr_hi)))
    tr2 = None
    if tr is not None:
        topic_of = np.asarray(tr.topic_of)
        kept = sorted(set(topic_of[s].tolist()))
        for t in range(len(tr.rep_lo)):
            if t not in kept:
                v0 += _band(ft[t], tr.rep_lo[t], tr.rep_hi[t]) + _band(flt[t], tr.ldr_lo[t], tr.ldr_hi[t])
        new = {t: i for i, t in enumerate(kept)}
        pick = lambda x: np.asarray(x, np.int32)[kept]
        tr2 = TopicRows(np.array([new[t] for t in topic_of[s]], np.int32), pick(tr.rep_lo), pick(tr.rep_hi),
                        pick(tr.ldr_lo), pick(tr.ldr_hi), [tr.names[t] for t in kept] if tr.names else None)
    return Reduced(red, tr2, rr2, v0, o0, s)


def expand(pb, red, reduced_replicas):
    """[P, RF] replica lists: the searched rows from `reduced_replicas`, the fixed ones as cur lists them."""
    out = np.full((pb.P, pb.RF), -1, np.int32)
    for p in range(pb.P):
        row = fixed_row(pb, p)[:pb.RF]
        out[p, :len(row)] = row
    out[red.searched] = reduced_replicas
    return out


def acceptable(pb, p, RF=None):
    """Whether the engine accepts row p as a fixed row: non-empty, brokers before any -1, distinct, at most RF."""
    row = [int(b) for b in pb.cur[p]]
    n = sum(b >= 0 for b in row)
    return 0 < n <= (pb.RF if RF is None else RF) and all(b >= 0 for b in row[:n]) and len(set(row[:n])) == n


def holds_own_rows(pb, p, rr=None):
    """Whether row p, kept as cur lists it, satisfies its own C1, C2/C5 and C7 (with `rr`: rf[p], ppr_lo[p]..ppr_hi[p])."""
    row = fixed_row(pb, p)
    n, lo, hi = (pb.RF, pb.ppr_lo, pb.ppr_hi) if rr is None else (int(rr.rf[p]), int(rr.ppr_lo[p]), int(rr.ppr_hi[p]))
    pr = np.bincount([int(pb.rack_of[b]) for b in row], minlength=pb.R)
    return len(row) == n and len(set(row)) == n and bool(((pr >= lo) & (pr <= hi)).all())


def random_mask(pb, seed, share=0.5, tr=None, own=False):
    """A seeded mask over the acceptable rows (whole topics when `tr` is given), with at least one row searched; own:
    only rows that satisfy their own rows (holds_own_rows, with pb.replication when the problem has one)."""
    rng = np.random.RandomState(seed)
    ok = np.array([acceptable(pb, p) for p in range(pb.P)])
    if own:
        ok &= np.array([holds_own_rows(pb, p, getattr(pb, "replication", None)) for p in range(pb.P)])
    if tr is None:
        fx = ok & (rng.random_sample(pb.P) < share)
    else:
        topic_of = np.asarray(tr.topic_of)
        whole = np.array([ok[topic_of == t].all() for t in range(len(tr.rep_lo))])
        pick = whole & (rng.random_sample(len(whole)) < share)
        if not pick.any() and whole.any():
            pick[np.flatnonzero(whole)[0]] = True
        fx = pick[topic_of]
    if fx.all():
        fx[np.flatnonzero(fx)[0]] = False
        if tr is not None:
            fx[np.asarray(tr.topic_of) == tr.topic_of[np.flatnonzero(~fx)[0]]] = False
    return fx
