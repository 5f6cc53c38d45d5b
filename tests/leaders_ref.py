"""TEST INFRASTRUCTURE — leader-only rebalancing (docs/MODEL.md §13) stated directly, sharing no code with the flow.

* :func:`solve_exact` writes the restricted program for HiGHS (``scipy.optimize.milp``): a binary ``l[p, k]`` for each
  current replica k of row p only (a fixed row's current leader forced to 1), C2 per row, C4 per broker and C4t per
  (topic, broker) with slack variables, and the objective ``M * slack - gain``; M exceeds every possible gain, so the
  optimum is the lexicographic one.
* :func:`enumerate_all` tries every choice of leaders (small instances only).
* :func:`fixed_part` is the violation of C1, C3, C5, C6, C7 and C3t of the current replica sets.
"""
import itertools

import numpy as np


def rows(pb):
    return [[int(b) for b in pb.cur[p] if b >= 0] for p in range(pb.P)]


def _band(c, lo, hi):
    return int(np.maximum(np.asarray(lo) - c, 0).sum() + np.maximum(c - np.asarray(hi), 0).sum())


def fixed_part(pb, tr=None):
    rs = rows(pb)
    v, cnt = 0, np.zeros(pb.B, np.int64)
    T = 0 if tr is None else len(tr.rep_lo)
    tcnt = np.zeros((T, pb.B), np.int64)
    for p, r in enumerate(rs):
        v += abs(len(r) - pb.RF) + (len(set(r)) != len(r))
        per = np.bincount([int(pb.rack_of[b]) for b in r], minlength=pb.R)
        v += _band(per, pb.ppr_lo, pb.ppr_hi)
        for b in r:
            cnt[b] += 1
            if tr is not None:
                tcnt[tr.topic_of[p], b] += 1
    v += _band(cnt, pb.rep_lo, pb.rep_hi)
    v += _band(np.bincount(pb.rack_of, weights=cnt, minlength=pb.R).astype(np.int64), pb.rack_lo, pb.rack_hi)
    if tr is not None:
        v += _band(tcnt, np.asarray(tr.rep_lo)[:, None], np.asarray(tr.rep_hi)[:, None])
    return v


def leader_part(pb, leaders, tr=None):
    """(C4 + C4t violation, objective) of the rows of pb.cur led from `leaders` [P]"""
    lc = np.bincount(np.asarray(leaders), minlength=pb.B)
    v = _band(lc, pb.ldr_lo, pb.ldr_hi)
    if tr is not None:
        tl = np.zeros((len(tr.rep_lo), pb.B), np.int64)
        for p, b in enumerate(leaders):
            tl[tr.topic_of[p], b] += 1
        v += _band(tl, np.asarray(tr.ldr_lo)[:, None], np.asarray(tr.ldr_hi)[:, None])
    obj = 0
    for p, r in enumerate(rows(pb)):
        obj += sum(int(pb.wL[p, b]) if b == leaders[p] else int(pb.wF[p, b]) for b in r)
    return v, obj


def solve_exact(pb, tr=None, fixed=None):
    """-> (C4 + C4t violation, objective, leaders [P]) of the lexicographic optimum"""
    import scipy.sparse as sp
    from scipy.optimize import Bounds, LinearConstraint, milp

    rs = rows(pb)
    fx = np.zeros(pb.P, bool) if fixed is None else np.asarray(fixed, bool)
    var = [(p, b) for p, r in enumerate(rs) for b in r]
    n = len(var)
    gain = np.array([int(pb.wL[p, b]) - int(pb.wF[p, b]) for p, b in var], np.float64)
    M = 1 + sum(max(int(pb.wL[p, b]) - int(pb.wF[p, b]) for b in r) - min(int(pb.wL[p, b]) - int(pb.wF[p, b]) for b in r)
                for p, r in enumerate(rs) if not fx[p])
    cells = [("b", b) for b in range(pb.B)]
    if tr is not None:
        cells += [("t", t, b) for t in range(len(tr.rep_lo)) for b in range(pb.B)]
    ns = 2 * len(cells)                                   # (over hi, under lo) per row
    A, lo, hi = [], [], []
    for p in range(pb.P):
        A.append(([i for i, (q, _) in enumerate(var) if q == p], [], []))
        lo.append(1), hi.append(1)
    for j, cell in enumerate(cells):
        if cell[0] == "b":
            idx = [i for i, (_, b) in enumerate(var) if b == cell[1]]
            clo, chi = int(pb.ldr_lo[cell[1]]), int(pb.ldr_hi[cell[1]])
        else:
            idx = [i for i, (q, b) in enumerate(var) if b == cell[2] and tr.topic_of[q] == cell[1]]
            clo, chi = int(tr.ldr_lo[cell[1]]), int(tr.ldr_hi[cell[1]])
        A.append((idx, [2 * j], [-1.0])); lo.append(-np.inf), hi.append(chi)
        A.append((idx, [2 * j + 1], [1.0])); lo.append(clo), hi.append(np.inf)
    data, ri, ci = [], [], []
    for r, (idx, sidx, sval) in enumerate(A):
        data += [1.0] * len(idx) + sval
        ri += [r] * (len(idx) + len(sidx))
        ci += idx + [n + s for s in sidx]
    mat = sp.csr_matrix((data, (ri, ci)), shape=(len(A), n + ns))
    c = np.concatenate([-gain, np.full(ns, float(M))])
    vlo, vhi = np.zeros(n + ns), np.concatenate([np.ones(n), np.full(ns, np.inf)])
    for i, (p, b) in enumerate(var):
        if fx[p]:
            vlo[i] = vhi[i] = 1.0 if b == rs[p][0] else 0.0
    res = milp(c, constraints=LinearConstraint(mat, lo, hi), integrality=np.concatenate([np.ones(n), np.zeros(ns)]),
               bounds=Bounds(vlo, vhi), options={"mip_rel_gap": 0.0})
    assert res.status == 0, res.message
    x = np.rint(res.x[:n]).astype(int)
    leaders = np.full(pb.P, -1)
    for i in np.flatnonzero(x):
        leaders[var[i][0]] = var[i][1]
    v, obj = leader_part(pb, leaders, tr)
    assert round(res.fun) == M * v - (obj - sum(int(pb.wF[p, b]) for p, r in enumerate(rs) for b in r))
    return v, obj, leaders


def enumerate_all(pb, tr=None, fixed=None):
    """-> the least (C4 + C4t violation, -objective) over every choice of leaders"""
    rs = rows(pb)
    fx = np.zeros(pb.P, bool) if fixed is None else np.asarray(fixed, bool)
    options = [[r[0]] if fx[p] else r for p, r in enumerate(rs)]
    best = None
    for leaders in itertools.product(*options):
        v, obj = leader_part(pb, leaders, tr)
        if best is None or (v, -obj) < best:
            best = (v, -obj)
    return best[0], -best[1]
