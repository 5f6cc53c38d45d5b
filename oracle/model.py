"""TEST INFRASTRUCTURE — exact CPU oracle for the assignment model (not shipped, not measured).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module.  The product path
(``kafka_assignment_optimizer_b200``) never does.

What this is
------------
A restatement of the 0/1 linear program the reference generates and hands to lp_solve
(``/root/reference/README.md:139-185``), solved here with HiGHS (``scipy.optimize.milp``)
because lp_solve 5.5 (``README.md:135-136``, ``:200``) is a third-party native dependency that
is neither vendored in the reference snapshot nor installed in this image.

PARITY STATUS: **parity unpinned against lp_solve** — the reference snapshot holds no source,
no tests and no golden vectors beyond one prose known-answer (``README.md:83-91``: remove
broker 19 → only partition 1 changes, ``[8,19] -> [8,1]``).  This oracle is pinned on that
vector (``tests/test_oracle_readme.py``).  HiGHS proves optimality, so the optimal objective
value (and every solver-independent quantity derived from it) is what lp_solve would also
return; lp_solve's *choice among co-optimal solutions* cannot be reproduced here.

Model (variables named as in README.md:146, ``t1b{b}p{p}`` / ``t1b{b}p{p}_l``)
    x[b,p] = 1  <=> broker b holds a follower replica of partition p
    l[b,p] = 1  <=> broker b holds the leader replica of partition p
    max  sum wF[p,b] x[b,p] + wL[p,b] l[b,p]                        README.md:145-146
    C1   sum_b x[b,p] + l[b,p]  = RF                    for all p   README.md:148-151
    C2   sum_b l[b,p]           = 1                     for all p   README.md:153-156
    C3   rep_lo[b] <= sum_p x[b,p]+l[b,p] <= rep_hi[b]  for all b   README.md:158-161
    C4   ldr_lo[b] <= sum_p l[b,p]        <= ldr_hi[b]  for all b   README.md:163-166
    C5   x[b,p] + l[b,p] <= 1                           for all b,p README.md:168-171
    C6   rack_lo[r] <= sum_{b in r} sum_p x+l <= rack_hi[r]  all r  README.md:173-176
    C7   ppr_lo <= sum_{b in r} x[b,p]+l[b,p] <= ppr_hi  all p,r    README.md:178-180
    C8   all variables binary                                       README.md:182-184

Everything the README does not determine (weights, bound formulas; SURVEY.md §A.3 G1-G4) is a
documented default in :func:`default_weights` / :func:`default_bounds`, mirrored by the product's
host code (``kafka_assignment_optimizer_b200/problem.py``) and by ``oracle/kao_ref.c``.
"""
from __future__ import annotations

import dataclasses
import math
import time
from typing import Dict, List, Optional, Sequence

import numpy as np

# --------------------------------------------------------------------------------------
# Problem description (dense broker indices 0..B-1 = position in the *target* broker list)
# --------------------------------------------------------------------------------------


@dataclasses.dataclass
class Problem:
    P: int
    B: int
    R: int
    RF: int
    rack_of: np.ndarray  # uint8 [B]
    wF: np.ndarray  # uint16 [P, B]  follower weight
    wL: np.ndarray  # uint16 [P, B]  leader weight
    rep_lo: np.ndarray  # int32 [B]   C3
    rep_hi: np.ndarray
    ldr_lo: np.ndarray  # int32 [B]   C4
    ldr_hi: np.ndarray
    rack_lo: np.ndarray  # int32 [R]  C6
    rack_hi: np.ndarray
    ppr_lo: int  # C7
    ppr_hi: int
    cur: np.ndarray  # int32 [P, RFcur]  dense indices, -1 = absent / on a removed broker
    broker_ids: np.ndarray  # int32 [B]   dense index -> Kafka broker id
    topics: Optional[list] = None  # per-row (topic, partition) labels for JSON round trip


WL_BY_POS = (4, 2, 1)  # SURVEY.md §A.3 G1 "reading A": leader weight by position in cur[p]
WF_BY_POS = (2, 2, 1)  # follower weight by position in cur[p]; positions >= 3 get 1


def _pos_weight(table, i):
    return table[i] if i < len(table) else 1


def default_weights(cur: np.ndarray, P: int, B: int):
    """README.md:116-120,131-133: existing placements get weight, the preferred (first) replica
    more.  Sample coefficients {1,2,4} at README.md:146."""
    wF = np.zeros((P, B), dtype=np.uint16)
    wL = np.zeros((P, B), dtype=np.uint16)
    for p in range(P):
        for i, b in enumerate(cur[p]):
            if b >= 0:
                wF[p, b] = _pos_weight(WF_BY_POS, i)
                wL[p, b] = _pos_weight(WL_BY_POS, i)
    return wF, wL


def default_bounds(P: int, B: int, R: int, RF: int, rack_of: np.ndarray):
    """SURVEY.md §A.3 G2-G4.  floor/ceil balance; rack totals proportional to rack size
    (uniform tot/R is infeasible after removing brokers)."""
    tot = P * RF
    rep_lo = np.full(B, tot // B, dtype=np.int32)
    rep_hi = np.full(B, -(-tot // B), dtype=np.int32)
    ldr_lo = np.full(B, P // B, dtype=np.int32)
    ldr_hi = np.full(B, -(-P // B), dtype=np.int32)
    size = np.bincount(rack_of, minlength=R).astype(np.int64)
    rack_lo = ((tot * size) // B).astype(np.int32)
    rack_hi = (-((-tot * size) // B)).astype(np.int32)
    ppr_lo = RF // R
    ppr_hi = -(-RF // R)
    return rep_lo, rep_hi, ldr_lo, ldr_hi, rack_lo, rack_hi, ppr_lo, ppr_hi


def build_problem(
    current: Sequence[Sequence[int]],
    broker_ids: Sequence[int],
    rack_by_broker: Dict[int, str],
    rf: int,
    topics: Optional[list] = None,
) -> Problem:
    """current[p] = ordered Kafka broker ids (leader first, README.md:52-63);
    broker_ids = target broker list (README.md:48); rack_by_broker = id -> rack/AZ name
    (README.md:27-29)."""
    broker_ids = sorted(int(b) for b in broker_ids)
    B = len(broker_ids)
    dense = {b: i for i, b in enumerate(broker_ids)}
    racks = sorted({str(rack_by_broker[b]) for b in broker_ids})
    ridx = {r: i for i, r in enumerate(racks)}
    rack_of = np.array([ridx[str(rack_by_broker[b])] for b in broker_ids], dtype=np.uint8)
    P = len(current)
    rfc = max(1, max(len(c) for c in current))
    cur = np.full((P, rfc), -1, dtype=np.int32)
    for p, reps in enumerate(current):
        for i, b in enumerate(reps):
            cur[p, i] = dense.get(int(b), -1)
    wF, wL = default_weights(cur, P, B)
    bounds = default_bounds(P, B, len(racks), rf, rack_of)
    return Problem(P, B, len(racks), rf, rack_of, wF, wL, *bounds, cur,
                   np.array(broker_ids, dtype=np.int32), topics)


def synthetic_problem(P: int, B0: int, R: int, RF: int, remove: int = 0,
                      perturb: float = 0.0, seed: int = 0) -> Problem:
    """SURVEY.md §8(d) synthetic input: rack_of[b] = b mod R, Kafka-style round robin
    cur[p] = [(p+i) mod B0 for i<RF]; `remove` drops the highest broker ids; `perturb` re-places
    that fraction of replicas at random (seeded) so that an already-optimal round robin
    (config 5) becomes a non-trivial search."""
    rng = np.random.RandomState(seed)
    current = [[(p + i) % B0 for i in range(RF)] for p in range(P)]
    if perturb > 0:
        n = int(round(perturb * P * RF))
        for _ in range(n):
            p = int(rng.randint(P))
            i = int(rng.randint(RF))
            nb = int(rng.randint(B0))
            if nb not in current[p]:
                current[p][i] = nb
    brokers = list(range(B0 - remove))
    racks = {b: "r%02d" % (b % R) for b in range(B0)}
    return build_problem(current, brokers, racks, RF)


def readme_problem() -> Problem:
    """The worked example, README.md:27-31 (topology), :48 (broker list), :52-63 (current)."""
    current = [[7, 18], [8, 19], [9, 10], [0, 11], [1, 12], [2, 13], [3, 14], [4, 15], [5, 16],
               [6, 17]]
    brokers = list(range(19))
    racks = {b: ("b" if b % 2 else "a") for b in range(20)}
    return build_problem(current, brokers, racks, 2,
                         topics=[("x.y.z.t", p) for p in range(10)])


def with_tiebreak(pb: Problem, K: Optional[int] = None) -> Problem:
    """SURVEY.md §8(c) T2: scale weights by K and add a per-(p,b) preference for the lowest
    broker index, K > P*RF*(B-1) so the preference can never outweigh one unit of real weight.
    Makes README.md:88's `[8,1]` the unique optimum of the worked example."""
    need = pb.P * pb.RF * (pb.B - 1) + 1
    if K is None:
        K = 1 << int(math.ceil(math.log2(need)))
    assert K >= need
    pref = (pb.B - 1 - np.arange(pb.B, dtype=np.int64))[None, :]
    wF = pb.wF.astype(np.int64) * K + pref
    wL = pb.wL.astype(np.int64) * K + pref
    if wF.max() > 65535 or wL.max() > 65535:
        raise ValueError("tie-broken weights exceed the 16-bit weight range of the C ABI")
    return dataclasses.replace(pb, wF=wF.astype(np.uint16), wL=wL.astype(np.uint16))


def with_random_tiebreak(pb: Problem, seed: int = 0) -> Problem:
    """T2 instances with a unique optimum on small problems: weights scaled by K plus a seeded
    random per-(p,b) preference whose total over any assignment stays below K, so only ties are
    broken.  Uniqueness is then *checked* with :func:`is_unique_optimum`, never assumed."""
    maxw = int(max(pb.wF.max(), pb.wL.max()))
    K = 1
    while (2 * K) * (maxw + 1) <= 65535:
        K *= 2
    q = (K - 1) // (pb.P * pb.RF)
    if q < 8:
        raise ValueError("problem too large for a 16-bit random tie-break")
    rng = np.random.RandomState(seed)
    wF = pb.wF.astype(np.int64) * K + rng.randint(0, q + 1, size=(pb.P, pb.B))
    wL = pb.wL.astype(np.int64) * K + rng.randint(0, q + 1, size=(pb.P, pb.B))
    assert wL.max() <= 65535 and wF.max() <= 65535
    return dataclasses.replace(pb, wF=wF.astype(np.uint16), wL=wL.astype(np.uint16))


# --------------------------------------------------------------------------------------
# Plain evaluation of one assignment (the model's semantics; loops, small cases)
# --------------------------------------------------------------------------------------


def evaluate(pb: Problem, replicas: np.ndarray):
    """replicas int [P, RF], leader first, dense indices.  Returns (violation, objective).
    violation = sum over C1..C7 of the amount by which each row is exceeded (0 <=> feasible)."""
    P, B, R = pb.P, pb.B, pb.R
    cnt = np.zeros(B, dtype=np.int64)
    lcnt = np.zeros(B, dtype=np.int64)
    viol = 0
    obj = 0
    for p in range(P):
        row = [int(b) for b in replicas[p] if b >= 0]
        uniq = set(row)
        viol += abs(len(uniq) - pb.RF)  # C1 (+C5: duplicates collapse)
        ld = row[0] if row else -1
        if ld < 0:
            viol += 1  # C2: no leader (C7's lower bound still applies to the empty row)
        else:
            lcnt[ld] += 1
            obj += int(pb.wL[p, ld])
        pr = np.zeros(R, dtype=np.int64)
        for b in uniq:
            cnt[b] += 1
            pr[pb.rack_of[b]] += 1
            if b != ld:
                obj += int(pb.wF[p, b])
        viol += int(np.maximum(pr - pb.ppr_hi, 0).sum() + np.maximum(pb.ppr_lo - pr, 0).sum())
    viol += int(np.maximum(cnt - pb.rep_hi, 0).sum() + np.maximum(pb.rep_lo - cnt, 0).sum())
    viol += int(np.maximum(lcnt - pb.ldr_hi, 0).sum() + np.maximum(pb.ldr_lo - lcnt, 0).sum())
    rc = np.bincount(pb.rack_of, weights=cnt, minlength=R).astype(np.int64)
    viol += int(np.maximum(rc - pb.rack_hi, 0).sum() + np.maximum(pb.rack_lo - rc, 0).sum())
    return viol, obj


def replica_moves(pb: Problem, replicas: np.ndarray) -> int:
    """SURVEY.md §A.2: number of (partition, broker) placements in the new assignment that the
    current one did not hold (data that must be copied); leader changes alone move nothing."""
    moves = 0
    for p in range(pb.P):
        have = {int(b) for b in pb.cur[p] if b >= 0}
        moves += sum(1 for b in replicas[p] if b >= 0 and int(b) not in have)     # -1 pads a short row
    return moves


# --------------------------------------------------------------------------------------
# The 0/1 program, solved exactly with HiGHS
# --------------------------------------------------------------------------------------


def _constraints(pb: Problem):
    """Sparse rows of C1..C7 over the variable vector [x (P*B) | l (P*B)], index p*B+b."""
    import scipy.sparse as sp

    P, B, R = pb.P, pb.B, pb.R
    n = P * B
    I = sp.identity(n, format="csr", dtype=np.float64)
    # per-partition sum over brokers: (P x n)
    Sp = sp.kron(sp.identity(P, format="csr"), np.ones((1, B)), format="csr")
    # per-broker sum over partitions: (B x n)
    Sb = sp.kron(np.ones((1, P)), sp.identity(B, format="csr"), format="csr")
    # rack membership (R x B)
    M = sp.csr_matrix((np.ones(B), (pb.rack_of.astype(np.int64), np.arange(B))), shape=(R, B))
    # per-partition-per-rack: (P*R x n)
    Spr = sp.kron(sp.identity(P, format="csr"), M, format="csr")
    Z = lambda m: sp.csr_matrix((m.shape[0], n))
    rows, lo, hi = [], [], []
    rows.append(sp.hstack([Sp, Sp]));  lo.append(np.full(P, pb.RF)); hi.append(np.full(P, pb.RF))  # C1
    rows.append(sp.hstack([Z(Sp), Sp])); lo.append(np.ones(P)); hi.append(np.ones(P))  # C2
    rows.append(sp.hstack([Sb, Sb])); lo.append(pb.rep_lo); hi.append(pb.rep_hi)  # C3
    rows.append(sp.hstack([Z(Sb), Sb])); lo.append(pb.ldr_lo); hi.append(pb.ldr_hi)  # C4
    rows.append(sp.hstack([I, I])); lo.append(np.zeros(n)); hi.append(np.ones(n))  # C5
    rows.append(sp.hstack([M @ Sb, M @ Sb])); lo.append(pb.rack_lo); hi.append(pb.rack_hi)  # C6
    rows.append(sp.hstack([Spr, Spr]))  # C7
    lo.append(np.full(P * R, pb.ppr_lo)); hi.append(np.full(P * R, pb.ppr_hi))
    A = sp.vstack(rows, format="csr")
    return A, np.concatenate(lo).astype(np.float64), np.concatenate(hi).astype(np.float64)


@dataclasses.dataclass
class Solution:
    status: str
    objective: Optional[int]
    replicas: Optional[np.ndarray]  # int32 [P, RF] leader first, followers ascending
    moves: Optional[int]
    solve_s: float
    build_s: float


def decode(pb: Problem, xv: np.ndarray) -> np.ndarray:
    """README.md:65-78,:88 — vars == 1 -> replicas list, leader first (Kafka's preferred leader
    is the first replica)."""
    P, B = pb.P, pb.B
    x = np.rint(xv[: P * B]).astype(np.int64).reshape(P, B)
    l = np.rint(xv[P * B:]).astype(np.int64).reshape(P, B)
    out = np.full((P, pb.RF), -1, dtype=np.int32)
    for p in range(P):
        ld = np.flatnonzero(l[p])
        fo = np.flatnonzero(x[p])
        row = list(ld) + list(fo)
        out[p, : len(row)] = row[: pb.RF]
    return out


def solve_exact(pb: Problem, time_limit: Optional[float] = None,
                extra_rows=None) -> Solution:
    from scipy.optimize import Bounds, LinearConstraint, milp

    t0 = time.perf_counter()
    A, lo, hi = _constraints(pb)
    if extra_rows is not None:
        import scipy.sparse as sp
        A = sp.vstack([A, extra_rows[0]], format="csr")
        lo = np.concatenate([lo, extra_rows[1]])
        hi = np.concatenate([hi, extra_rows[2]])
    c = -np.concatenate([pb.wF.reshape(-1), pb.wL.reshape(-1)]).astype(np.float64)
    t1 = time.perf_counter()
    opts = {"mip_rel_gap": 0.0}
    if time_limit:
        opts["time_limit"] = time_limit
    res = milp(c, constraints=LinearConstraint(A, lo, hi), integrality=np.ones(c.size),
               bounds=Bounds(0, 1), options=opts)
    t2 = time.perf_counter()
    if res.status == 0 and res.x is not None:
        reps = decode(pb, res.x)
        return Solution("optimal", int(round(-res.fun)), reps, replica_moves(pb, reps),
                        t2 - t1, t1 - t0)
    status = {2: "infeasible", 1: "limit", 3: "unbounded"}.get(res.status, "other")
    return Solution(status, None, None, None, t2 - t1, t1 - t0)


def is_unique_optimum(pb: Problem, sol: Solution) -> bool:
    """Add a no-good cut excluding `sol` and re-solve: unique iff the optimum drops."""
    import scipy.sparse as sp

    P, B = pb.P, pb.B
    n = P * B
    cols = []
    for p in range(P):
        cols.append(n + p * B + int(sol.replicas[p, 0]))
        for b in sol.replicas[p, 1:]:
            cols.append(p * B + int(b))
    row = sp.csr_matrix((np.ones(len(cols)), (np.zeros(len(cols), dtype=int), cols)),
                        shape=(1, 2 * n))
    cut = (row, np.array([-np.inf]), np.array([len(cols) - 1.0]))
    again = solve_exact(pb, extra_rows=cut)
    return again.status != "optimal" or again.objective < sol.objective


# --------------------------------------------------------------------------------------
# Kafka JSON helpers (README.md:52-63 in, :67-78 out)
# --------------------------------------------------------------------------------------


def to_kafka_json(pb: Problem, replicas: np.ndarray) -> dict:
    parts = []
    for p in range(pb.P):
        topic, part = pb.topics[p] if pb.topics else ("t1", p)
        parts.append({"topic": topic, "partition": part,
                      "replicas": [int(pb.broker_ids[b]) for b in replicas[p]]})
    return {"version": 1, "partitions": parts}
