"""The Lagrangian LP bound (docs/MODEL.md §9) without a GPU: its plain-C restatement (tests/lp_ref) is sound — never
below the LP relaxation of the 0/1 program or the exact optimum, never above L(0) — and exact: L re-evaluated at
the multipliers it returns, in rational arithmetic with an independent enumeration of every partition's rows, floors
to the reported bound.  It proves the small golden optima within the default cap.  kao_lp_bound refuses infeasible
assignments and, without a device, fails loudly."""
import dataclasses
import itertools
from fractions import Fraction

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import lp_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import LAYOUT_SHAPES, SHAPES

ALL = {**SHAPES, **LAYOUT_SHAPES}
SOUND = ["readme", "readme_tb", "cfg2", "cfg2_rm2", "cfg3_small", "tiny", "one_partition", "dense_small", "dense_unique",
         "ppr11_w4", "rack4_w2", "rack3_w8", "rack5_w2", "dense_rack4_w1", "dense_rack4_w2", "dense_ppr11_w4",
         "dense_s64_r1"]
SMALL = ["readme", "readme_tb", "tiny", "one_partition", "dense_small", "dense_unique", "dense_unique2"]


def far_assignment(pb):
    """A feasible assignment far from the optimum: the optimum of the same constraints under unrelated weights."""
    rng = np.random.RandomState(4)
    other = dataclasses.replace(pb, wF=rng.randint(0, 3, size=pb.wF.shape).astype(np.uint16),
                                wL=rng.randint(0, 5, size=pb.wL.shape).astype(np.uint16))
    reps = m.solve_exact(other).replicas
    assert m.evaluate(pb, reps)[0] == 0
    return reps


def lp_relaxation(pb):
    """The LP relaxation of the whole 0/1 program (oracle/model.py's rows, integrality off), by HiGHS."""
    from scipy.optimize import Bounds, LinearConstraint, milp

    A, lo, hi = m._constraints(pb)
    c = -np.concatenate([pb.wF.reshape(-1), pb.wL.reshape(-1)]).astype(np.float64)
    res = milp(c, constraints=LinearConstraint(A, lo, hi), integrality=np.zeros(c.size), bounds=Bounds(0, 1))
    assert res.status == 0
    return -res.fun


def lagrangian(pb, u):
    """L(u) of MODEL §9 as a Fraction, u given with lp_ref.fraction_bits() fractional bits; best_p by enumerating
    every row (RF distinct brokers, one of them the leader) that satisfies C7."""
    one = 1 << lp_ref.fraction_bits()
    B, R = pb.B, pb.R
    u3 = [Fraction(int(x), one) for x in u[:B]]
    u4 = [Fraction(int(x), one) for x in u[B:2 * B]]
    u6 = [Fraction(int(x), one) for x in u[2 * B:]]
    tot = pb.P * pb.RF
    rows = [(u3[b], pb.rep_lo[b], min(pb.rep_hi[b], tot)) for b in range(B)] + \
           [(u4[b], pb.ldr_lo[b], min(pb.ldr_hi[b], pb.P)) for b in range(B)] + \
           [(u6[r], pb.rack_lo[r], min(pb.rack_hi[r], tot)) for r in range(R)]
    L = sum((x * int(hi) if x > 0 else x * int(lo)) for x, lo, hi in rows)
    for p in range(pb.P):
        best = None
        for s in itertools.combinations(range(B), pb.RF):
            per_rack = np.bincount(pb.rack_of[list(s)], minlength=R)
            if per_rack.min() < pb.ppr_lo or per_rack.max() > pb.ppr_hi:
                continue
            fol = sum(int(pb.wF[p, b]) - u3[b] - u6[pb.rack_of[b]] for b in s)
            for ld in s:
                v = fol - (int(pb.wF[p, ld]) - u3[ld] - u6[pb.rack_of[ld]]) + int(pb.wL[p, ld]) - u3[ld] - u4[ld] - u6[pb.rack_of[ld]]
                best = v if best is None or v > best else best
        L += best
    return L


@pytest.mark.parametrize("name", SOUND)
def test_the_restatement_is_sound(name):
    pb = ALL[name]()
    sol = m.solve_exact(pb)
    assert sol.status == "optimal"
    lp = lp_relaxation(pb)
    L0 = lp_ref.lp_bound(pb, sol.objective, 1)[0]
    for T in (sol.objective, m.evaluate(pb, far_assignment(pb))[1]):
        bound, its, _ = lp_ref.lp_bound(pb, T, kopt.LP_ITERATIONS)
        assert int(np.floor(lp + 1e-6)) <= bound <= L0 and bound >= sol.objective, (T, lp, bound, L0)
        assert 1 <= its <= kopt.LP_ITERATIONS


@pytest.mark.parametrize("name", SMALL)
def test_the_bound_is_exact(name):
    """Aimed below the optimum the iteration cannot stop early, so the multipliers move; L at the multipliers it
    returns, in rational arithmetic, floors to its bound."""
    pb = ALL[name]()
    opt = m.solve_exact(pb).objective
    moved = False
    for T, cap in ((opt, kopt.LP_ITERATIONS), (opt - 3, 7), (opt - 3, 60)):
        bound, its, u = lp_ref.lp_bound(pb, T, cap)
        L = lagrangian(pb, u)
        assert L.numerator // L.denominator == bound and bound >= opt, (T, cap)
        moved |= bool(u.any())
        assert (np.abs(u) <= lp_ref.box()).all()
    assert moved or lp_ref.lp_bound(pb, opt, 1)[0] == opt      # moved unless L(0) is already the optimum


@pytest.mark.parametrize("name", ["readme", "cfg2", "cfg2_rm2", "cfg3_small"])
def test_the_restatement_proves_the_small_optima(name):
    pb = ALL[name]()
    opt = m.solve_exact(pb).objective
    bound, its, _ = lp_ref.lp_bound(pb, opt, kopt.LP_ITERATIONS)
    assert bound == opt and its <= kopt.LP_ITERATIONS


def test_an_infeasible_or_malformed_assignment_is_refused():
    pb = SHAPES["cfg2_rm2"]()
    kp = kao.Problem.from_fields(pb)
    reps = m.solve_exact(pb).replicas
    bad = reps.copy()
    bad[3, 1] = bad[3, 0]                                    # a broker twice (C5)
    with pytest.raises(kao.KaoError, match="twice"):
        kopt.lp_bound(kp, bad)
    bad = reps.copy()
    bad[0] = [0, 4, 8]                                       # three replicas in one rack: C7 (0..1 here)
    assert pb.rack_of[0] == pb.rack_of[4] == pb.rack_of[8]
    with pytest.raises(kao.KaoError, match="violates C7"):
        kopt.lp_bound(kp, bad)
    bad = reps.copy()
    bad[5, 2] = -1                                           # a short row (C1)
    with pytest.raises(kao.KaoError, match="C1"):
        kopt.lp_bound(kp, bad)
    with pytest.raises(kao.KaoError, match="max_iterations"):
        kopt.lp_bound(kp, reps, max_iterations=0)


def test_no_gpu_means_loud_failure():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    pb = SHAPES["cfg2_rm2"]()
    with pytest.raises(kao.KaoError, match="libkao error -2: no CUDA device"):
        kopt.lp_bound(kao.Problem.from_fields(pb), m.solve_exact(pb).replicas)


def test_service_passes_the_lp_certificate_on():
    """POST /submit {"lp_certificate": true} asks the solver for the LP bound (kao_solve's KAO_FLAG_LP_BOUND)."""
    import json

    from kafka_assignment_optimizer_b200 import service
    from test_host import README_CURRENT
    from test_service import SEEN, oracle_solver

    body = {"assignment": json.loads(README_CURRENT), "brokers": ",".join(map(str, range(19))),
            "racks": ",".join("%d:%s" % (b, "b" if b % 2 else "a") for b in range(20)), "rf": 2}
    for flag in (True, False):
        out = service.handle_submit({**body, "lp_certificate": flag}, solver=oracle_solver)
        assert SEEN["lp_bound"] is flag and out["objective"] == 58
