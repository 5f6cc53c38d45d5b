"""kao_lp_bound on the GPU at the build limits of docs/MODEL.md §9 (csrc/kao_lagrange.cu), on the limit shapes of
tests/test_lp_limits.py and the CTA grids of this device: after every iteration cap the kernel returns the
restatement's bound, iterations and multipliers bit for bit, from a good and from a far feasible assignment; its bound
is ⌊L_exact(u) / 2^F⌋ at its own multipliers (tests/lp_exact.py, no DP in common with either); a second call returns
the same.  At 8,160 × 64 × RF 8, kao_solve with the flow and the LP bound returns objective <= bound <= flow bound.

From 8,159 rows on, the rows of these shapes (64 and 256 slots) do not fit the shared-memory search, which refuses
them; kao_solve_fixed with no row fixed searches them on the HBM path and computes the LP bound on the whole problem
(docs/MODEL.md §12), so that is how the search's result and kao_solve's LP bound are taken there."""
import functools

import numpy as np
import pytest
import torch

import kafka_assignment_optimizer_b200 as kao
import lp_exact
import lp_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from test_lp_bound import far_assignment
from test_lp_limits import LIMITS, SMS, grid_shapes, instance, iterations, last_cta, windows_assignment

pytestmark = pytest.mark.gpu
N = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else SMS
GRIDS = grid_shapes(N)
SEARCH = dict(seed=11, rounds=20000, round_size=1 << 12, patience=500)


def problem(name):
    if name in LIMITS:
        return instance(name)
    pb = GRIDS[name][0]()
    reps = windows_assignment(pb)
    viol, obj = m.evaluate(pb, reps)
    assert viol == 0
    return pb, reps, obj


@functools.lru_cache(maxsize=None)
def searched(name, tight_bound=False):
    """kao_solve's result with the LP bound (KAO_FLAG_LP_BOUND), and with the flow bound too (KAO_FLAG_BOUND: host
    time that grows with the brokers, minutes at 8,160 x 256; so only where it is checked, at 64 brokers)"""
    pb = problem(name)[0]
    kp = kao.Problem.from_fields(pb)
    if pb.P >= 8159:
        kp.fixed = np.zeros(pb.P, bool)
    return kopt.solve(kp, tight_bound=tight_bound, lp_bound=True, **SEARCH)


def assignments(name):
    """the optimum or the search's result, and a feasible assignment further from it (far_assignment, or the windows
    assignment, which ignores the re-placed replicas)"""
    pb, reps, _ = problem(name)
    if LIMITS.get(name, (None, "windows"))[1] == "exact":
        return [reps, far_assignment(pb)]
    res = searched(name)
    assert res.feasible, name
    return [res.replicas, reps]


def _same(name, pb, replicas):
    kp = kao.Problem.from_fields(pb)
    T = m.evaluate(pb, replicas)[1]
    for k in iterations(name):
        got = kopt.lp_bound(kp, replicas, max_iterations=k, multipliers=True)
        want = lp_ref.lp_bound(pb, T, k)
        assert got[:2] == want[:2] and (got[2] == want[2]).all(), (name, k, got[:2], want[:2])
        assert lp_exact.lagrangian_fixed(pb, got[2]) >> lp_exact.F == got[0], (name, k)
        assert got[0] >= T
    again = kopt.lp_bound(kp, replicas, max_iterations=k, multipliers=True)
    assert again[:2] == got[:2] and (again[2] == got[2]).all()
    return got


@pytest.mark.parametrize("name", list(LIMITS) + list(GRIDS))
def test_kernel_matches_the_restatement_at_the_limits(name):
    pb = problem(name)[0]
    for reps in assignments(name):
        _same(name, pb, reps)


def test_the_grid_has_a_short_last_cta():
    assert any(last_cta(P, N)[1] < last_cta(P, N)[0] for P in (2 * N + 1, 8159, 8160))


def test_solve_with_the_lp_bound_at_8160_partitions():
    """4,096 iterations at 8,160 x 64 x RF 8 inside kao_solve, with the flow bound: the bound it returns is the smaller
    of the flow bound and kao_lp_bound's at the same objective, never below that objective, and optimality is claimed
    exactly when it meets the objective"""
    pb = problem("size_8160_b64")[0]
    res = searched("size_8160_b64", tight_bound=True)
    assert res.feasible and m.evaluate(pb, res.replicas) == (0, res.objective)
    assert (res.replicas == searched("size_8160_b64").replicas).all()
    kp = kao.Problem.from_fields(pb)
    lp, its = kopt.lp_bound(kp, res.replicas)
    assert 1 <= its <= kopt.LP_ITERATIONS
    assert res.objective <= res.objective_bound <= min(lp, searched("size_8160_b64").objective_bound), (res.objective, res.objective_bound, lp)
    assert res.optimal == (res.objective == res.objective_bound)
