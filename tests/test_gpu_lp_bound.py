"""kao_lp_bound on the GPU (csrc/kao_lagrange.cu, docs/MODEL.md §9): the kernel's integer iteration is the
restatement's (tests/lp_ref) bit for bit — bound, iterations run and multipliers — and it proves optima the flow
bound cannot: config 4 (1000 x 64 x 8, brokers 62 and 63 removed) through kao_solve, kao_lp_bound and kao-cli."""
import json
import os
import subprocess

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import lp_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import LAYOUT_SHAPES, SHAPES
from test_lp_bound import far_assignment

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CLI = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "kao-cli")
CFG4_RECIPE = dict(seed=7, rounds=400, round_size=1 << 12, patience=150, restarts=12)    # tests/test_gpu_configs.py
CFG3_RECIPE = dict(rounds=2000, round_size=1 << 14, patience=100)                         # INTEGRATION.md 5
# shapes of every layout class and C7 form, dense and 12-bit weights
PARITY = ["readme", "readme_tb", "cfg2_rm2", "cfg3_small", "rf_up", "rf_down", "w4_s16", "s64_r1", "dense_small",
          "dense_unique", "rf1", "rack5_w8_r4", "ppr11_w4", "rack4_w2", "rack3_w4", "dense_rack4_w1", "dense_ppr11_w4",
          "w12_cfg2_rm2", "w12_readme"]
KS = (1, 7, 100, kopt.LP_ITERATIONS)


@pytest.fixture(scope="module")
def optima():
    with open(os.path.join(GOLDEN, "optima.json")) as f:
        return json.load(f)


def _same(pb, replicas, T=None):
    """kernel vs restatement after every k of KS; T defaults to the objective of `replicas`"""
    kp = kao.Problem.from_fields(pb)
    T = m.evaluate(pb, replicas)[1] if T is None else T
    out = []
    for k in KS:
        bound, its, u = kopt.lp_bound(kp, replicas, max_iterations=k, multipliers=True)
        want = lp_ref.lp_bound(pb, T, k)
        assert (bound, its) == want[:2], (k, (bound, its), want[:2])
        assert (u == want[2]).all(), k
        out.append((bound, its))
    return out


@pytest.mark.parametrize("name", PARITY)
def test_kernel_matches_the_restatement_bit_for_bit(name):
    """From the optimum (the iteration aims at a reachable target) and from a far feasible assignment (it cannot
    reach its target and runs to the cap): every trajectory is the restatement's."""
    pb = {**SHAPES, **LAYOUT_SHAPES}[name]()
    sol = m.solve_exact(pb)
    got = _same(pb, sol.replicas)
    assert all(b >= sol.objective for b, _ in got)
    far = far_assignment(pb)
    got = _same(pb, far)
    assert all(b >= sol.objective for b, _ in got)


def test_kernel_matches_the_restatement_on_config5_prime(optima):
    """Config 5' (4096 x 256 x 16, 2 % of the replicas re-placed; W = 8 rows, 16 racks): from its exact optimum
    (tests/golden/cfg5_p02_optimum.npy) the kernel and the restatement walk the same trajectory."""
    e = optima["cfg5_p02"]
    pb = m.synthetic_problem(*e["args"])
    opt = np.load(os.path.join(GOLDEN, "cfg5_p02_optimum.npy")).astype(np.int32)
    assert m.evaluate(pb, opt) == (0, e["objective"])
    got = _same(pb, opt)
    assert all(b >= e["objective"] for b, _ in got)


def test_config4_is_proven_optimal_through_kao_solve(optima):
    """The README's headline use case, removing brokers: the flow bound stops at 6790 here, the LP bound proves
    the search's 6787 optimal."""
    e = optima["cfg4"]
    pb = m.synthetic_problem(*e["args"])
    kp = kao.Problem.from_fields(pb)
    flow = kopt.solve(kp, tight_bound=True, **CFG4_RECIPE)
    assert (flow.objective, flow.moves) == (e["objective"], e["moves"]) and flow.objective_bound > flow.objective
    res = kopt.solve(kp, lp_bound=True, **CFG4_RECIPE)
    assert (res.replicas == flow.replicas).all()
    assert res.feasible and res.objective == res.objective_bound == e["objective"] and res.optimal


@pytest.mark.parametrize("cfg", ["cfg3", "cfg4"])
def test_configs_3_and_4_are_proven_through_kao_lp_bound(optima, cfg):
    e = optima[cfg]
    pb = m.synthetic_problem(*e["args"])
    kp = kao.Problem.from_fields(pb)
    res = kopt.solve(kp, **(CFG4_RECIPE if cfg == "cfg4" else CFG3_RECIPE))
    assert res.feasible and res.objective == e["objective"]
    bound, its = kopt.lp_bound(kp, res.replicas)
    assert bound == e["objective"] and 1 <= its <= kopt.LP_ITERATIONS
    assert (bound, its) == lp_ref.lp_bound(pb, e["objective"], kopt.LP_ITERATIONS)[:2]


def test_the_bound_is_never_below_the_exact_optimum(optima):
    """Every optima.json instance, from a feasible assignment: the exact optimum (small ones), the search's result
    (configs 3 and 4), the stored optimum (config 5')."""
    for name, e in optima.items():
        pb = m.readme_problem() if e["args"] is None else m.synthetic_problem(*e["args"])
        kp = kao.Problem.from_fields(pb)
        if name == "cfg5_p02":
            reps = np.load(os.path.join(GOLDEN, "cfg5_p02_optimum.npy")).astype(np.int32)
        elif name in ("cfg3", "cfg4"):
            reps = kopt.solve(kp, **(CFG4_RECIPE if name == "cfg4" else CFG3_RECIPE)).replicas
        else:
            reps = m.solve_exact(pb).replicas
        assert m.evaluate(pb, reps)[0] == 0
        for k in (1, 50, kopt.LP_ITERATIONS):
            assert kopt.lp_bound(kp, reps, max_iterations=k)[0] >= e["objective"], (name, k)


def test_cli_lp_certificate_proves_config4(tmp_path, optima):
    e = optima["cfg4"]
    P, B0, R, RF, remove = e["args"]
    doc = {"version": 1, "partitions": [{"topic": "t1", "partition": p, "replicas": [(p + i) % B0 for i in range(RF)]}
                                        for p in range(P)]}
    f = tmp_path / "current.json"
    f.write_text(json.dumps(doc))
    racks = ",".join("%d:r%02d" % (b, b % R) for b in range(B0))
    r = CFG4_RECIPE
    p = subprocess.run([CLI, "--assignment", str(f), "--brokers", ",".join(map(str, range(B0 - remove))), "--racks", racks,
                        "--seed", str(r["seed"]), "--rounds", str(r["rounds"]), "--round-size", str(r["round_size"]),
                        "--patience", str(r["patience"]), "--restarts", str(r["restarts"]), "--lp-certificate", "--stats"],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    assert "objective %d (upper bound %d: proven optimal)" % (e["objective"], e["objective"]) in p.stderr, p.stderr
