"""Fixed partitions on the GPU (docs/MODEL.md §12): kao_solve_fixed is kao_solve* on the reduced problem that the
Python restatement (tests/fixed_ref.py) builds, bit for bit on the searched rows, key and rounds; fixed rows come back as
cur lists them; the full output scored on the full problem is the reported violation / objective; a cluster above 8,160
partitions with at most 8,160 free rows runs on the shared-memory path, with its options and certificates; V0 > 0 is
KAO_INFEASIBLE."""
import dataclasses

import numpy as np
import pytest

import fixed_ref as F
import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import SHAPES, SLOT255_TOPIC_SHAPES
from test_replication_cpu import readme_mixed, seeded_mixed
from test_topics_cpu import sixteen_topics

pytestmark = pytest.mark.gpu

OPTS = dict(seed=0xF1, rounds=24, round_size=4096, restarts=2)


def big_plain():
    return m.synthetic_problem(20000, 64, 8, 3, remove=1, perturb=0.02, seed=3)


def big_topics():
    return SLOT255_TOPIC_SHAPES["sized_big"]()


def big_mixed():
    return seeded_mixed(8, [6] * 8, [(4000, 3), (3000, 2), (2500, 1)], removed=1)


def _mask_of_share(pb, seed, share, tr=None, own=True):
    fx = F.random_mask(pb, seed, share=share, tr=tr, own=own)
    assert fx.any() and not fx.all()
    return fx


# name -> (problem, topic rows or None, mask); every mask is one the engine accepts
def _cases():
    out = {}
    out["cfg2"] = lambda: (lambda pb: (pb, None, _mask_of_share(pb, 1, 0.5)))(SHAPES["cfg2_rm2"]())
    out["plain_free_below"] = lambda: (lambda pb: (pb, None, _mask_of_share(pb, 2, 0.8)))(big_plain())
    out["plain_free_between"] = lambda: (lambda pb: (pb, None, _mask_of_share(pb, 10, 0.64)))(big_plain())
    out["plain_free_above"] = lambda: (lambda pb: (pb, None, _mask_of_share(pb, 3, 0.3)))(big_plain())
    out["topics_small"] = lambda: (lambda t: (t[0], t[1], _mask_of_share(t[0], 4, 0.5, t[1])))(sixteen_topics())
    out["topics_below"] = lambda: (lambda pb: (lambda tr: (pb, tr, _mask_of_share(pb, 5, 0.5, tr, own=False)))(
        kao.topic_rows(kao.Problem.from_fields(pb))))(big_topics())
    out["topics_above"] = lambda: (lambda pb: (lambda tr: (pb, tr, _mask_of_share(pb, 6, 0.0, tr, own=False)))(
        kao.topic_rows(kao.Problem.from_fields(pb))))(big_topics())
    out["mixed_small"] = lambda: (lambda pb: (pb, None, _mask_of_share(pb, 7, 0.5)))(readme_mixed())
    out["mixed_below"] = lambda: (lambda pb: (pb, None, _mask_of_share(pb, 8, 0.7)))(big_mixed())
    out["mixed_above"] = lambda: (lambda pb: (pb, None, _mask_of_share(pb, 9, 0.05)))(big_mixed())
    return out


CASES = _cases()
# the masks of these cases fix only rows that satisfy their own rows, so the full output can be scored on the full problem
SCORED = {"cfg2", "plain_free_below", "plain_free_between", "plain_free_above", "topics_small", "mixed_small",
          "mixed_below", "mixed_above"}
# 33..64 broker slots: the shared-memory plan holds at most 7,680 rows (make_plan, packed entries), so between that and
# 8,160 rows the reduced problem runs on the HBM path with uniform replication rows
SMEM_W2_ROWS = 7680


def _uniform(pb):
    return kao.ReplicationRows(np.full(pb.P, pb.RF, np.int32), np.full(pb.P, pb.ppr_lo, np.int32),
                               np.full(pb.P, pb.ppr_hi, np.int32))


def _solve_both(opb, tr, fx, **kw):
    pb = kao.Problem.from_fields(opb)
    rr = pb.replication
    red = F.reduce(pb, fx, tr, rr)
    rrr = red.replication
    if rr is None and tr is None and SMEM_W2_ROWS < red.pb.P <= 8160:
        rrr = _uniform(red.pb)
    rpb = dataclasses.replace(red.pb, replication=rrr)
    opts = dict(OPTS, **kw)
    got = kopt.solve(dataclasses.replace(pb, fixed=fx), topics=tr, **opts)
    want = kopt.solve(rpb, topics=red.topics, **opts)
    return pb, rr, red, got, want


@pytest.mark.parametrize("name", sorted(CASES))
def test_solve_fixed_is_the_reduced_solve(name):
    opb, tr, fx = CASES[name]()
    pb, rr, red, got, want = _solve_both(opb, tr, fx)
    if "below" in name:
        assert red.pb.P <= 8160 < pb.P
    if "between" in name:
        assert SMEM_W2_ROWS < red.pb.P <= 8160
    if "above" in name:
        assert red.pb.P > 8160
    # the searched rows, key and rounds of the reduced search; the constants on top
    assert np.array_equal(got.replicas[red.searched], want.replicas)
    assert (got.key, got.rounds, got.key_obj_bits, got.moves) == (want.key, want.rounds, want.key_obj_bits, want.moves)
    assert got.violation == want.violation + red.V0 and got.objective == want.objective + red.O0
    assert got.objective_bound == want.objective_bound + red.O0
    assert got.feasible == (got.violation == 0) and got.optimal == (want.optimal and red.V0 == 0)
    # fixed rows byte for byte as cur lists them
    assert np.array_equal(got.replicas[fx], F.expand(pb, red, want.replicas)[fx])
    # where the fixed rows satisfy their own rows, the full output scored on the full problem is the result
    full = got.replicas
    whole = F.evaluate(opb, fx, full, tr, rr) == F.evaluate(opb, np.zeros(pb.P, bool), full, tr, rr)
    assert whole or name not in SCORED
    if whole:
        if tr is None and rr is None:
            v, o = kopt.evaluate(pb, full)
            assert (int(v[0]), int(o[0])) == (got.violation, got.objective)
        else:
            s = kao.Session(pb, topics=tr)
            s.set_base(full)
            _, v, o, _ = s.get_base()
            s.close()
            assert (v, o) == (got.violation, got.objective)


def test_options_of_the_shared_memory_path_apply_to_the_reduced_problem():
    """A cluster of 20,000 partitions with 4,932 free rows: row-major evaluation and the LP certificate are accepted for
    the fixed call and refused for the whole cluster (the HBM path)"""
    opb = big_plain()
    pb = kao.Problem.from_fields(opb)
    fx = _mask_of_share(pb, 2, 0.8)
    red = F.reduce(pb, fx)
    assert red.pb.P <= 8160 < pb.P
    for kw in (dict(row_major=True), dict(lp_bound=True)):
        _, _, _, got, want = _solve_both(opb, None, fx, **kw)
        assert np.array_equal(got.replicas[red.searched], want.replicas) and got.key == want.key
        with pytest.raises(kopt.KaoError):
            kopt.solve(pb, **dict(OPTS, **kw))


def test_reduced_problem_too_large_for_shared_memory_runs_on_the_hbm_path():
    """7,680 < P' <= 8,160 rows at 64 brokers: the call is served on the HBM path (kao_solve of that reduced problem is
    refused); KAO_FLAG_LP_BOUND still adds the LP bound of the plain reduced problem, row-major evaluation is refused"""
    opb, _, fx = CASES["plain_free_between"]()
    pb = kao.Problem.from_fields(opb)
    red = F.reduce(pb, fx)
    with pytest.raises(kopt.KaoError, match="too large"):
        kopt.solve(red.pb, **OPTS)
    _, _, _, got, want = _solve_both(opb, None, fx, tight_bound=True)
    lp = kopt.solve(dataclasses.replace(pb, fixed=fx), tight_bound=True, lp_bound=True, **OPTS)
    assert np.array_equal(lp.replicas, got.replicas) and lp.key == got.key
    if want.feasible:
        bound = min(want.objective_bound, kopt.lp_bound(red.pb, want.replicas)[0])
        assert lp.objective_bound == bound + red.O0 and lp.optimal == (lp.objective == lp.objective_bound)
    with pytest.raises(kopt.KaoError, match="does not fit the shared memory"):
        kopt.solve(dataclasses.replace(pb, fixed=fx), row_major=True, **OPTS)


def _one_topic_cluster():
    """8,200 partitions in 205 topics of 40, round robin over 16 brokers in 4 racks; topic t007's partitions start
    perturbed, and only that topic is moved"""
    rng = np.random.RandomState(4)           # the flow bound is tight for this seed (checked with HiGHS)
    rows = [[(p + i) % 16 for i in range(3)] for p in range(8200)]
    for p in range(280, 320):
        rows[p] = [int(b) for b in rng.choice(16, size=3, replace=False)]
    topics = [("t%03d" % (p // 40), p % 40) for p in range(8200)]
    return kao.build_problem(rows, range(16), {b: "r%d" % (b % 4) for b in range(16)}, 3, topics,
                             topics_to_move=["t007"])


def test_a_moved_topic_reaches_the_restricted_optimum():
    pb = _one_topic_cluster()
    assert int((~pb.fixed).sum()) == 40
    opb = m.Problem(**{f.name: getattr(pb, f.name) for f in dataclasses.fields(m.Problem)})
    sol = F.solve_exact(opb, pb.fixed)
    assert sol.status == "optimal"
    res = kopt.solve(pb, seed=5, rounds=64, round_size=1 << 15, restarts=4, tight_bound=True, lp_bound=True)
    assert res.feasible and res.objective == sol.objective and res.optimal, (res.objective, sol.objective,
                                                                             res.objective_bound)


def test_fixed_load_above_the_bounds_is_infeasible():
    opb = SHAPES["cfg2"]()
    opb = dataclasses.replace(opb, rep_lo=np.zeros(opb.B, np.int32), rep_hi=np.full(opb.B, 5, np.int32))
    pb = kao.Problem.from_fields(opb)
    fx = _mask_of_share(pb, 4, 0.8)
    red = F.reduce(pb, fx)
    assert red.V0 > 0
    _, _, _, got, want = _solve_both(opb, None, fx)
    assert not got.feasible and got.violation == want.violation + red.V0
    with pytest.raises(kopt.KaoError, match="fixed partitions alone"):
        kopt.solve(dataclasses.replace(pb, fixed=fx), require_feasible=True, **OPTS)
