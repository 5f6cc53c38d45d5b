"""Replication factors 5 to 8 and RF = B - 1 on the GPU (problems.RF_SHAPES): the shared-memory kernels built for sm_90a
(row-major, both column-major schedules, the delta search) and the HBM-base kernels, held bit for bit to the
restatement (oracle/kao_ref.c, tests/rf_ref, tests/topics_ref) and the exact model from the initial base, damaged bases
(RF 7 and RF 8 rows short by up to RF), a base whose every row leads from another replica and a base of well-formed
rows; kao_solve_fixed at RF 8 above 8,160 partitions against the reduced solve; and kao_solve with both bounds on
instances HiGHS solves.  tests/test_rf_edges_cpu.py runs the same device code on the CPU and says what each shape is
for."""
import dataclasses

import numpy as np
import pytest

import fixed_ref as F
import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import optimizer as kopt
from kafka_assignment_optimizer_b200 import tuning
from oracle import model as m
from problems import RF_EXACT_SHAPES, RF_SHAPES
from test_gpu_fixed import _solve_both
from test_gpu_home255 import all_runners, check_end
from test_gpu_large_layouts import assert_keys, empty_rows, walk_and_rebuild
from test_gpu_smem_walks import check_base, open_runner, runners, search
from test_rf_edges_cpu import bases

pytestmark = pytest.mark.gpu

SMALL = sorted(n for n in RF_SHAPES if not n.startswith("big_"))
BIG = ["big_rf8", "big_rf8_b9"]
SIZE = 1024                         # candidates of a key round on the shared-memory kernels; the last is the identity
WALK, PROBE = 24, 200               # rounds of the long walk (two calls) and of the probe walk (rounds of 4)


def keys(sess, runner, seed, rnd, size):
    return (sess.candidate_keys_delta if runner[3] else sess.candidate_keys)(seed, rnd, size, 0, size)


@pytest.mark.parametrize("name", SMALL)
def test_keys_on_every_runner_from_every_base(ref_lib, name):
    """A free and a cycle round on the row-major evaluator, each column-major schedule the layout takes (the popcount
    schedule (4, 0x22, 1024) and the tensor-core default (1, 0x300, 512)) and the delta keys; get_base after set_base
    is the restatement's base and scores as the model does"""
    pb = RF_SHAPES[name]()
    r = ref_lib.Ref(pb)
    run = runners(pb)
    assert [x[0] for x in run][0] == "row_major" and run[-1][0] == "delta"
    assert len(run) == (4 if any(x[1] for x in run) else 2)
    for runner in run:
        sess = open_runner(pb, runner)
        for what, b in bases(pb, r).items():
            sess.set_base(b)
            bits, ld = r.encode(b)
            check_base(sess, pb, r, bits, ld, (runner[0], what))
            for rnd in (4, 7):
                assert_keys(keys(sess, runner, 0x7F8, rnd, SIZE), r.candidate_keys(bits, ld, 0x7F8, rnd, SIZE, 0, SIZE),
                            (runner[0], what, rnd))
        sess.close()


@pytest.mark.parametrize("name", SMALL)
def test_walks_on_every_runner_from_every_base(ref_lib, name):
    """24 rounds of 1,024 in two calls (the second restages the base, lists and planes from HBM) and 200 rounds of 4 on
    every runner; the walked base is the restatement's and scores as the model does"""
    pb = RF_SHAPES[name]()
    r = ref_lib.Ref(pb)
    run = runners(pb)
    for what, start in bases(pb, r).items():
        seed = 0x5EED0 + len(what)
        bits, ld = r.encode(start)
        _, want_long = r.search(bits, ld, seed, 0, WALK, SIZE)
        pbits, pld = r.encode(start)
        _, want_probe = r.search(pbits, pld, seed ^ 0x77, 0, PROBE, 4)
        for runner in run:
            tag = (what, runner[0])
            sess = open_runner(pb, runner)
            sess.set_base(start)
            got = np.concatenate([search(sess, runner, seed, 0, WALK // 2, SIZE),
                                  search(sess, runner, seed, WALK // 2, WALK - WALK // 2, SIZE)])
            assert_keys(got, want_long, tag + ("long walk",))
            check_base(sess, pb, r, bits, ld, tag + ("long walk",))
            sess.close()
            sess = open_runner(pb, runner)
            sess.set_base(start)
            assert_keys(search(sess, runner, seed ^ 0x77, 0, PROBE, 4), want_probe, tag + ("probe walk",))
            check_base(sess, pb, r, pbits, pld, tag + ("probe walk",))
            sess.close()


def test_the_engine_picks_the_evaluator_the_plane_count_allows():
    """kao_get_evaluator: eight term planes (RFcur 7) and RF 8 in eight racks run column-major on the tensor-core
    default; nine (RFcur 8) are beyond the column-major evaluator, so the session runs row-major and refuses it"""
    for name, cm in (("rf7_cm", True), ("rf7_cur7", True), ("rf8_cm", True), ("rf2_b3_r3", True), ("rf7_cur8", False)):
        sess = kao.Session(kao.Problem.from_fields(RF_SHAPES[name]()))
        st = sess.stats()
        assert st["column_major"] == cm, name
        if cm:
            assert st["schedule"] == tuning.DEFAULT_SCHEDULE, name
        else:
            assert not sess.set_evaluator(True) and not sess.stats()["column_major"], name
        sess.close()


# ---- above 8,160 partitions: the HBM path -----------------------------------------------------------------------------
@pytest.mark.parametrize("name", BIG)
def test_hbm_keys_and_walks(ref_lib, name):
    """Delta keys of a free and a cycle round from the initial and the damaged bases, and 12 rounds of 512 from the
    initial and the emptied base, then a fresh session on the walked base scores as the walked one"""
    pb = RF_SHAPES[name]()
    r = ref_lib.Ref(pb)
    reps = r.decode(*r.init_base())
    damaged = bases(pb, r)
    sess = kao.Session(kao.Problem.from_fields(pb))
    assert sess.stats()["words_per_row"] == r.W
    for what in ("initial", "moved", "emptied", "reordered"):
        sess.set_base(damaged[what])
        bits, ld = r.encode(damaged[what])
        assert sess.get_base()[1:3] == r.evaluate(bits, ld) == m.evaluate(pb, r.decode(bits, ld)), what
        for rnd in (4, 7):
            assert_keys(sess.candidate_keys_delta(0xB16, rnd, 1024, 0, 1024),
                        r.candidate_keys(bits, ld, 0xB16, rnd, 1024, 0, 1024), (what, rnd))
    sess.close()
    for what in ("initial", "emptied"):
        walked, end = walk_and_rebuild(pb, r, damaged[what], 0x77, 12, 512)
        if what == "emptied":
            assert empty_rows(end) > 0
        walked.close()


@pytest.mark.parametrize("kind", ["replication", "topics"])
@pytest.mark.parametrize("name", BIG)
def test_hbm_replication_and_topic_sessions(ref_lib, name, kind):
    """rf[p] over 1..min(8, B - 1) with mixed C7 forms (tests/rf_ref), and five interleaved topics (tests/topics_ref):
    keys of a free and a cycle round and 12 rounds of 512 in two calls from the initial base"""
    pb = RF_SHAPES[name]()
    run = all_runners(pb, ref_lib)[kind]
    r = run.r
    start = r.decode(*r.init_base())
    sess = run.open()
    sess.set_base(start)
    bits, ld = r.encode(start)
    check_end(sess, run, bits, ld, (kind, "initial"))
    for rnd in (4, 7):
        assert_keys(run.keys(sess, 0xB16, rnd, 1024, 0, 1024), r.candidate_keys(bits, ld, 0xB16, rnd, 1024, 0, 1024),
                    (kind, rnd))
    for first, n in ((0, 6), (6, 6)):
        _, want = r.search(bits, ld, 0x77, first, n, 512)
        assert_keys(run.search(sess, 0x77, first, n, 512), want, (kind, first))
    check_end(sess, run, bits, ld, (kind, "walked"))
    sess.close()


@pytest.mark.parametrize("name", BIG)
def test_solve_fixed_is_the_reduced_solve(name):
    """Half the partitions fixed: the searched rows, key and rounds are the reduced problem's solve, the fixed rows
    are cur's"""
    opb = RF_SHAPES[name]()
    fx = F.random_mask(kao.Problem.from_fields(opb), 0x8F, share=0.5)
    assert fx.any() and not fx.all()
    pb, _, red, got, want = _solve_both(opb, None, fx)
    assert red.pb.RF == 8 and red.pb.P < pb.P
    assert np.array_equal(got.replicas[red.searched], want.replicas)
    assert (got.key, got.rounds, got.moves) == (want.key, want.rounds, want.moves)
    assert got.violation == want.violation + red.V0 and got.objective == want.objective + red.O0
    for p in np.flatnonzero(fx):
        row = [int(b) for b in pb.cur[p] if b >= 0]
        assert [int(b) for b in got.replicas[p] if b >= 0] == row, p


# ---- kao_solve against HiGHS ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(RF_EXACT_SHAPES))
def test_solve_reaches_the_optimum_and_its_bounds_hold(name):
    """kao_solve with the flow bound and the Lagrangian LP bound: the HiGHS optimum, a bound never below it, and
    "optimal" only where the bound meets the objective"""
    opb = RF_EXACT_SHAPES[name]()
    sol = m.solve_exact(opb)
    assert sol.status == "optimal"
    res = kopt.solve(kao.Problem.from_fields(opb), rounds=300, round_size=4096, tight_bound=True, lp_bound=True)
    assert (res.violation, res.objective) == (0, sol.objective) == m.evaluate(opb, res.replicas)
    assert res.objective_bound >= sol.objective
    assert res.optimal == (res.objective == res.objective_bound)
    lp, _ = kopt.lp_bound(kao.Problem.from_fields(opb), res.replicas)
    assert lp >= sol.objective
