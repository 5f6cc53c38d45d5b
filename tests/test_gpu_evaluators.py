"""GPU parity of BOTH full evaluators on the layouts the column-major one covers (kao_set_evaluator,
csrc/kao_device_t.cuh): the column-major evaluator is the engine's default there, so the other GPU tests
exercise it; here each test runs the column-major and the row-major evaluator explicitly and holds both
to the restatement and the golden streams — same keys, trajectories and winners."""
import json
import os

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import SHAPES

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
SUPPORTED = ["cfg2", "cfg2_rm2", "cfg3_small", "rf1", "rf_down"]


def product(pb):
    return kao.Problem.from_fields(pb)


@pytest.fixture(scope="module")
def golden_streams():
    with open(os.path.join(GOLDEN, "streams.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("column_major", [True, False])
@pytest.mark.parametrize("name", SUPPORTED)
def test_golden_streams_both_evaluators(golden_streams, name, column_major):
    g = golden_streams[name]
    sess = kao.Session(product(SHAPES[name]()))
    assert sess.set_evaluator(column_major)
    assert [int(k) for k in sess.candidate_keys(0xC0FFEE, 2, 1024, 0, 192)] == g["keys_round2"]
    assert [int(k) for k in sess.candidate_keys(0xC0FFEE, 3, 1024, 0, 192)] == g["keys_round3"]      # a cycle round
    assert int(sess.candidate_keys(0xC0FFEE, 2, 1024, 1023, 1)[0]) == g["identity_key"]
    keys, _ = sess.search(0xC0FFEE, 0, 8, 512)
    assert [int(k) for k in keys] == g["trajectory"]
    assert sess.get_base()[0].tolist() == g["final_base"]
    sess.close()


@pytest.mark.parametrize("column_major", [True, False])
@pytest.mark.parametrize("name", ["cfg2_rm2", "cfg3_small", "rf_down"])
def test_keys_and_trajectory_vs_restatement_both_evaluators(ref_lib, name, column_major):
    pb = SHAPES[name]()
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    sess = kao.Session(product(pb))
    assert sess.set_evaluator(column_major)
    for rnd, size, lo, n in [(0, 1024, 0, 1024), (5, 4096, 4096 - 700, 700), (9, 2, 0, 2)]:
        want = r.candidate_keys(bits, ld, 0xC0FFEE, rnd, size, lo, n)
        got = sess.candidate_keys(0xC0FFEE, rnd, size, lo, n)
        assert (want == got).all()
    _, want = r.search(bits, ld, 0xABCDEF12345, 3, 12, 1500)
    got, _ = sess.search(0xABCDEF12345, 3, 12, 1500)
    assert (want == got).all()
    reps, v, o, moves = sess.get_base()
    assert (reps == r.decode(bits, ld)).all()
    assert (v, o) == m.evaluate(pb, reps) and moves == m.replica_moves(pb, reps)
    sess.close()


@pytest.mark.parametrize("shape", [(3800, 32, 4, 3, 1), (2000, 64, 8, 3, 0), (1100, 64, 8, 3, 2), (8160, 16, 4, 2, 1)])
def test_large_shapes_column_major(ref_lib, shape):
    """120 / 64 / 40 / 256 partition words per slot: several words per lane in the row pass, rotated rows that wrap,
    64 chunks per column (the largest row count the engine accepts)."""
    P, B, R, RF, rm = shape
    pb = m.synthetic_problem(P, B, R, RF, remove=rm)
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    sess = kao.Session(product(pb))
    assert sess.set_evaluator(True)
    want = r.candidate_keys(bits, ld, 0xC0FFEE, 1, 2048, 0, 768)
    assert (want == sess.candidate_keys(0xC0FFEE, 1, 2048, 0, 768)).all()
    _, want = r.search(bits, ld, 0xABCDEF12345, 0, 3, 1024)
    got, _ = sess.search(0xABCDEF12345, 0, 3, 1024)
    assert (want == got).all()
    assert (sess.get_base()[0] == r.decode(bits, ld)).all()
    sess.close()


def test_malformed_base_column_major(ref_lib):
    """Short rows, duplicate brokers, random placement: every violation term is non-zero."""
    pb = SHAPES["cfg3_small"]()
    r = ref_lib.Ref(pb)
    sess = kao.Session(product(pb))
    assert sess.set_evaluator(True)
    rng = np.random.RandomState(3)
    for it in range(3):
        reps = np.stack([rng.choice(pb.B, size=pb.RF, replace=False) for _ in range(pb.P)]).astype(np.int32)
        if it == 1:
            for _ in range(5):
                reps[rng.randint(pb.P), -1] = -1
        if it == 2:
            for _ in range(5):
                p = rng.randint(pb.P)
                reps[p, 1] = reps[p, 0]
        sess.set_base(reps)
        bits, ld = r.encode(reps)
        want = r.candidate_keys(bits, ld, 11 + it, it, 2048, 0, 2048)
        assert (want == sess.candidate_keys(11 + it, it, 2048, 0, 2048)).all()
    sess.close()


def test_config3_same_winner_both_evaluators():
    """Headline shape: the two full evaluators walk the same trajectory and reach the same assignment."""
    pb = m.synthetic_problem(1000, 64, 8, 3)
    a = kao.Session(product(pb))
    b = kao.Session(product(pb))
    assert a.set_evaluator(False) and b.set_evaluator(True)
    ka, _ = a.search(0x5EED, 0, 6, 65536)
    kb, _ = b.search(0x5EED, 0, 6, 65536)
    assert (ka == kb).all()
    assert (a.get_base()[0] == b.get_base()[0]).all() and a.get_base()[1:3] == b.get_base()[1:3]
    a.close()
    b.close()
    r1 = kopt.solve(product(pb), seed=3, rounds=6, round_size=8192)
    r2 = kopt.solve(product(pb), seed=3, rounds=6, round_size=8192, row_major=True)
    assert (r1.replicas == r2.replicas).all() and (r1.violation, r1.objective, r1.key) == (r2.violation, r2.objective, r2.key)


def test_wide_open_rack_bounds_both_evaluators(ref_lib):
    """C6 bounds are plain int32 of the caller ("no upper bound" as 10^6, a lower bound no rack can reach): both
    full evaluators charge them exactly as the restatement does."""
    import dataclasses

    base = SHAPES["cfg2_rm2"]()
    for lo, hi in [(0, 1_000_000), (70_000, 1_000_000), (3, 5)]:
        pb = dataclasses.replace(base, rack_lo=np.full(base.R, lo, np.int32), rack_hi=np.full(base.R, hi, np.int32))
        r = ref_lib.Ref(pb)
        bits, ld = r.init_base()
        want = r.candidate_keys(bits, ld, 5, 1, 2048, 0, 512)
        for column_major in (True, False):
            sess = kao.Session(product(pb))
            assert sess.set_evaluator(column_major)
            assert (want == sess.candidate_keys(5, 1, 2048, 0, 512)).all(), (lo, hi, column_major)
            sess.close()


def test_unsupported_layouts_are_refused():
    for name in ["readme", "w8_s16", "dense_small", "w2_rows6000"]:   # w2_rows6000: the planes do not fit in shared memory
        sess = kao.Session(product(SHAPES[name]()))
        assert not sess.set_evaluator(True)
        sess.close()


def test_every_schedule_gives_the_same_keys():
    """kao_set_schedule: tensor cores or popcount streams, column loop, threads per CTA — same results,
    on the headline shape (32 partition words, compile-time offsets) and on a small one-word shape."""
    from kafka_assignment_optimizer_b200 import tuning

    for pb, n, size in [(m.synthetic_problem(1000, 64, 8, 3), 8192, 16384), (SHAPES["cfg2"](), 2048, 4096)]:
        base = kao.Session(product(pb))
        assert base.set_evaluator(False)
        want_keys = base.candidate_keys(0x5EED, 1, n, 0, n)
        want_traj, _ = base.search(0x5EED, 0, 4, size)
        want_base = base.get_base()[0]
        base.close()
        for sched in tuning.SCHEDULES:                   # (sync, pop, threads)
            sess = kao.Session(product(pb))
            assert sess.set_evaluator(True) and sess.set_schedule(*sched), sched
            assert (want_keys == sess.candidate_keys(0x5EED, 1, n, 0, n)).all(), sched
            got, _ = sess.search(0x5EED, 0, 4, size)
            assert (want_traj == got).all() and (want_base == sess.get_base()[0]).all(), sched
            sess.close()
    sess = kao.Session(product(SHAPES["cfg2"]()))
    assert not sess.set_schedule(1, 0x12345, 768) and not sess.set_schedule(2, 0x11111, 768)   # only what is built
    for retired in [(1, 0x1300, 512), (1, 0x200, 512), (1, 0x100, 512), (4, 0x22, 896)]:        # superseded, no longer built
        assert not sess.set_schedule(*retired), retired
    sess.close()


def test_column_major_is_the_default_where_it_applies():
    """VERDICT r1 #2: a plain session / kao_solve runs the fast evaluator without flags or environment."""
    pb = product(m.synthetic_problem(1000, 64, 8, 3))
    a, b = kao.Session(pb), kao.Session(pb)
    assert a.stats()["column_major"] and b.set_evaluator(True)
    rounds, size = 16, 1 << 17
    a.search(1, 0, rounds, size)
    _, ms_default = a.search(1, 100, rounds, size)
    b.search(1, 0, rounds, size)
    _, ms_col = b.search(1, 100, rounds, size)
    assert a.set_evaluator(False) and not a.stats()["column_major"]
    a.search(1, 200, rounds, size)
    _, ms_row = a.search(1, 300, rounds, size)
    a.close()
    b.close()
    assert abs(ms_default - ms_col) < 0.1 * ms_col and ms_row > 1.1 * ms_default, (ms_default, ms_col, ms_row)
    assert not kao.Session(product(SHAPES["w8_s16"]())).stats()["column_major"]          # other layouts: row-major
