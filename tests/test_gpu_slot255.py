"""Clusters that use all 256 broker slots, on the GPU (problems.SLOT255_SHAPES: a cluster of 255 brokers grown by one,
the new broker on slot 255).  Slot 255 is then a real broker while several tables use the byte 0xFF for "none" or
"padding" (DESIGN.md 7.1).  Topic sessions whose rows bind on that broker, with and without per-partition rows, at and
above 8,160 partitions; plain sessions on the shared-memory row-major kernel, the delta search and the HBM path over
long walks; the initial base of every create call where a current leader sits on slot 255; and both objective bounds at
their widest multiplier vector (2 B + R = 544).  Keys and trajectories are compared bit for bit with the restatements
(oracle/kao_ref.c, tests/topics_ref, tests/rf_ref), evaluations with the model."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import lp_ref
import rf_ref
import topics_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import LEADER255_SHAPES, SLOT255_SHAPES, SLOT255_TOPIC_SHAPES, emptied_base, mixed_rows, moved_base
from test_gpu_large_layouts import WALK, assert_keys, one_loose_topic, walk_and_rebuild
from test_gpu_smem_walks import PROBE, check_base, open_runner, runners, search
from test_slot255_cpu import assert_model4

pytestmark = pytest.mark.gpu

BIG = 8160


def topic_case(name, rows):
    """(problem, topic rows, restatement, session factory) of a topic shape, with mixed per-partition rows or without"""
    pb = SLOT255_TOPIC_SHAPES[name]()
    kp = kao.Problem.from_fields(pb)
    if rows:
        kp.replication = mixed_rows(kp, 0x255)
    tr = kao.topic_rows(kp)
    r = rf_ref.RRef(kp, kp.replication, tr) if rows else topics_ref.TRef(pb, tr)
    evaluate = (lambda reps: rf_ref.evaluate(kp, kp.replication, reps, tr)) if rows else \
        (lambda reps: topics_ref.evaluate(pb, tr, reps))
    return kp, tr, r, evaluate, lambda: kao.Session(kp, topics=tr)


# ---- topic sessions whose rows bind on broker 255 ------------------------------------------------------------------
@pytest.mark.parametrize("rows", [False, True], ids=["topics", "topics_rf"])
@pytest.mark.parametrize("name", sorted(SLOT255_TOPIC_SHAPES))
def test_topic_sessions_count_the_broker_on_slot_255(name, rows):
    """get_base equals the model with topic rows from the initial, moved and emptied bases; delta keys of a free and a
    cycle round equal the restatement's; a long walk equals the restatement's, and a fresh session on the walked base
    scores the next rounds as the walked one does"""
    kp, tr, r, evaluate, open_session = topic_case(name, rows)
    big = kp.P > BIG
    size, rounds = (512, 12) if big else (1024, WALK)
    sess = open_session()
    bits, ld = r.init_base()
    reps = r.decode(bits, ld)
    if not rows:
        assert topics_ref._topic_counts(kp, tr, reps)[0][:, 255].sum() == 0 and (tr.rep_lo >= 1).all()
    assert (sess.get_base()[0] == reps).all()
    for what, b in (("initial", reps), ("moved", moved_base(kp, reps, 6)), ("emptied", emptied_base(kp, reps, 5))):
        sess.set_base(b)
        bits, ld = r.encode(b)
        got_reps, v, o, _ = sess.get_base()
        assert (got_reps == r.decode(bits, ld)).all(), what
        assert (v, o) == r.evaluate(bits, ld) == evaluate(got_reps), what
        for rnd in (4, 7):                                   # a free and a cycle round
            got = sess.candidate_keys_delta(0xB16, rnd, size, 0, size)
            assert_keys(got, r.candidate_keys(bits, ld, 0xB16, rnd, size, 0, size), (what, rnd))
    sess.close()
    bits, ld = r.encode(reps)
    sess = open_session()
    half = rounds // 2
    for first, n in ((0, half), (half, rounds - half)):
        _, want = r.search(bits, ld, 0x5EED, first, n, size)
        got, _ = sess.search_delta(0x5EED, first, n, size)
        assert_keys(got, want, ("walk round", first))
    end, v, o, _ = sess.get_base()
    assert (end == r.decode(bits, ld)).all() and (v, o) == evaluate(end)
    fresh = open_session()
    fresh.set_base(end)
    assert fresh.get_base()[1:3] == (v, o)
    for rnd in (rounds, rounds + 3):
        assert_keys(sess.candidate_keys_delta(0x5EED, rnd, size, 0, size),
                    fresh.candidate_keys_delta(0x5EED, rnd, size, 0, size), ("rebuilt", rnd))
    fresh.close()
    sess.close()


@pytest.mark.parametrize("name", ["one_topic_r16", "sized_r32"])
def test_topic_balance_reports_feasible_only_without_violated_topic_rows(name):
    pb = SLOT255_TOPIC_SHAPES[name]()
    kp = kao.Problem.from_fields(pb)
    tr = kao.topic_rows(kp)
    res = kopt.solve(kp, rounds=600, round_size=4096, patience=150, topic_balance=True)
    assert (res.violation, res.objective) == topics_ref.evaluate(pb, tr, res.replicas)
    if res.feasible:
        assert topics_ref.violated_rows(pb, tr, res.replicas) == 0 and m.evaluate(pb, res.replicas)[0] == 0
    else:
        assert topics_ref.violated_rows(pb, tr, res.replicas) + m.evaluate(pb, res.replicas)[0] > 0


# ---- plain sessions: the shared-memory kernels and the HBM path ----------------------------------------------------
@pytest.mark.parametrize("name", sorted(SLOT255_SHAPES))
def test_plain_walks_use_every_slot(ref_lib, name):
    """The long (48 x 1,024, two calls) and probe (400 x 4) walks of test_gpu_smem_walks.py on the row-major kernel and
    the delta search, and the long walk on the HBM path (a loose-topic session), from the initial, moved and emptied
    bases.  Above 8,160 partitions: the HBM path alone, keys of two rounds and a shorter walk."""
    pb = SLOT255_SHAPES[name]()
    r = ref_lib.Ref(pb)
    assert r.W == 8
    reps = r.decode(*r.init_base())
    starts = {"initial": reps, "moved": moved_base(pb, reps, 6), "emptied": emptied_base(pb, reps, 5)}
    if pb.P > BIG:
        sess = kao.Session(kao.Problem.from_fields(pb))
        for what, b in starts.items():
            sess.set_base(b)
            bits, ld = r.encode(b)
            assert sess.get_base()[1:3] == r.evaluate(bits, ld) == m.evaluate(pb, sess.get_base()[0]), what
            for rnd in (0, 3):
                got = sess.candidate_keys_delta(0xB16, rnd, 1024, 0, 1024)
                assert_keys(got, r.candidate_keys(bits, ld, 0xB16, rnd, 1024, 0, 1024), (what, rnd))
        sess.close()
        for what in ("initial", "emptied"):
            walk_and_rebuild(pb, r, starts[what], 0x77, 12, 512)[0].close()
        return
    run = runners(pb)
    assert run[0][0] == "row_major"
    for what, start in starts.items():
        seed = 0x5EED0 + len(what)
        bits, ld = r.encode(start)
        _, want_long = r.search(bits, ld, seed, 0, WALK, 1024)
        pbits, pld = r.encode(start)
        _, want_probe = r.search(pbits, pld, seed ^ 0x77, 0, PROBE, 4)
        for runner in run:
            tag = (what, runner[0])
            sess = open_runner(pb, runner)
            sess.set_base(start)
            got = np.concatenate([search(sess, runner, seed, 0, WALK // 2, 1024),
                                  search(sess, runner, seed, WALK // 2, WALK - WALK // 2, 1024)])
            assert_keys(got, want_long, tag + ("long walk",))
            check_base(sess, pb, r, bits, ld, tag + ("long walk",))
            sess.close()
            sess = open_runner(pb, runner)
            sess.set_base(start)
            assert_keys(search(sess, runner, seed ^ 0x77, 0, PROBE, 4), want_probe, tag + ("probe walk",))
            check_base(sess, pb, r, pbits, pld, tag + ("probe walk",))
            sess.close()
        sess, _ = walk_and_rebuild(pb, r, start, seed, WALK, 1024)
        sess.close()


# ---- the initial base where a current leader sits on slot 255 -------------------------------------------------------
@pytest.mark.parametrize("name", sorted(LEADER255_SHAPES))
def test_every_create_call_keeps_the_leader_on_slot_255(name):
    """get_base right after kao_create, kao_create_topics and kao_create_replication is MODEL §4's initial base"""
    pb = LEADER255_SHAPES[name]()
    kp = kao.Problem.from_fields(pb)
    rr = kp.RF * np.ones(kp.P, np.int32)
    for what, sess in (("kao_create", lambda: kao.Session(kp)),
                       ("kao_create_topics", lambda: kao.Session(kp, topics=one_loose_topic(pb)))):
        s = sess()
        assert_model4(pb, s.get_base()[0], what)
        s.close()
    kp.replication = kao.ReplicationRows(rr, np.full(kp.P, pb.ppr_lo, np.int32), np.full(kp.P, pb.ppr_hi, np.int32))
    s = kao.Session(kp)
    assert_model4(pb, s.get_base()[0], "kao_create_replication")
    s.close()


# ---- both bounds at the widest multiplier vector ----------------------------------------------------------------------
def test_bounds_at_544_multipliers():
    """B = 256 in 32 racks of 8: kao_lp_bound's 2 B + R = 544 multipliers, the most docs/MODEL.md §9 allows.  The kernel
    equals the restatement bit for bit after every k of KS, and both bounds are at least the search's objective."""
    from test_gpu_lp_bound import KS

    pb = SLOT255_SHAPES["s255_r32"]()
    assert 2 * pb.B + pb.R == 544
    kp = kao.Problem.from_fields(pb)
    res = kopt.solve(kp, rounds=800, round_size=4096, patience=200)
    assert res.feasible and m.evaluate(pb, res.replicas) == (0, res.objective)
    for k in KS:
        bound, its, u = kopt.lp_bound(kp, res.replicas, max_iterations=k, multipliers=True)
        want = lp_ref.lp_bound(pb, res.objective, k)
        assert (bound, its) == want[:2] and (u == want[2]).all(), k
        assert bound >= res.objective, k
    assert kopt.objective_bound(kp) >= res.objective and kopt.objective_bound(kp, res.replicas) >= res.objective
