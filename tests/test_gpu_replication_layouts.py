"""Replication sessions (kao_create_replication, docs/MODEL.md §11) on every layout of the HBM-base search path, from
damaged and saturated bases, over long trajectories and at its count limits: test_gpu_large_layouts.py with
per-partition rows whose C7 forms differ from row to row (problems.mixed_rows).  Keys and trajectories are compared bit
for bit with the restatement (tests/rf_ref), evaluations with the model; after a long walk, a fresh session built from
the walked base must score every candidate as the walked session does."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import rf_ref
from oracle import model as m
from problems import (C7_SHAPES, LARGE_SHAPES, LAYOUT_SHAPES, SHAPES, emptied_base, mixed_rows, moved_base,
                      off_rf_base)
from test_gpu_large_layouts import WALK, assert_keys, check_delta_keys, concentrated, empty_rows, malformed

pytestmark = pytest.mark.gpu

SMALL = {**SHAPES, **LAYOUT_SHAPES, **C7_SHAPES}
ROUND = {"max_rows": 1024, "w2_rows6000": 1024}      # the restatement scores every candidate in O(P)
TOPIC_SHAPES = ["cfg2", "rack3_w4", "rack4_w8", "c7_w2_s8_lo", "s64_r1", "ragged"]


def with_rows(pb, seed=0x7F, topics=False):
    """(problem with mixed per-partition rows, its topic rows or None, the restatement)"""
    kp = kao.Problem.from_fields(pb)
    kp.replication = mixed_rows(kp, seed)
    tr = None
    if topics:
        kp.topics = [("t%d" % (p % 5), p) for p in range(kp.P)]
        tr = kao.topic_rows(kp)
    return kp, tr, rf_ref.RRef(kp, kp.replication, tr)


def model(kp, tr, reps):
    return rf_ref.evaluate(kp, kp.replication, reps, tr)


# ---- every small layout ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SMALL))
def test_replication_keys_and_evaluations_from_every_base(name):
    """Delta keys equal the restatement's from the initial, a random, an off-rf, an emptied and a moved base; get_base
    after set_base equals the model on random, short-row, duplicate-broker and emptied assignments."""
    pb = SMALL[name]()
    kp, tr, r = with_rows(pb)
    sess = kao.Session(kp)
    assert sess.stats()["words_per_row"] == r.W
    size = ROUND.get(name, 4096)
    rng = np.random.RandomState(7)
    bits, ld = r.init_base()
    reps = r.decode(bits, ld)
    got = sess.get_base()
    assert (got[0] == reps).all() and got[1:3] == r.evaluate(bits, ld) == model(kp, tr, reps)
    bases = {"initial": reps, "random": malformed(kp, reps, rng)["random"], "off_rf": off_rf_base(kp, reps, 6),
             "emptied": emptied_base(kp, reps, 5), "moved": moved_base(kp, reps, 6)}
    assert empty_rows(bases["emptied"]) > 0 and empty_rows(bases["moved"]) == 0
    for what, b in bases.items():
        sess.set_base(b)
        bits, ld = r.encode(b)
        got_reps, v, o, _ = sess.get_base()
        assert (got_reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == model(kp, tr, got_reps)
        check_delta_keys(sess, r, bits, ld, size, what)
    for what, b in malformed(kp, reps, rng).items():
        sess.set_base(b)
        assert sess.get_base()[1:3] == model(kp, tr, b), what
    sess.close()


def walk_and_rebuild(kp, tr, r, start, seed, rounds, size, keys_size=4096):
    """search_delta from `start` over `rounds` rounds in two calls against the restatement; then a fresh replication
    session on the walked base scores the next free and cycle rounds as the walked one does.  -> the walked session"""
    bits, ld = r.encode(start)
    sess = kao.Session(kp, topics=tr)
    sess.set_base(start)
    half = rounds // 2
    for first, n in ((0, half), (half, rounds - half)):
        _, want = r.search(bits, ld, seed, first, n, size)
        got, _ = sess.search_delta(seed, first, n, size)
        assert_keys(got, want, ("round", first))
    reps, v, o, _ = sess.get_base()
    assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == model(kp, tr, reps)
    fresh = kao.Session(kp, topics=tr)
    fresh.set_base(reps)
    for rnd in (rounds, rounds + 3):
        assert_keys(sess.candidate_keys_delta(seed, rnd, keys_size, 0, keys_size),
                    fresh.candidate_keys_delta(seed, rnd, keys_size, 0, keys_size), ("rebuilt", rnd))
    fresh.close()
    return sess, reps


@pytest.mark.parametrize("name", sorted(SMALL) + ["%s+topics" % n for n in TOPIC_SHAPES])
def test_replication_long_walks_from_every_base(name):
    """48 rounds from the initial, an emptied and a moved base, without and (on a subset) with topic rows"""
    base_name = name.split("+")[0]
    pb = SMALL[base_name]()
    kp, tr, r = with_rows(pb, topics=name.endswith("+topics"))
    size = 256 if base_name in ROUND else 1024
    reps = r.decode(*r.init_base())
    for what, start in (("initial", reps), ("emptied", emptied_base(kp, reps, 5)), ("moved", moved_base(kp, reps, 6))):
        sess, end = walk_and_rebuild(kp, tr, r, start, 0x5EED + len(what), WALK, size)
        if what == "emptied":
            assert empty_rows(end) == empty_rows(start) > 0
        sess.close()


def uniform(kp):
    return kao.ReplicationRows(np.full(kp.P, kp.RF, np.int32), np.full(kp.P, kp.ppr_lo, np.int32),
                               np.full(kp.P, kp.ppr_hi, np.int32))


@pytest.mark.parametrize("name", ["cfg2", "ragged", "rf_up", "rack5_w4", "dense_rack4_w2", "sat_cfg2"])
def test_replication_patience(name):
    """Uniform rows: patience stops on the round a plain shared-memory session stops on, with its keys.  Mixed rows:
    the keys up to the stop equal the restatement's."""
    pb = SMALL[name]()
    kp = kao.Problem.from_fields(pb)
    got = {}
    for rows in (None, uniform(kp)):
        kp.replication = rows
        sess = kao.Session(kp)
        sess.set_patience(2)
        keys, _ = sess.search_delta(0x5A7, 0, 300, 512)
        got[len(got)] = (sess.last_rounds(), keys[:sess.last_rounds()])
        sess.close()
    (n0, k0), (n1, k1) = got[0], got[1]
    assert 0 < n0 < 300 and n0 == n1 and (k0 == k1).all()
    kp, tr, r = with_rows(pb)
    sess = kao.Session(kp)
    sess.set_patience(2)
    keys, _ = sess.search_delta(0x5A7, 0, 300, 512)
    n = sess.last_rounds()
    assert 0 < n <= 300
    assert_keys(keys[:n], r.search(*r.init_base(), 0x5A7, 0, n, 512)[1], "patience")
    sess.close()


# ---- a violation field saturated by C7 rows -------------------------------------------------------------------------
SAT_EXCESS = 10      # round 0's winner (about 7 better than the base) stays saturated, round 1's does not


def c7_saturated(excess=SAT_EXCESS):
    """LARGE_SHAPES["big_obj24"] (key_obj_bits 24: a violation cap of 32,767) with per-partition rows at RF and the
    problem's C7, then rows raised to lo = hi = 63, and the last ones to lo = L (hi 127), until the initial base
    violates the rows by the cap + excess"""
    kp = kao.Problem.from_fields(LARGE_SHAPES["big_obj24"]())
    rf = np.full(kp.P, kp.RF, np.int32)
    lo, hi = np.full(kp.P, kp.ppr_lo, np.int32), np.full(kp.P, kp.ppr_hi, np.int32)
    r = rf_ref.RRef(kp, kao.ReplicationRows(rf, lo, hi))
    reps = r.decode(*r.init_base())
    cap = (1 << (39 - r.obj_bits)) - 1
    need = cap + excess - r.evaluate(*r.init_base())[0]
    term = lambda p, a, b: rf_ref._row_terms(kp, reps, p, int(rf[p]), a, b)
    for p in range(0, kp.P, 13):
        if need == 0:
            break
        old = term(p, int(lo[p]), int(hi[p]))
        for a, b in [(63, 63)] + [(L, 127) for L in range(63, 0, -1)]:
            if 0 <= term(p, a, b) - old <= need:
                need -= term(p, a, b) - old
                lo[p], hi[p] = a, b
                break
    assert need == 0
    kp.replication = kao.ReplicationRows(rf, lo, hi)
    r = rf_ref.RRef(kp, kp.replication)
    bits, ld = r.init_base()
    assert (r.decode(bits, ld) == reps).all() and r.evaluate(bits, ld)[0] == cap + excess
    assert (lo == 63).sum() > 100
    return kp, r, cap


def test_replication_search_leaves_a_c7_saturated_base_like_the_restatement():
    """Round 0's winner is a saturated key: the search kernel re-evaluates its base with every row's own C1 / C7
    (block_eval<W, true>) before round 1.  The trajectory, the final base and the round patience stops at equal the
    restatement's."""
    kp, r, cap = c7_saturated()
    bits, ld = r.init_base()
    _, want = r.search(bits, ld, 0x5A7, 0, 10, 1024)
    viols = [r.unpack_key(k)[0] for k in want]
    assert viols[0] == cap and min(viols[1:]) < cap, viols
    sess = kao.Session(kp)
    assert sess.get_base()[1] == cap + SAT_EXCESS
    got, _ = sess.search_delta(0x5A7, 0, 10, 1024)
    assert_keys(got, want, "saturated walk")
    reps, v, o, _ = sess.get_base()
    assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == model(kp, None, reps)
    sess.close()
    # rounds of 8 candidates: saturated winners round after round, each base re-evaluated in full, until patience
    sess = kao.Session(kp)
    sess.set_patience(2)
    got, _ = sess.search_delta(0x5A7, 0, 100, 8)
    n = sess.last_rounds()
    assert 0 < n < 100
    assert_keys(got[:n], r.search(*r.init_base(), 0x5A7, 0, n, 8)[1], "patience")
    assert r.unpack_key(got[1])[0] == cap
    sess.close()


# ---- above 8,160 partitions ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(LARGE_SHAPES) + ["big_rf_up+topics", "big_ppr11_w8+topics"])
def test_large_replication_keys_and_trajectories(name):
    base_name = name.split("+")[0]
    kp, tr, r = with_rows(LARGE_SHAPES[base_name](), topics=name.endswith("+topics"))
    reps = r.decode(*r.init_base())
    sess = kao.Session(kp, topics=tr)
    assert sess.stats()["words_per_row"] == r.W
    for what, b in (("initial", reps), ("moved", moved_base(kp, reps, 6)), ("emptied", emptied_base(kp, reps, 5))):
        sess.set_base(b)
        bits, ld = r.encode(b)
        assert sess.get_base()[1:3] == r.evaluate(bits, ld)
        for rnd in (0, 3):
            got = sess.candidate_keys_delta(0xB16, rnd, 1024, 0, 1024)
            assert_keys(got, r.candidate_keys(bits, ld, 0xB16, rnd, 1024, 0, 1024), (what, rnd))
    sess.close()
    for what, start in (("initial", reps), ("emptied", emptied_base(kp, reps, 5))):
        walk_and_rebuild(kp, tr, r, start, 0x77, 12, 512)[0].close()


# ---- count limits at 65,280 partitions ----------------------------------------------------------------------------
def test_concentrated_bases_at_65280_with_mixed_rf():
    kp, tr, r = with_rows(m.synthetic_problem(65280, 16, 4, 2, remove=1))
    assert set(kp.replication.rf.tolist()) == {1, 2}
    sess = kao.Session(kp)
    for what, reps in concentrated(kp.P, kp.B).items():
        sess.set_base(reps)
        bits, ld = r.encode(reps)
        assert sess.get_base()[1:3] == r.evaluate(bits, ld) == model(kp, None, reps), what
        for rnd in (0, 3):
            got = sess.candidate_keys_delta(0x8160, rnd, 4096, 0, 256)
            assert_keys(got, r.candidate_keys(bits, ld, 0x8160, rnd, 4096, 0, 256), (what, rnd))
    sess.close()


@pytest.mark.parametrize("topics", [False, True])
def test_long_replication_run_at_65280_equals_a_rebuilt_session(topics):
    """300 rounds of 4,096 candidates with mixed rows; then a fresh session on the walked base scores the next rounds
    as the walked one does, and get_base equals the model"""
    pb = m.synthetic_problem(65280, 64, 8, 3, remove=1)
    kp = kao.Problem.from_fields(pb)
    kp.replication = mixed_rows(kp, 0x7F)
    tr = None
    if topics:
        kp.topics = [("t%d" % (p // 50), p) for p in range(kp.P)]
        tr = kao.topic_rows(kp)
    sess = kao.Session(kp, topics=tr)
    sess.search_delta(0x5EED, 0, 150, 4096)
    sess.search_delta(0x5EED, 150, 150, 4096)
    reps, v, o, _ = sess.get_base()
    assert (v, o) == model(kp, tr, reps)
    fresh = kao.Session(kp, topics=tr)
    fresh.set_base(reps)
    assert fresh.get_base()[1:3] == (v, o)
    for rnd in (300, 303):
        assert_keys(sess.candidate_keys_delta(0x5EED, rnd, 4096, 0, 4096),
                    fresh.candidate_keys_delta(0x5EED, rnd, 4096, 0, 4096), ("rebuilt", rnd))
    sess.close()
    fresh.close()
