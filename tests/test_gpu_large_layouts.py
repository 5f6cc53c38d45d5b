"""The HBM-base search path (kao_large.cu, DESIGN.md 7.1/7.2) on every layout, from damaged and saturated bases, over
long trajectories and at its count limits.  Below 8,161 partitions a topic session with one topic whose rows no
assignment can violate runs the same kernels with the same keys as the plain search.  Keys and trajectories are
compared bit for bit with the restatement (oracle/kao_ref.c, tests/topics_ref), evaluations with the model; after a
long walk, a fresh session built from the walked base must score every candidate as the walked session does, which
checks the patched lists, planes and counts without the restatement."""
import ctypes as C

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import topics_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import C7_SHAPES, LARGE_SHAPES, LAYOUT_SHAPES, SHAPES, emptied_base, moved_base
from conftest import make_problem

pytestmark = pytest.mark.gpu

SMALL = {**SHAPES, **LAYOUT_SHAPES, **C7_SHAPES}
ROUND = {"max_rows": 1024, "w2_rows6000": 1024}      # the restatement scores every candidate in O(P)
WALK = 48                                           # rounds of a long walk, in two calls


def sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def one_loose_topic(pb):
    """One topic over every partition with rows no assignment violates"""
    return kao.TopicRows(np.zeros(pb.P, np.int32), [0], [pb.P * pb.RF], [0], [pb.P], ["all"])


def hbm_session(pb):
    """A session on the HBM kernels at any P: above 8,160 partitions a plain one, else one with a loose topic"""
    if pb.P > 8160:
        return kao.Session(kao.Problem.from_fields(pb))
    return kao.Session(kao.Problem.from_fields(pb), topics=one_loose_topic(pb))


def assert_keys(got, want, what):
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (what, int(bad[0]), int(got[bad[0]]), int(want[bad[0]]))


def malformed(pb, reps, rng):
    """random rows; the same with a short row, with a duplicate broker, with rows emptied"""
    rand = np.stack([rng.choice(pb.B, size=pb.RF, replace=False) for _ in range(pb.P)]).astype(np.int32)
    short, dup, empty = rand.copy(), rand.copy(), rand.copy()
    short[rng.randint(pb.P), -1] = -1
    if pb.RF > 1:
        p = rng.randint(pb.P)
        dup[p, 1] = dup[p, 0]
    empty[rng.choice(pb.P, size=max(1, pb.P // 50), replace=False)] = -1
    return {"random": rand, "short": short, "duplicate": dup, "emptied": empty}


def check_delta_keys(sess, r, bits, ld, size, what, n_two=None):
    """free and cycle round: the smallest round, a full one, a sub-range, one candidate more than a thread each"""
    n_two = n_two or sms() * 512 + 1
    for rnd in (4, 7):
        for rs, lo, n in ((2, 0, 2), (size, 0, size), (size, size // 4, size // 3)):
            got = sess.candidate_keys_delta(0xB16, rnd, rs, lo, n)
            assert_keys(got, r.candidate_keys(bits, ld, 0xB16, rnd, rs, lo, n), (what, rnd, rs, lo))
        got = sess.candidate_keys_delta(0xB16, rnd, n_two, 0, n_two)
        for lo in (0, n_two - 256):          # the last candidate is some thread's second one
            assert_keys(got[lo:lo + 256], r.candidate_keys(bits, ld, 0xB16, rnd, n_two, lo, 256), (what, rnd, "two", lo))


def empty_rows(reps):
    return int((reps < 0).all(1).sum())


# ---- every small layout through the HBM kernels ----------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SMALL))
def test_hbm_keys_and_evaluations_from_every_base(ref_lib, name):
    """A loose-topic session is on the HBM path (it refuses the shared-memory evaluators), its rows add nothing, and
    its delta keys equal the restatement's from the initial, a random and both damaged bases; get_base after set_base
    equals the model on random, short-row, duplicate-broker and emptied assignments."""
    pb = SMALL[name]()
    r = ref_lib.Ref(pb)
    sess = hbm_session(pb)
    lib = kopt.load_library()
    assert lib.kao_set_evaluator(sess._h, C.c_int32(0)) == -1 and "topic rows" in lib.kao_last_error().decode()
    assert sess.stats()["words_per_row"] == r.W
    size = ROUND.get(name, 4096)
    rng = np.random.RandomState(7)
    bits, ld = r.init_base()
    reps = r.decode(bits, ld)
    assert topics_ref.evaluate(pb, one_loose_topic(pb), reps) == m.evaluate(pb, reps)
    bases = {"initial": reps, "random": malformed(pb, reps, rng)["random"], "emptied": emptied_base(pb, reps, 5),
             "moved": moved_base(pb, reps, 6)}
    assert empty_rows(bases["emptied"]) > 0 and empty_rows(bases["moved"]) == 0
    for what, b in bases.items():
        sess.set_base(b)
        bits, ld = r.encode(b)
        got_reps, v, o, _ = sess.get_base()
        assert (got_reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == m.evaluate(pb, got_reps)
        check_delta_keys(sess, r, bits, ld, size, what)
    for what, b in malformed(pb, reps, rng).items():
        sess.set_base(b)
        assert sess.get_base()[1:3] == m.evaluate(pb, b), what
    sess.close()


def walk_and_rebuild(pb, r, start, seed, rounds, size, keys_size=4096):
    """search_delta from `start` over `rounds` rounds in two calls against the restatement; then a fresh session on
    the walked base scores the next free and cycle rounds as the walked one does.  -> the walked session"""
    bits, ld = r.encode(start)
    sess = hbm_session(pb)
    sess.set_base(start)
    half = rounds // 2
    for first, n in ((0, half), (half, rounds - half)):
        _, want = r.search(bits, ld, seed, first, n, size)
        got, _ = sess.search_delta(seed, first, n, size)
        assert_keys(got, want, ("round", first))
    reps, v, o, _ = sess.get_base()
    assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == m.evaluate(pb, reps)
    fresh = hbm_session(pb)
    fresh.set_base(reps)
    for rnd in (rounds, rounds + 3):
        assert_keys(sess.candidate_keys_delta(seed, rnd, keys_size, 0, keys_size),
                    fresh.candidate_keys_delta(seed, rnd, keys_size, 0, keys_size), ("rebuilt", rnd))
    fresh.close()
    return sess, reps


@pytest.mark.parametrize("name", sorted(SMALL))
def test_hbm_long_walks_from_every_base(ref_lib, name):
    """48 rounds from the initial base and both damaged ones.  From the emptied base a partition stays led from a slot
    it does not hold in every round (an empty row is never refilled): the generator reads leader bytes throughout."""
    pb = SMALL[name]()
    r = ref_lib.Ref(pb)
    size = 256 if name in ROUND else 1024
    reps = r.decode(*r.init_base())
    for what, start in (("initial", reps), ("emptied", emptied_base(pb, reps, 5)), ("moved", moved_base(pb, reps, 6))):
        sess, end = walk_and_rebuild(pb, r, start, 0x5EED + len(what), WALK, size)
        if what == "emptied":
            assert empty_rows(end) == empty_rows(start) > 0
        sess.close()


@pytest.mark.parametrize("name", ["cfg2", "ragged", "rf_up", "rack5_w4", "dense_rack4_w2", "sat_cfg2"])
def test_hbm_patience_stops_where_the_shared_memory_search_does(ref_lib, name):
    pb = SMALL[name]()
    r = ref_lib.Ref(pb)
    got = {}
    for sess in (kao.Session(kao.Problem.from_fields(pb)), hbm_session(pb)):
        sess.set_patience(2)
        keys, _ = sess.search_delta(0x5A7, 0, 300, 512)
        got[len(got)] = (sess.last_rounds(), keys[:sess.last_rounds()])
        sess.close()
    (n0, k0), (n1, k1) = got[0], got[1]
    assert 0 < n0 < 300 and n0 == n1 and (k0 == k1).all()
    assert (k1 == r.search(*r.init_base(), 0x5A7, 0, n1, 512)[1]).all()


# ---- above 8,160 partitions ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(LARGE_SHAPES))
def test_large_layout_keys_and_trajectories(ref_lib, name):
    pb = LARGE_SHAPES[name]()
    r = ref_lib.Ref(pb)
    reps = r.decode(*r.init_base())
    sess = hbm_session(pb)
    assert sess.stats()["words_per_row"] == r.W
    for what, b in (("initial", reps), ("moved", moved_base(pb, reps, 6)), ("emptied", emptied_base(pb, reps, 5))):
        sess.set_base(b)
        bits, ld = r.encode(b)
        assert sess.get_base()[1:3] == r.evaluate(bits, ld)
        for rnd in (0, 3):
            got = sess.candidate_keys_delta(0xB16, rnd, 1024, 0, 1024)
            assert_keys(got, r.candidate_keys(bits, ld, 0xB16, rnd, 1024, 0, 1024), (what, rnd))
    sess.close()
    for what, start in (("initial", reps), ("emptied", emptied_base(pb, reps, 5))):
        walk_and_rebuild(pb, r, start, 0x77, 12, 512)[0].close()


@pytest.mark.parametrize("name", sorted(LARGE_SHAPES))
def test_large_layout_eval_equals_the_model(ref_lib, name):
    pb = LARGE_SHAPES[name]()
    r = ref_lib.Ref(pb)
    reps = r.decode(*r.init_base())
    batch = [reps] + list(malformed(pb, reps, np.random.RandomState(9)).values()) + [emptied_base(pb, reps, 11)]
    v, o = kopt.evaluate(kao.Problem.from_fields(pb), np.stack(batch))
    for i, b in enumerate(batch):
        assert (int(v[i]), int(o[i])) == m.evaluate(pb, b), i


def test_large_search_leaves_a_saturated_base_like_the_restatement(ref_lib):
    """Round 0's winner is a saturated key: the kernel re-evaluates its base in full before round 1.  The trajectory
    and the round patience stops it at equal the restatement's."""
    pb = LARGE_SHAPES["big_sat"]()
    r = ref_lib.Ref(pb)
    cap = (1 << (39 - r.obj_bits)) - 1
    bits, ld = r.init_base()
    assert r.evaluate(bits, ld)[0] > cap
    _, want = r.search(bits, ld, 0x5A7, 0, 10, 1024)
    viols = [r.unpack_key(k)[0] for k in want]
    assert viols[0] == cap and max(viols[1:]) < cap, viols
    sess = hbm_session(pb)
    got, _ = sess.search_delta(0x5A7, 0, 10, 1024)
    assert_keys(got, want, "saturated walk")
    reps, v, o, _ = sess.get_base()
    assert (reps == r.decode(bits, ld)).all() and (v, o) == m.evaluate(pb, reps)
    sess.close()
    # rounds of 8 candidates: saturated winners round after round, each base re-evaluated in full, until patience
    sess = hbm_session(pb)
    sess.set_patience(2)
    got, _ = sess.search_delta(0x5A7, 0, 100, 8)
    n = sess.last_rounds()
    assert 0 < n < 100
    assert_keys(got[:n], r.search(*r.init_base(), 0x5A7, 0, n, 8)[1], "patience")
    assert r.unpack_key(got[1])[0] == cap
    sess.close()


# ---- count limits at 65,280 partitions ----------------------------------------------------------------------------
def concentrated(P, B):
    """every partition on brokers 0 and 1 and led from broker 0; every partition led from broker 0, followers spread"""
    return {"brokers 0 and 1": np.tile(np.array([0, 1], np.int32), (P, 1)),
            "led from broker 0": np.stack([np.zeros(P, np.int32), 1 + np.arange(P, dtype=np.int32) % (B - 1)], 1)}


def test_concentrated_bases_at_65280(ref_lib):
    pb = m.synthetic_problem(65280, 16, 4, 2, remove=1)
    r = ref_lib.Ref(pb)
    bases = concentrated(pb.P, pb.B)
    v, o = kopt.evaluate(kao.Problem.from_fields(pb), np.stack(list(bases.values())))
    sess = hbm_session(pb)
    for i, (what, reps) in enumerate(bases.items()):
        want = m.evaluate(pb, reps)
        assert (int(v[i]), int(o[i])) == want, what
        sess.set_base(reps)
        assert sess.get_base()[1:3] == want, what
        bits, ld = r.encode(reps)
        for rnd in (0, 3):
            got = sess.candidate_keys_delta(0x8160, rnd, 4096, 0, 256)
            assert_keys(got, r.candidate_keys(bits, ld, 0x8160, rnd, 4096, 0, 256), (what, rnd))
    sess.close()


def test_one_topic_holding_65280_partitions(ref_lib):
    """A u16 topic cell at 65,280 next to its neighbour in the same 32-bit word of the count kernel's atomics"""
    pb = m.synthetic_problem(65280, 16, 4, 2, remove=1)
    pb.topics = [("t0", p) for p in range(pb.P)]
    tr = kao.topic_rows(kao.Problem.from_fields(pb))
    r = topics_ref.TRef(pb, tr)
    sess = kao.Session(kao.Problem.from_fields(pb), topics=tr)
    for what, reps in concentrated(pb.P, pb.B).items():
        sess.set_base(reps)
        bits, ld = r.encode(reps)
        assert sess.get_base()[1:3] == r.evaluate(bits, ld) == topics_ref.evaluate(pb, tr, reps), what
        for rnd in (0, 3):
            got = sess.candidate_keys_delta(0x7091, rnd, 4096, 0, 128)
            assert_keys(got, r.candidate_keys(bits, ld, 0x7091, rnd, 4096, 0, 128), (what, rnd))
    sess.close()


def test_one_topic_per_partition_at_65280_in_eight_word_rows(ref_lib):
    """T = P = 65,280 at W = 8: 16.7 M (topic, slot) cells (DESIGN.md 7.2).  16 racks of up to 16."""
    pb = make_problem(65280, [16] * 15 + [15], 3, seed=44, removed=3)
    pb.topics = [("t%d" % p, p) for p in range(pb.P)]
    tr = kao.topic_rows(kao.Problem.from_fields(pb))
    r = topics_ref.TRef(pb, tr)
    assert r.W == 8 and tr.T == pb.P
    sess = kao.Session(kao.Problem.from_fields(pb), topics=tr)
    bits, ld = r.init_base()
    for rnd in (0, 3):
        got = sess.candidate_keys_delta(0x7A, rnd, 4096, 0, 48)
        assert_keys(got, r.candidate_keys(bits, ld, 0x7A, rnd, 4096, 0, 48), ("keys", rnd))
    _, want = r.search(bits, ld, 0x7A, 0, 3, 32)
    got, _ = sess.search_delta(0x7A, 0, 3, 32)
    assert_keys(got, want, "walk")
    reps, v, o, _ = sess.get_base()
    assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == topics_ref.evaluate(pb, tr, reps)
    sess.close()


@pytest.mark.parametrize("topics", [False, True])
def test_long_run_at_65280_equals_a_rebuilt_session(topics):
    """300 rounds of 4,096 candidates; then a fresh session on the walked base scores the next rounds as the walked
    one does, and get_base equals the model"""
    pb = m.synthetic_problem(65280, 64, 8, 3, remove=1)
    tr = None
    if topics:
        pb.topics = [("t%d" % (p // 50), p) for p in range(pb.P)]
        tr = kao.topic_rows(kao.Problem.from_fields(pb))
    kp = kao.Problem.from_fields(pb)
    sess = kao.Session(kp, topics=tr)
    sess.search_delta(0x5EED, 0, 150, 4096)
    sess.search_delta(0x5EED, 150, 150, 4096)
    reps, v, o, _ = sess.get_base()
    assert (v, o) == (topics_ref.evaluate(pb, tr, reps) if topics else m.evaluate(pb, reps))
    fresh = kao.Session(kp, topics=tr)
    fresh.set_base(reps)
    assert fresh.get_base()[1:3] == (v, o)
    for rnd in (300, 303):
        assert_keys(sess.candidate_keys_delta(0x5EED, rnd, 4096, 0, 4096),
                    fresh.candidate_keys_delta(0x5EED, rnd, 4096, 0, 4096), ("rebuilt", rnd))
    sess.close()
    fresh.close()
