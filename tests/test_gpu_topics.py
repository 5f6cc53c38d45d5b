"""Per-topic balance rows (docs/MODEL.md §10, DESIGN.md 7.2) through the C ABI, below and above 8,160 partitions:
delta keys, trajectories and kao_get_base are bit-identical to the restatement (tests/topics_ref) and the model with
topic rows; non-binding rows leave kao_solve's result as it is; small instances reach the HiGHS optimum; what a topic
session does not offer is refused with KAO_E_ARG."""
import ctypes as C

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import topics_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import with_dense_weights
from conftest import make_problem

pytestmark = pytest.mark.gpu


def with_topics(pb, topic_of):
    """pb labelled with the topic of every row (name "t<k>"); -> (pb, default TopicRows of kao.topic_rows)."""
    pb.topics = [("t%d" % int(t), p) for p, t in enumerate(topic_of)]
    return pb, kao.topic_rows(kao.Problem.from_fields(pb))


SHAPES = {
    "p700_w1_t30": lambda: with_topics(m.synthetic_problem(700, 20, 2, 2, remove=1), np.arange(700) % 30),
    "p8161_w1": lambda: with_topics(m.synthetic_problem(8161, 32, 4, 3, remove=1), np.arange(8161) // 50),
    "p20000_w2_t400": lambda: with_topics(m.synthetic_problem(20000, 48, 8, 3, remove=1), np.arange(20000) // 50),
    # 3 racks of 20: padding slots, which carry no topic row
    "p6000_w4": lambda: with_topics(make_problem(6000, [20, 20, 20], 3, seed=41, removed=2), np.arange(6000) // 40),
    "p65280_w2": lambda: with_topics(m.synthetic_problem(65280, 64, 8, 3, remove=1), np.arange(65280) // 50),
    "p3000_w8": lambda: with_topics(make_problem(3000, [16] * 15 + [15], 3, seed=42, removed=2), np.arange(3000) // 30),
    "p9000_dense": lambda: with_topics(with_dense_weights(m.synthetic_problem(9000, 32, 4, 3, remove=1), 43),
                                       np.random.RandomState(3).randint(0, 180, 9000)),
}
ROUND = {"p65280_w2": 512, "p20000_w2_t400": 1024}     # candidates per round of the restatement comparisons


def _damage(pb, reps, seed):
    """Replicas moved to random brokers (duplicates collapse), rows cut short, a few emptied."""
    rng = np.random.RandomState(seed)
    out = reps.copy()
    for p in rng.choice(pb.P, size=min(300, pb.P // 2), replace=False):
        out[p, rng.randint(pb.RF)] = rng.randint(pb.B)
    out[rng.choice(pb.P, size=20, replace=False), -1] = -1
    out[rng.choice(pb.P, size=5, replace=False), :] = -1
    return out


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_topic_delta_keys_equal_the_restatement(ref_lib, name):
    pb, tr = SHAPES[name]()
    r = topics_ref.TRef(pb, tr)
    sess = kao.Session(kao.Problem.from_fields(pb), topics=tr)
    assert sess.stats()["words_per_row"] == r.W
    size = ROUND.get(name, 2048)
    bits, ld = r.init_base()
    for base in ("initial", "damaged"):
        if base == "damaged":
            bits, ld = r.encode(_damage(pb, r.decode(bits, ld), 5))
            sess.set_base(r.decode(bits, ld))
        assert sess.get_base()[1:3] == r.evaluate(bits, ld)
        for rnd in (0, 3):                        # a free round and a cycle round (round mod 4 = 3)
            got = sess.candidate_keys_delta(0xB16, rnd, size, 0, size)
            want = r.candidate_keys(bits, ld, 0xB16, rnd, size, 0, size)
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, (base, rnd, int(bad[0]), sess.unpack_key(got[bad[0]]), r.unpack_key(want[bad[0]]))
    sess.close()


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_topic_search_walks_the_restatement_trajectory(ref_lib, name):
    pb, tr = SHAPES[name]()
    r = topics_ref.TRef(pb, tr)
    size = ROUND.get(name, 2048)
    bits, ld = r.init_base()
    _, want = r.search(bits, ld, 0x5EED, 0, 8, size)
    sess = kao.Session(kao.Problem.from_fields(pb), topics=tr)
    got, _ = sess.search_delta(0x5EED, 0, 8, size)
    assert (got == want).all()
    reps, v, o, _ = sess.get_base()
    assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld)
    # a second call continues from the patched base and its patched topic counts
    _, want2 = r.search(bits, ld, 0x77, 8, 4, size)
    got2, _ = sess.search_delta(0x77, 8, 4, size)
    assert (got2 == want2).all()
    reps, v, o, _ = sess.get_base()
    assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld)
    sess.close()


@pytest.mark.parametrize("name", ["p700_w1_t30", "p6000_w4", "p9000_dense"])
def test_get_base_after_set_base_equals_the_model(ref_lib, name):
    pb, tr = SHAPES[name]()
    r = topics_ref.TRef(pb, tr)
    sess = kao.Session(kao.Problem.from_fields(pb), topics=tr)
    rng = np.random.RandomState(9)
    generated = r.decode(*r.init_base())
    random = np.stack([rng.choice(pb.B, size=pb.RF, replace=False) for _ in range(pb.P)]).astype(np.int32)
    malformed = _damage(pb, generated, 11)
    malformed[7, :] = malformed[7, 0]
    for reps in (generated, random, malformed):
        sess.set_base(reps)
        _, v, o, _ = sess.get_base()
        assert (v, o) == topics_ref.evaluate(pb, tr, reps)
    sess.close()


def _loose(pb, tr):
    """The same topics with rows no assignment can violate"""
    n = np.bincount(tr.topic_of, minlength=tr.T).astype(np.int32)
    return kao.TopicRows(tr.topic_of, np.zeros_like(n), n * pb.RF, np.zeros_like(n), n, tr.names)


@pytest.mark.parametrize("name", ["p700_w1_t30", "p8161_w1", "p9000_dense"])
def test_non_binding_topic_rows_leave_the_delta_solve_as_it_is(name):
    pb, tr = SHAPES[name]()
    kp = kao.Problem.from_fields(pb)
    plain = kopt.solve(kp, seed=0xC0FFEE, rounds=40, round_size=4096, restarts=2, delta=True)
    loose = kopt.solve(kp, seed=0xC0FFEE, rounds=40, round_size=4096, restarts=2, topics=_loose(pb, tr))
    for f in ("objective", "violation", "moves", "feasible", "key", "n_candidates", "rounds", "objective_bound", "optimal"):
        assert getattr(loose, f) == getattr(plain, f), f
    assert (loose.replicas == plain.replicas).all()


def _ref_solve(r, seed, restarts, rounds, size):
    best = None
    for k in range(restarts):
        bits, ld = r.init_base()
        r.search(bits, ld, (seed + 0x9E3779B97F4A7C15 * k) % 2 ** 64, 0, rounds, size)
        v, o = r.evaluate(bits, ld)
        if best is None or (v, -o) < (best[0], -best[1]):
            best = (v, o, r.decode(bits, ld))
    return best


@pytest.mark.parametrize("spread", [False, True])
def test_topic_solve_with_restarts_equals_the_restatement(ref_lib, spread):
    import torch

    pb, tr = SHAPES["p700_w1_t30"]()
    r = topics_ref.TRef(pb, tr)
    v, o, reps = _ref_solve(r, 0xC0FFEE, 3, 6, 2048)
    n = torch.cuda.device_count() if spread else 1
    res = kopt.solve(kao.Problem.from_fields(pb), seed=0xC0FFEE, rounds=6, round_size=2048, restarts=3,
                     spread_restarts=spread, n_gpus=n, topic_balance=True)
    assert (res.violation, res.objective) == (v, o) and (res.replicas == reps).all()
    assert res.rounds == 18


def readme_three_topics():
    """The README topology (20 brokers in racks a / b by parity, broker 19 removed) with 20 partitions in three topics
    of 10, 6 and 4; RF 3, because with RF 2 the rack totals of 40 replicas cannot be met (every partition puts one
    replica in each rack)."""
    cur = [[p % 20, (p + 11) % 20, (p + 2) % 20] for p in range(20)]
    topics = [("a", p) for p in range(10)] + [("b", p) for p in range(6)] + [("c", p) for p in range(4)]
    pb = m.build_problem(cur, list(range(19)), {b: ("b" if b % 2 else "a") for b in range(20)}, 3, topics=topics)
    return pb, kao.topic_rows(kao.Problem.from_fields(pb))


def s256_sixteen_topics():
    return with_topics(m.synthetic_problem(256, 32, 4, 3, remove=1), np.arange(256) // 16)


@pytest.mark.parametrize("make", [readme_three_topics, s256_sixteen_topics])
def test_topic_solve_reaches_the_highs_optimum(make):
    pb, tr = make()
    sol = topics_ref.solve_exact(pb, tr)
    assert sol.status == "optimal"
    res = kopt.solve(kao.Problem.from_fields(pb), seed=0x5EED, rounds=2000, round_size=1 << 14, restarts=8,
                     patience=400, topic_balance=True)
    assert res.feasible and topics_ref.evaluate(pb, tr, res.replicas) == (0, res.objective)
    assert res.objective == sol.objective, (res.objective, sol.objective)
    assert res.objective <= res.objective_bound


def test_one_broker_removed_keeps_every_topic_spread():
    """Broker 47 removed from 20,000 partitions in 400 topics of 50 on 48 brokers (the instance test_gpu_large pins
    for plain kao_solve at 1,273 moves): with topic rows the result must be feasible including them.  The plain result
    violates 983 topic rows; the pinned recipe (same candidate stream, deterministic trajectory) reaches a feasible
    assignment with 2,073 moves against the lower bound of 1,248 (DESIGN.md 7.2)."""
    pb, tr = with_topics(m.synthetic_problem(20000, 48, 8, 3, remove=1), np.arange(20000) // 50)
    kp = kao.Problem.from_fields(pb)
    lower = int((pb.cur < 0).sum())
    plain = kopt.solve(kp, seed=0x5EED, rounds=3000, round_size=1 << 13, patience=500)
    res = kopt.solve(kp, seed=0x5EED, rounds=3000, round_size=1 << 13, patience=500, topic_balance=True)
    plain_rows = topics_ref.violated_rows(pb, tr, plain.replicas)
    print("broker removal with topic rows: feasible %s, violation %d, moves %d (lower bound %d), objective %d, "
          "rounds %d, %.1f ms; the plain result (%d moves) violates %d topic rows"
          % (res.feasible, res.violation, res.moves, lower, res.objective, res.rounds, res.total_ms, plain.moves,
             plain_rows))
    assert plain.moves == 1273 and plain_rows == 983
    assert res.feasible and topics_ref.evaluate(pb, tr, res.replicas) == (0, res.objective)
    assert topics_ref.violated_rows(pb, tr, res.replicas) == 0
    assert res.moves == m.replica_moves(pb, res.replicas) == 2073 and res.objective == 135890


def test_what_a_topic_session_does_not_offer_is_refused():
    lib = kopt.load_library()
    pb, tr = SHAPES["p700_w1_t30"]()
    sess = kao.Session(kao.Problem.from_fields(pb), topics=tr)
    h = sess._h
    keys = np.zeros(16, np.uint64)
    null = C.c_void_p()

    def refused(rc):
        return rc == -1 and "topic rows" in lib.kao_last_error().decode()

    assert refused(lib.kao_search(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(1), C.c_uint32(16), C.c_void_p(keys.ctypes.data), null))
    assert refused(lib.kao_candidate_keys(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(16), C.c_uint32(0), C.c_uint32(16),
                                          C.c_void_p(keys.ctypes.data)))
    assert refused(lib.kao_set_evaluator(h, C.c_int32(0)))
    assert refused(lib.kao_set_schedule(h, C.c_int32(1), C.c_int32(0x200), C.c_int32(512)))
    assert refused(lib.kao_round_launch(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(16), C.c_uint32(0), C.c_uint32(16),
                                        C.c_void_p(keys.ctypes.data), null))
    assert refused(lib.kao_round_apply(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(16), C.c_void_p(keys.ctypes.data), null))
    a, b = C.c_double(), C.c_double()
    assert refused(lib.kao_profile_rounds(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(1), C.c_uint32(16), C.byref(a), C.byref(b)))
    blob = (C.c_uint8 * 128)()
    assert refused(lib.kao_p2p_export(h, blob))
    assert refused(lib.kao_p2p_connect(h, C.c_int32(0), C.c_int32(2), blob))
    for fn in (lib.kao_search_sharded, lib.kao_search_sharded_delta):
        assert refused(fn(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(1), C.c_uint32(16), C.c_void_p(keys.ctypes.data), C.byref(a)))
    # the session is still usable for what it does offer
    got, _ = sess.search_delta(1, 0, 2, 256)
    assert got.size == 2 and sess.last_rounds() == 2
    sess.close()
    cp, ct = kopt._CProblem(kao.Problem.from_fields(pb)), kopt._CTopics(tr)
    for flags, n_gpus in ((0x200, 1), (0x1, 2)):              # KAO_FLAG_ROW_MAJOR; rounds sharded over two GPUs
        reps = np.zeros((pb.P, pb.RF), np.int32)
        opt = kopt._KaoOptions(1, 2, 256, 0, flags, n_gpus, 0)
        res = kopt._KaoResult()
        res.replicas = reps.ctypes.data
        assert refused(lib.kao_solve_topics(cp.ref(), ct.ref(), C.byref(opt), C.byref(res)))
