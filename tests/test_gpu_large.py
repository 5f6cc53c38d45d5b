"""The large path (DESIGN.md 7.1): 8,161 .. 65,280 partitions with the base in HBM, through the C ABI.  Delta keys,
trajectories, kao_solve (restarts, spread restarts) and kao_eval are bit-identical to the plain-C restatement and the
model; what the large path does not offer is refused with KAO_E_ARG."""
import ctypes as C

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import with_dense_weights
from conftest import make_problem

pytestmark = pytest.mark.gpu

SHAPES = {
    "p8161_w1": lambda: m.synthetic_problem(8161, 32, 4, 3, remove=1),                       # 32 slots, one word
    "p65280_w2": lambda: m.synthetic_problem(65280, 64, 8, 3, remove=1),                     # 64 slots, 8 racks
    "p20000_w4": lambda: make_problem(20000, [20, 20, 20], 3, seed=41, removed=2),           # 3 racks of 20: padding slots
    # 16 racks of up to 16: slot 255 stays padding (DESIGN.md 7.1: a home replica there reads as "no home slot")
    "p12000_w8": lambda: make_problem(12000, [16] * 15 + [15], 3, seed=42, removed=2),
    "p9000_dense": lambda: with_dense_weights(m.synthetic_problem(9000, 32, 4, 3, remove=1), 43),
}
ROUND = {"p65280_w2": 512}          # candidates per round of the restatement comparisons (each costs O(P) on the CPU)


def _damage(pb, reps, seed):
    """Replicas moved to random brokers (duplicates collapse), rows cut short, a few emptied."""
    rng = np.random.RandomState(seed)
    out = reps.copy()
    for p in rng.choice(pb.P, size=300, replace=False):
        out[p, rng.randint(pb.RF)] = rng.randint(pb.B)
    out[rng.choice(pb.P, size=20, replace=False), -1] = -1
    out[rng.choice(pb.P, size=5, replace=False), :] = -1
    return out


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_delta_keys_equal_the_restatement(ref_lib, name):
    pb = SHAPES[name]()
    r = ref_lib.Ref(pb)
    sess = kao.Session(kao.Problem.from_fields(pb))
    assert sess.stats()["words_per_row"] == r.W
    size = ROUND.get(name, 2048)
    bits, ld = r.init_base()
    for base in ("initial", "damaged"):
        if base == "damaged":
            bits, ld = r.encode(_damage(pb, r.decode(bits, ld), 5))
            sess.set_base(r.decode(bits, ld))
        for rnd in (0, 3):                        # a free round and a cycle round (round mod 4 = 3)
            got = sess.candidate_keys_delta(0xB16, rnd, size, 0, size)
            want = r.candidate_keys(bits, ld, 0xB16, rnd, size, 0, size)
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, (base, rnd, int(bad[0]), sess.unpack_key(got[bad[0]]), r.unpack_key(want[bad[0]]))
    sess.close()


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_delta_search_walks_the_restatement_trajectory(ref_lib, name):
    pb = SHAPES[name]()
    r = ref_lib.Ref(pb)
    size = ROUND.get(name, 2048)
    bits, ld = r.init_base()
    _, want = r.search(bits, ld, 0x5EED, 0, 8, size)
    sess = kao.Session(kao.Problem.from_fields(pb))
    got, ms = sess.search_delta(0x5EED, 0, 8, size)
    assert (got == want).all()
    assert sess.last_rounds() == 8
    reps, v, o, _ = sess.get_base()
    assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld)
    # a second call continues from the patched base, the lists and planes kept in step with it
    _, want2 = r.search(bits, ld, 0x77, 8, 4, size)
    got2, _ = sess.search_delta(0x77, 8, 4, size)
    assert (got2 == want2).all() and (sess.get_base()[0] == r.decode(bits, ld)).all()
    sess.close()


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
def test_solve_with_restarts_equals_the_restatement(ref_lib, spread):
    import torch

    pb = SHAPES["p8161_w1"]()
    r = ref_lib.Ref(pb)
    v, o, reps = _ref_solve(r, 0xC0FFEE, 3, 6, 2048)
    n = torch.cuda.device_count() if spread else 1
    res = kopt.solve(kao.Problem.from_fields(pb), seed=0xC0FFEE, rounds=6, round_size=2048, restarts=3,
                     spread_restarts=spread, n_gpus=n)
    assert (res.violation, res.objective) == (v, o) and (res.replicas == reps).all()
    assert res.rounds == 18


def test_eval_equals_the_model(ref_lib):
    for name in ("p8161_w1", "p9000_dense"):
        pb = SHAPES[name]()
        r = ref_lib.Ref(pb)
        rng = np.random.RandomState(9)
        generated = r.decode(*r.init_base())
        random = np.stack([rng.choice(pb.B, size=pb.RF, replace=False) for _ in range(pb.P)]).astype(np.int32)
        malformed = _damage(pb, generated, 11)
        malformed[7] = [3, 3, 3]
        batch = np.stack([generated, random, malformed])
        v, o = kopt.evaluate(kao.Problem.from_fields(pb), batch)
        for i in range(3):
            assert (int(v[i]), int(o[i])) == m.evaluate(pb, batch[i]), (name, i)


def test_one_broker_removed_from_a_balanced_cluster():
    """48 brokers in 8 racks, 20,000 partitions in round robin, broker 47 removed: every replica it held must move
    (1,248, a lower bound every assignment meets).  The pinned recipe (deterministic trajectory) reaches a feasible
    assignment 25 moves above that bound; no recipe tried that runs in test time reached the bound (DESIGN.md 7.1)."""
    pb = m.synthetic_problem(20000, 48, 8, 3, remove=1)
    lower = int((pb.cur < 0).sum())
    assert lower == 1248
    res = kopt.solve(kao.Problem.from_fields(pb), seed=0x5EED, rounds=3000, round_size=1 << 13, patience=500)
    assert res.feasible and m.evaluate(pb, res.replicas) == (0, res.objective)
    assert res.moves == m.replica_moves(pb, res.replicas) == 1273 and res.objective == 136833
    assert res.objective <= res.objective_bound == 137088
    print("broker removal: moves %d (lower bound %d), objective %d, bound %d, rounds %d, %.1f ms"
          % (res.moves, lower, res.objective, res.objective_bound, res.rounds, res.total_ms))


def _lib():
    return kopt.load_library()


def test_what_the_large_path_does_not_offer_is_refused():
    lib = _lib()
    pb = SHAPES["p8161_w1"]()
    sess = kao.Session(kao.Problem.from_fields(pb))
    h = sess._h
    keys = np.zeros(16, np.uint64)
    null = C.c_void_p()

    def refused(rc):
        return rc == -1 and "8,160" in lib.kao_last_error().decode()

    assert refused(lib.kao_search(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(1), C.c_uint32(16), C.c_void_p(keys.ctypes.data), null))
    assert refused(lib.kao_candidate_keys(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(16), C.c_uint32(0), C.c_uint32(16),
                                          C.c_void_p(keys.ctypes.data)))
    assert refused(lib.kao_set_evaluator(h, C.c_int32(0)))
    assert refused(lib.kao_set_schedule(h, C.c_int32(1), C.c_int32(0x200), C.c_int32(512)))
    assert refused(lib.kao_round_launch(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(16), C.c_uint32(0), C.c_uint32(16),
                                        C.c_void_p(keys.ctypes.data), null))
    assert refused(lib.kao_round_apply(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(16), C.c_void_p(keys.ctypes.data), null))
    blob = (C.c_uint8 * 128)()
    assert refused(lib.kao_p2p_export(h, blob))
    assert refused(lib.kao_p2p_connect(h, C.c_int32(0), C.c_int32(2), blob))
    ms = C.c_double()
    for fn in (lib.kao_search_sharded, lib.kao_search_sharded_delta):
        assert refused(fn(h, C.c_uint64(1), C.c_uint32(0), C.c_uint32(1), C.c_uint32(16), C.c_void_p(keys.ctypes.data), C.byref(ms)))
    # the session is still usable for what it does offer
    got, _ = sess.search_delta(1, 0, 2, 256)
    assert got.size == 2 and sess.stats()["words_per_row"] == 1
    sess.close()
    cp = kopt._CProblem(kao.Problem.from_fields(pb))
    for flags, n_gpus in ((0x200, 1), (0x1, 2)):              # KAO_FLAG_ROW_MAJOR; rounds sharded over two GPUs
        reps = np.zeros((pb.P, pb.RF), np.int32)
        opt = kopt._KaoOptions(1, 2, 256, 0, flags, n_gpus, 0)
        res = kopt._KaoResult()
        res.replicas = reps.ctypes.data
        assert refused(lib.kao_solve(cp.ref(), C.byref(opt), C.byref(res)))
    # the LP bound's build limit (P * RF < 2^16, P <= 8,160): refused before any search
    reps = np.zeros((pb.P, pb.RF), np.int32)
    opt = kopt._KaoOptions(1, 2, 256, 0, 0x1000, 1, 0)
    res = kopt._KaoResult()
    res.replicas = reps.ctypes.data
    assert lib.kao_solve(cp.ref(), C.byref(opt), C.byref(res)) == -1 and "2^16" in lib.kao_last_error().decode()
    with pytest.raises(kopt.KaoError, match="2\\^16"):
        kopt.lp_bound(kao.Problem.from_fields(pb), reps)
