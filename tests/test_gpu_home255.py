"""Home replicas on slot 255, on the GPU: 256-broker clusters where broker 255 sits on slot 255 and holds current
replicas (problems.HOME255_SHAPES).  When every slot is a broker the home byte 0xFF is slot 255 itself, and the guided
operations (REPLACE back to a missing home, LEADER back to home0, the cycle rounds) and the displaced lists D / DL must
count it as docs/MODEL.md §5.1 does.  Every runner a shape reaches (the row-major full search, the delta search, the
HBM path, topic and replication sessions, kao_solve_fixed on a reduced eight-word problem) is held bit for bit to its
restatement (oracle/kao_ref.c, tests/topics_ref, tests/rf_ref) from bases whose lists hold only partitions displaced
from slot 255 (problems.home255_bases), over long walks, through the per-round entry points and patience; and config
5' (4,096 x 256 brokers, broker 255 on slot 255) over a 64-round trajectory from its initial base."""
import copy
import dataclasses
import json
import os

import numpy as np
import pytest

import fixed_ref as F
import kafka_assignment_optimizer_b200 as kao
import rf_ref
import topics_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import HOME255_SHAPES, home255_bases, mixed_rows
from test_gpu_large_layouts import assert_keys, hbm_session
from test_gpu_smem_walks import open_runner, restatement_until_stop, runners

pytestmark = pytest.mark.gpu

BIG = 8160
SMALL = sorted(n for n, f in HOME255_SHAPES.items() if n != "h255_big")
WALK, PROBE = 48, 400


@pytest.fixture(scope="module")
def optima():
    with open(os.path.join(os.path.dirname(__file__), "golden", "optima.json")) as f:
        return json.load(f)


class Runner:
    """One session configuration with the restatement and the model evaluation it is held to"""

    def __init__(self, name, open_session, r, evaluate, delta):
        self.name, self.open, self.r, self.evaluate, self.delta = name, open_session, r, evaluate, delta

    def keys(self, sess, seed, rnd, size, lo, n):
        return (sess.candidate_keys_delta if self.delta else sess.candidate_keys)(seed, rnd, size, lo, n)

    def search(self, sess, seed, first, n, size):
        return (sess.search_delta if self.delta else sess.search)(seed, first, n, size)[0]


def all_runners(pb, ref_lib):
    """name -> Runner for every runner the shape reaches: the shared-memory runners (row-major full search, delta) up
    to 8,160 partitions, the HBM path, a topic session (five interleaved topics) and a replication session (mixed
    per-partition rows)"""
    r = ref_lib.Ref(pb)
    plain = lambda reps: m.evaluate(pb, reps)
    out = {}
    if pb.P <= BIG:
        for run in runners(pb):
            out[run[0]] = Runner(run[0], lambda run=run: open_runner(pb, run), r, plain, run[3])
        assert set(out) == {"row_major", "delta"}, sorted(out)
    out["hbm"] = Runner("hbm", lambda: hbm_session(pb), r, plain, True)
    tpb = copy.copy(pb)
    tpb.topics = [("t%d" % (p % 5), p) for p in range(pb.P)]
    tr = kao.topic_rows(kao.Problem.from_fields(tpb))
    out["topics"] = Runner("topics", lambda: kao.Session(kao.Problem.from_fields(tpb), topics=tr),
                           topics_ref.TRef(tpb, tr), lambda reps: topics_ref.evaluate(tpb, tr, reps), True)
    kp = kao.Problem.from_fields(pb)
    kp.replication = mixed_rows(kp, 0x255)
    out["replication"] = Runner("replication", lambda: kao.Session(kp), rf_ref.RRef(kp, kp.replication, None),
                                lambda reps: rf_ref.evaluate(kp, kp.replication, reps, None), True)
    return out


def targeted(pb, ref_lib):
    """the initial base and the bases whose displaced lists hold only partitions displaced from slot 255"""
    r = ref_lib.Ref(pb)
    reps = r.decode(*r.init_base())
    return {"initial": reps, **home255_bases(pb, reps)}


def check_end(sess, run, bits, ld, what):
    reps, v, o, _ = sess.get_base()
    assert (reps == run.r.decode(bits, ld)).all(), what
    assert (v, o) == run.r.evaluate(bits, ld) == run.evaluate(reps), what
    return reps


# ---- candidate keys --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(HOME255_SHAPES))
def test_keys_of_free_and_cycle_rounds_from_home255_bases(ref_lib, name):
    """A free round (4) and a cycle round (7, every candidate guided) on every runner from every targeted base; get_base
    after set_base equals the restatement and the model"""
    pb = HOME255_SHAPES[name]()
    size = 1024
    bases = targeted(pb, ref_lib)
    for run in all_runners(pb, ref_lib).values():
        sess = run.open()
        assert sess.stats()["words_per_row"] == 8
        for what, b in bases.items():
            sess.set_base(b)
            bits, ld = run.r.encode(b)
            check_end(sess, run, bits, ld, (run.name, what))
            for rnd in (4, 7):
                assert_keys(run.keys(sess, 0xB16, rnd, size, 0, size),
                            run.r.candidate_keys(bits, ld, 0xB16, rnd, size, 0, size), (run.name, what, rnd))
        sess.close()


# ---- walks -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SMALL)
def test_walks_from_home255_bases(ref_lib, name):
    """48 rounds of 1,024 in two calls (the second restages the base and the lists from HBM) and 400 rounds of 4 on
    every runner from every targeted base; then the rebuild check: a fresh session on the walked base scores the next
    free and cycle rounds as the walked one does, and on the shared-memory runners the row-major per-round kernel reads
    the displaced lists the search left in HBM"""
    pb = HOME255_SHAPES[name]()
    bases = targeted(pb, ref_lib)
    for run in all_runners(pb, ref_lib).values():
        for what, start in bases.items():
            tag = (run.name, what)
            seed = 0x5EED0 + len(what)
            bits, ld = run.r.encode(start)
            _, want = run.r.search(bits, ld, seed, 0, WALK, 1024)
            sess = run.open()
            sess.set_base(start)
            got = np.concatenate([run.search(sess, seed, 0, WALK // 2, 1024),
                                  run.search(sess, seed, WALK // 2, WALK - WALK // 2, 1024)])
            assert_keys(got, want, tag + ("long walk",))
            reps = check_end(sess, run, bits, ld, tag + ("long walk",))
            fresh = run.open()
            fresh.set_base(reps)
            for rnd in (WALK, WALK + 3):
                want_k = run.r.candidate_keys(bits, ld, seed, rnd, 4096, 0, 4096)
                for who, s in (("walked", sess), ("fresh", fresh)):
                    assert_keys(run.keys(s, seed, rnd, 4096, 0, 4096), want_k, tag + (who, rnd))
            if run.name in ("row_major", "delta"):
                assert sess.set_evaluator(False)
                for rnd in (WALK, WALK + 3):
                    assert_keys(sess.candidate_keys(seed, rnd, 4096, 0, 4096),
                                run.r.candidate_keys(bits, ld, seed, rnd, 4096, 0, 4096), tag + ("walked row-major", rnd))
            fresh.close()
            sess.close()
            pbits, pld = run.r.encode(start)
            _, want = run.r.search(pbits, pld, seed ^ 0x77, 0, PROBE, 4)
            sess = run.open()
            sess.set_base(start)
            assert_keys(run.search(sess, seed ^ 0x77, 0, PROBE, 4), want, tag + ("probe walk",))
            check_end(sess, run, pbits, pld, tag + ("probe walk",))
            sess.close()


def test_walks_above_8160_partitions(ref_lib):
    """h255_big (8,200 partitions): the HBM path, topic and replication sessions over 24 rounds of 512 in two calls from
    every targeted base, then a fresh session on the walked base"""
    pb = HOME255_SHAPES["h255_big"]()
    for run in all_runners(pb, ref_lib).values():
        for what, start in targeted(pb, ref_lib).items():
            bits, ld = run.r.encode(start)
            sess = run.open()
            sess.set_base(start)
            for first, n in ((0, 12), (12, 12)):
                _, want = run.r.search(bits, ld, 0x77, first, n, 512)
                assert_keys(run.search(sess, 0x77, first, n, 512), want, (run.name, what, first))
            reps = check_end(sess, run, bits, ld, (run.name, what))
            fresh = run.open()
            fresh.set_base(reps)
            for rnd in (24, 27):
                assert_keys(run.keys(sess, 0x77, rnd, 1024, 0, 1024), run.keys(fresh, 0x77, rnd, 1024, 0, 1024),
                            (run.name, what, "rebuilt", rnd))
            fresh.close()
            sess.close()


# ---- entry points and patience ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SMALL)
def test_round_launch_and_apply_between_searches(ref_lib, name):
    """search, round_launch / round_apply (each round in three shards), search_delta and search again on one session
    from the D-targeted base, with consecutive rounds of one seed: each entry point reads the lists the one before it
    left in HBM"""
    import torch

    pb = HOME255_SHAPES[name]()
    r = ref_lib.Ref(pb)
    start = targeted(pb, ref_lib)["d255"]
    bits, ld = r.encode(start)
    seed, size, first = 0xE17, 1024, 0
    sess = kao.Session(kao.Problem.from_fields(pb))
    sess.set_base(start)

    def by_shards(f, n):
        key = torch.empty(1, dtype=torch.int64, device="cuda")
        got = []
        for rnd in range(f, f + n):
            key.fill_(kopt.KEY_NONE)
            for lo, hi in [(0, 300), (300, 301), (301, size)]:
                sess.round_launch(seed, rnd, size, lo, hi, key.data_ptr())
            sess.round_apply(seed, rnd, size, key.data_ptr())
            torch.cuda.synchronize()
            got.append(int(key.item()) & 0xFFFFFFFFFFFFFFFF)
        return np.array(got, np.uint64)

    for what, call in (("search", lambda f, n: sess.search(seed, f, n, size)[0]), ("round_launch / round_apply", by_shards),
                       ("search_delta", lambda f, n: sess.search_delta(seed, f, n, size)[0]),
                       ("search again", lambda f, n: sess.search(seed, f, n, size)[0])):
        got = call(first, 8)
        _, want = r.search(bits, ld, seed, first, 8, size)
        assert_keys(got, want, what)
        first += 8
        reps, v, o, _ = sess.get_base()
        assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == m.evaluate(pb, reps), what
    sess.close()


@pytest.mark.parametrize("name", ["h255_r16_rr", "h255_rf_down"])
def test_patience_from_home255_bases(ref_lib, name):
    """The round patience stops at on the row-major, delta and HBM runners from the targeted bases is its definition's
    over the restatement's keys"""
    pb = HOME255_SHAPES[name]()
    seed, size, cap, n = 0x9A7, 512, 2000, 5
    runs = {k: v for k, v in all_runners(pb, ref_lib).items() if k in ("row_major", "delta", "hbm")}
    for what, start in targeted(pb, ref_lib).items():
        if what == "initial":
            continue
        stop, want = restatement_until_stop(ref_lib.Ref(pb), *ref_lib.Ref(pb).encode(start), seed, n, cap, size)
        assert 0 < stop < cap, (what, stop)
        for run in runs.values():
            sess = run.open()
            sess.set_base(start)
            sess.set_patience(n)
            got = run.search(sess, seed, 0, cap, size)
            assert sess.last_rounds() == stop, (run.name, what, sess.last_rounds(), stop)
            assert_keys(got[:stop], want, (run.name, what))
            sess.close()


# ---- fixed partitions ----------------------------------------------------------------------------------------------------
def test_solve_fixed_on_an_eight_word_reduced_problem(ref_lib):
    """kao_solve_fixed with half the partitions of h255_r16_rr fixed: the reduced problem keeps 256 brokers and home
    replicas on slot 255, and its search is the restatement's trajectory on the reduced problem, bit for bit"""
    opb = HOME255_SHAPES["h255_r16_rr"]()
    pb = kao.Problem.from_fields(opb)
    fx = F.random_mask(pb, 0x255, share=0.5)
    assert fx.any() and not fx.all()
    red = F.reduce(pb, fx)
    r = ref_lib.Ref(red.pb)
    assert r.W == 8 and (red.pb.cur == 255).any()
    seed, rounds, size = 0xF1, 24, 4096
    got = kopt.solve(dataclasses.replace(pb, fixed=fx), seed=seed, rounds=rounds, round_size=size)
    want = kopt.solve(red.pb, seed=seed, rounds=rounds, round_size=size)
    assert np.array_equal(got.replicas[red.searched], want.replicas) and got.key == want.key
    bits, ld = r.init_base()
    r.search(bits, ld, seed, 0, rounds, size)
    assert np.array_equal(want.replicas, r.decode(bits, ld))
    assert (want.violation, want.objective) == r.evaluate(bits, ld)


# ---- config 5' at full size ---------------------------------------------------------------------------------------------
def test_config5_prime_trajectory_of_64_rounds(ref_lib, optima):
    """BASELINE config 5 with 2 % of the replicas re-placed (4,096 x 256 brokers x 16 racks, broker 255 on slot 255 with
    home replicas): 64 rounds of 2,048 from the initial base, bit for bit against the restatement, in two calls"""
    pb = m.synthetic_problem(*optima["cfg5_p02"]["args"])
    r = ref_lib.Ref(pb)
    assert r.W == 8 and (pb.cur == 255).any()
    bits, ld = r.init_base()
    sess = kao.Session(kao.Problem.from_fields(pb))
    for first, n in ((0, 32), (32, 32)):
        _, want = r.search(bits, ld, 0x5EED, first, n, 2048)
        got, _ = sess.search(0x5EED, first, n, 2048)
        assert_keys(got, want, ("round", first))
    reps, v, o, moves = sess.get_base()
    assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == m.evaluate(pb, reps)
    sess.close()
