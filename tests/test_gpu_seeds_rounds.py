"""64-bit seeds, late and wrapping round numbers, restarts, and searches after or beside other sessions, on the GPU.
A candidate is a pure function of (base, seed, round, idx) (docs/MODEL.md §5) and a trajectory depends on nothing else:
not on how its rounds are split into calls, nor on what ran before (§6).  Every search path built for sm_90a is held
bit for bit to its restatement (oracle/kao_ref.c, tests/topics_ref, tests/rf_ref) at every (seed, first round) pair of
problems.SEEDS x problems.ROUNDS: the shared-memory runners (row-major, both column-major schedules, delta) at W = 1, 2,
4 and 8, the tensor-core body with sorted batches and with a CTA share beyond its list, the HBM path above 8,160
partitions and topic and replication sessions, kao_round_launch / kao_round_apply, and calls chained across 2^16, 2^24
and 2^32 (a call runs rounds first_round + i mod 2^32).  kao_solve's restarts (seed + r * 0x9E3779B97F4A7C15 mod 2^64,
each from the initial base, the best by (violation, -objective), the lowest restart on a tie) are held to
problems.ref_solve on every shared-memory configuration, with and without patience, and so are kao_solve_fixed, a
topic solve and kao-cli.  Sessions of the same buffer sizes run and are destroyed first (the device and pinned buffer
pools recycle them uncleared), two sessions alternate their calls, and four host threads solve at once."""
import copy
import json
import os
import subprocess
import threading

import numpy as np
import pytest

import fixed_ref as F
import kafka_assignment_optimizer_b200 as kao
import topics_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from kafka_assignment_optimizer_b200 import tuning
from oracle import model as m
from problems import (LARGE_SHAPES, PHI, ROUNDS, RF_SHAPES, SEEDS, SHAPES, WRAP, emptied_base, mixed_rows, moved_base,
                      ref_solve, round_at, with_12bit_weights, with_saturating_bounds)
from test_gpu_home255 import all_runners, check_end
from test_gpu_large_layouts import assert_keys
from test_gpu_smem_walks import check_base, open_runner, runners, search
from test_host import README_CURRENT

pytestmark = pytest.mark.gpu

CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kafka_assignment_optimizer_b200",
                   "kao-cli")
# W = 1 and 2 on every column-major schedule, W = 4 and 8 row-major and delta, RF 8 column-major
SMEM = {"cfg2": SHAPES["cfg2"], "cfg3_small": SHAPES["cfg3_small"], "w4_s16": SHAPES["w4_s16"],
        "w8_s16": SHAPES["w8_s16"], "rf8_cm": RF_SHAPES["rf8_cm"]}
SIZE, WALK = 1024, 8                # candidates of a key round and of a walk round; rounds of a walk
PAIRS = [(sn, s, rn, rnd) for sn, s in sorted(SEEDS.items()) for rn, rnd in sorted(ROUNDS.items())]
HIGH = [SEEDS[n] for n in ("all_ones", "high_word", "goldens_low", "2^32", "restart1_of_0")]


def product(pb):
    return kao.Problem.from_fields(pb)


def start_base(pb, r):
    return moved_base(pb, r.decode(*r.init_base()), 6)


def ref_walks(r, start, size, walk=WALK):
    """(seed, first round) -> (round keys of a walk of `walk` rounds from `start`, walked (bits, ld))"""
    out = {}
    for sn, s, rn, rnd in PAIRS:
        bits, ld = r.encode(start)
        _, keys = r.search(bits, ld, s, rnd, walk, size)
        out[sn, rn] = keys, (bits, ld)
    return out


# ---- round keys and walks at every (seed, round) pair --------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(SMEM))
def test_keys_and_walks_on_every_runner_at_every_seed_and_round(ref_lib, name):
    """From a damaged base: the keys of round `first` and a walk of 8 rounds from it, in one call, on every runner"""
    pb = SMEM[name]()
    r = ref_lib.Ref(pb)
    start = start_base(pb, r)
    bits, ld = r.encode(start)
    want_keys = {(sn, rn): r.candidate_keys(bits, ld, s, rnd, SIZE, 0, SIZE) for sn, s, rn, rnd in PAIRS}
    walks = ref_walks(r, start, SIZE)
    run = runners(pb)
    assert len(run) == (4 if r.W <= 2 else 2), [x[0] for x in run]
    for runner in run:
        sess = open_runner(pb, runner)
        sess.set_base(start)
        for sn, s, rn, rnd in PAIRS:
            keys = (sess.candidate_keys_delta if runner[3] else sess.candidate_keys)(s, rnd, SIZE, 0, SIZE)
            assert_keys(keys, want_keys[sn, rn], (runner[0], sn, rn))
        for sn, s, rn, rnd in PAIRS:
            sess.set_base(start)
            want, end = walks[sn, rn]
            assert_keys(search(sess, runner, s, rnd, WALK, SIZE), want, (runner[0], sn, rn, "walk"))
            check_base(sess, pb, r, *end, (runner[0], sn, rn, "walk"))
        sess.close()


def test_sorted_batches_and_a_share_beyond_the_list_at_late_rounds(ref_lib):
    """The default tensor-core schedule on the headline layout: rounds of 2^16 candidates (every CTA sorts a share of
    about 500) at every seed, at a cycle round above 2^31 and across 2^32; then rounds of 2^24 (a share beyond any list,
    walked unsorted) held to the restatement on windows and to the popcount schedule, which does not sort, in full"""
    pb = m.synthetic_problem(1000, 64, 8, 3)
    r = ref_lib.Ref(pb)
    start = start_base(pb, r)
    bits, ld = r.encode(start)
    sess = kao.Session(product(pb))
    assert sess.stats()["schedule"] == tuning.DEFAULT_SCHEDULE == (1, 0x300, 512)
    sess.set_base(start)
    size = 1 << 16
    for sn, s in sorted(SEEDS.items()):
        for rnd in (ROUNDS["2^31+3"], WRAP + 1):
            assert_keys(sess.candidate_keys(s, rnd, size, 0, size), r.candidate_keys(bits, ld, s, rnd, size, 0, size),
                        (sn, rnd))
    s = SEEDS["all_ones"]
    wbits, wld = r.encode(start)
    _, want = r.search(wbits, wld, s, WRAP, 4, size)
    assert_keys(sess.search(s, WRAP, 4, size)[0], want, "sorted walk")
    check_base(sess, pb, r, wbits, wld, "sorted walk")
    pop = kao.Session(product(pb))
    assert pop.set_schedule(4, 0x22, 1024)
    big = 1 << 24
    for sess_ in (sess, pop):
        sess_.set_base(start)
    for rnd in (WRAP + 1, ROUNDS["2^24"]):
        got = sess.candidate_keys(s, rnd, big, 0, big)
        assert np.array_equal(got, pop.candidate_keys(s, rnd, big, 0, big)), rnd
        for lo in (0, big // 2 + 77, big - 2048):
            assert_keys(got[lo:lo + 2048], r.candidate_keys(bits, ld, s, rnd, big, lo, 2048), (rnd, lo))
    ka, kb = sess.search(s, WRAP, 4, big)[0], pop.search(s, WRAP, 4, big)[0]
    assert np.array_equal(ka, kb) and np.array_equal(sess.get_base()[0], pop.get_base()[0])
    # each round's winner is the restatement's candidate at its index, with the restatement's key, and the walked base
    # is the restatement's base after those winners (the minimum over 2^24 is the popcount schedule's, above)
    for i, k in enumerate(ka):
        rnd, idx = round_at(WRAP, i), int(k) & 0xFFFFFF
        assert_keys(np.array([k]), r.candidate_keys(bits, ld, s, rnd, big, idx, 1), ("2^24 winner", i))
        bits, ld = r.gen(bits, ld, s, rnd, idx, big)
    check_base(sess, pb, r, bits, ld, "2^24 walk")
    sess.close()
    pop.close()


# ---- the HBM path ----------------------------------------------------------------------------------------------------------
def test_hbm_plain_session_at_every_seed_and_round(ref_lib):
    """8,200 partitions: delta keys at every pair, and a walk of 8 rounds from 2^32 - 2 at every seed in two calls"""
    pb = LARGE_SHAPES["big_rf_up"]()
    r = ref_lib.Ref(pb)
    start = start_base(pb, r)
    bits, ld = r.encode(start)
    sess = kao.Session(product(pb))
    sess.set_base(start)
    for sn, s, rn, rnd in PAIRS:
        assert_keys(sess.candidate_keys_delta(s, rnd, 512, 0, 512), r.candidate_keys(bits, ld, s, rnd, 512, 0, 512),
                    (sn, rn))
    for sn, s in sorted(SEEDS.items()):
        sess.set_base(start)
        wbits, wld = r.encode(start)
        _, want = r.search(wbits, wld, s, WRAP, WALK, 512)
        got = np.concatenate([sess.search_delta(s, WRAP, 3, 512)[0], sess.search_delta(s, 1, WALK - 3, 512)[0]])
        assert_keys(got, want, (sn, "walk"))
        check_base(sess, pb, r, wbits, wld, (sn, "walk"))
    sess.close()


@pytest.mark.parametrize("kind", ["hbm", "topics", "replication"])
def test_hbm_topic_and_replication_sessions_at_every_seed_and_round(ref_lib, kind):
    """w4_s16 on the HBM kernels (a loose topic), with five interleaved topics and with mixed per-partition rows:
    keys at every pair and a walk of 8 rounds from every first round"""
    pb = SHAPES["w4_s16"]()
    run = all_runners(pb, ref_lib)[kind]
    r = run.r
    start = r.decode(*r.init_base())
    bits, ld = r.encode(start)
    walks = ref_walks(r, start, 512)
    sess = run.open()
    sess.set_base(start)
    for sn, s, rn, rnd in PAIRS:
        assert_keys(run.keys(sess, s, rnd, 512, 0, 512), r.candidate_keys(bits, ld, s, rnd, 512, 0, 512), (kind, sn, rn))
    for sn, s, rn, rnd in PAIRS:
        sess.set_base(start)
        want, end = walks[sn, rn]
        assert_keys(run.search(sess, s, rnd, WALK, 512), want, (kind, sn, rn, "walk"))
        check_end(sess, run, *end, (kind, sn, rn, "walk"))
    sess.close()


# ---- chained calls and the per-round entry points ------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cfg2", "cfg3_small", "w4_s16"])
def test_chained_calls_across_2_16_2_24_and_2_32_equal_one_call(ref_lib, name):
    """8 rounds from c - 3 for c = 2^16, 2^24, 2^32: one call, and two calls split at c, on every runner; then on one
    session search (c - 3 .. c - 1), round_launch / round_apply in three shards (c, c + 1) and search_delta (c + 2 ..
    c + 4)"""
    import torch

    pb = SMEM[name]()
    r = ref_lib.Ref(pb)
    start = start_base(pb, r)
    s = SEEDS["high_word"]
    for c in (1 << 16, 1 << 24, 1 << 32):
        first = c - 3
        bits, ld = r.encode(start)
        _, want = r.search(bits, ld, s, first, WALK, SIZE)
        for runner in runners(pb):
            for split in (False, True):
                tag = (c, runner[0], split)
                sess = open_runner(pb, runner)
                sess.set_base(start)
                got = (np.concatenate([search(sess, runner, s, first, 3, SIZE),
                                       search(sess, runner, s, c % (1 << 32), WALK - 3, SIZE)]) if split
                       else search(sess, runner, s, first, WALK, SIZE))
                assert_keys(got, want, tag)
                check_base(sess, pb, r, bits, ld, tag)
                sess.close()
        sess = kao.Session(product(pb))
        sess.set_base(start)
        key = torch.empty(1, dtype=torch.int64, device="cuda")
        got = list(sess.search(s, first, 3, SIZE)[0])
        for i in (3, 4):
            rnd = round_at(first, i)
            key.fill_(kopt.KEY_NONE)
            for lo, hi in [(0, 300), (300, 301), (301, SIZE)]:
                sess.round_launch(s, rnd, SIZE, lo, hi, key.data_ptr())
            sess.round_apply(s, rnd, SIZE, key.data_ptr())
            torch.cuda.synchronize()
            got.append(int(key.item()) & 0xFFFFFFFFFFFFFFFF)
        got += list(sess.search_delta(s, round_at(first, 5), 3, SIZE)[0])
        assert_keys(np.array(got, np.uint64), want, (c, "entry points"))
        check_base(sess, pb, r, bits, ld, (c, "entry points"))
        sess.close()


# ---- sessions that ran before, and sessions side by side ---------------------------------------------------------------------
def run_other_sessions(pb, ref_lib):
    """Sessions of pb's buffer sizes with other content, each searched, then destroyed: other weights, saturated bounds,
    a damaged base, a topic session and a replication session.  Their device and pinned buffers go back to the pools
    uncleared, and the next session of these sizes gets them."""
    r = ref_lib.Ref(pb)
    damaged = emptied_base(pb, r.decode(*r.init_base()), 5)
    for other, base in ((with_12bit_weights(pb, 61), None), (with_saturating_bounds(pb), None), (pb, damaged)):
        sess = kao.Session(product(other))
        if base is not None:
            sess.set_base(base)
        sess.search(0xBAD5EED, 7, 6, 512)
        sess.search_delta(0xBAD5EED, 13, 6, 512)
        sess.close()
    tpb = copy.copy(pb)
    tpb.topics = [("t%d" % (p % 7), p) for p in range(pb.P)]
    kp = product(pb)
    kp.replication = mixed_rows(kp, 0xBAD)
    for sess in (kao.Session(product(tpb), topics=kao.topic_rows(product(tpb))), kao.Session(kp)):
        sess.search_delta(0xBAD5EED, 3, 6, 512)
        sess.close()


SOLVE = dict(round_size=512)
ROUNDS_NO_PATIENCE, ROUNDS_CAP, PATIENCE = 6, 60, 4
CONFIGS = {"default": {}, "row_major": dict(row_major=True), "delta": dict(delta=True), "popcount": {}}
_want = {}


def _ref(ref_lib, name, seed, restarts, patience):
    """problems.ref_solve of SHAPES[name], cached over the configurations"""
    k = (name, seed, restarts, patience)
    if k not in _want:
        rounds = ROUNDS_CAP if patience else ROUNDS_NO_PATIENCE
        _want[k] = ref_solve(ref_lib.Ref(SHAPES[name]()), seed, restarts, rounds, SOLVE["round_size"], patience)
    return _want[k]


def assert_solved(res, want, size, what):
    assert (res.violation, res.objective) == (want["violation"], want["objective"]), what
    assert np.array_equal(res.replicas, want["replicas"]) and res.key == want["key"], what
    assert res.rounds == want["rounds"] and res.n_candidates == want["rounds"] * size, what


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_solve_restarts_equal_the_restatement_at_high_seeds(ref_lib, monkeypatch, config):
    """cfg2_rm2 (column-major where allowed, restarts that end apart): 1 to 5 restarts from seeds with the high word set,
    with and without patience, after sessions of the same sizes ran; the popcount schedule through KAO_SCHEDULE, which
    each session reads when it is created"""
    pb = SHAPES["cfg2_rm2"]()
    run_other_sessions(pb, ref_lib)
    if config == "popcount":
        monkeypatch.setenv("KAO_SCHEDULE", "4,22,1024")
    sess = kao.Session(product(pb))
    st = sess.stats()
    sess.close()
    assert st["column_major"] and st["schedule"] == ((4, 0x22, 1024) if config == "popcount" else tuning.DEFAULT_SCHEDULE)
    outcomes = set()
    for restarts, seed in zip(range(1, 6), HIGH):
        for patience in (0, PATIENCE):
            want = _ref(ref_lib, "cfg2_rm2", seed, restarts, patience)
            outcomes.add(want["restart"])
            res = kopt.solve(product(pb), seed=seed, rounds=ROUNDS_CAP if patience else ROUNDS_NO_PATIENCE,
                             restarts=restarts, patience=patience, **SOLVE, **CONFIGS[config])
            assert_solved(res, want, SOLVE["round_size"], (config, restarts, hex(seed), patience))
            if patience:
                assert want["rounds"] < restarts * ROUNDS_CAP, (restarts, hex(seed))
    assert len(outcomes) >= 3, outcomes             # restarts other than the first win


@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_on_a_tie_the_lowest_restart_wins(ref_lib, monkeypatch, config):
    """The README example at 16 rounds of 256: all three restarts reach the optimum 58 in other assignments; kao_solve
    returns restart 0's"""
    if config == "popcount":
        monkeypatch.setenv("KAO_SCHEDULE", "4,22,1024")
    pb = SHAPES["readme"]()
    r = ref_lib.Ref(pb)
    seed = SEEDS["high_word"]
    ends = []
    for k in range(3):
        bits, ld = r.init_base()
        r.search(bits, ld, (seed + k * PHI) % (1 << 64), 0, 16, 256)
        ends.append((r.evaluate(bits, ld), r.decode(bits, ld)))
    assert ends[0][0] == ends[1][0] == ends[2][0] == (0, 58)
    assert not np.array_equal(ends[0][1], ends[1][1]) and not np.array_equal(ends[0][1], ends[2][1])
    want = ref_solve(r, seed, 3, 16, 256)
    assert want["restart"] == 0
    res = kopt.solve(product(pb), seed=seed, rounds=16, round_size=256, restarts=3, **CONFIGS[config])
    assert_solved(res, want, 256, config)


def test_solve_fixed_and_topic_solve_restarts_at_high_seeds(ref_lib):
    """kao_solve_fixed (half of cfg2_rm2 fixed) is the restatement's solve of the reduced problem; a topic solve is
    tests/topics_ref's, both with three restarts from a seed with the high word set"""
    seed = SEEDS["goldens_low"]
    pb = product(SHAPES["cfg2_rm2"]())
    fx = F.random_mask(pb, 0x5EED, share=0.5)
    assert fx.any() and not fx.all()
    red = F.reduce(pb, fx)
    run_other_sessions(red.pb, ref_lib)
    got = kopt.solve(_fixed(pb, fx), seed=seed, rounds=8, round_size=1024, restarts=3)
    want = ref_solve(ref_lib.Ref(red.pb), seed, 3, 8, 1024)
    assert np.array_equal(got.replicas[red.searched], want["replicas"]) and got.key == want["key"]
    assert (got.violation, got.objective) == (want["violation"] + red.V0, want["objective"] + red.O0)
    assert got.rounds == want["rounds"]
    tpb = SHAPES["cfg3_small"]()
    tpb.topics = [("t%d" % (p % 5), p) for p in range(tpb.P)]
    tr = kao.topic_rows(product(tpb))
    want = ref_solve(topics_ref.TRef(tpb, tr), seed, 3, 8, 1024)
    res = kopt.solve(product(tpb), seed=seed, rounds=8, round_size=1024, restarts=3, topics=tr)
    assert_solved(res, want, 1024, "topics")


def _fixed(pb, fx):
    import dataclasses

    return dataclasses.replace(pb, fixed=fx)


@pytest.mark.parametrize("seed", ["0xDEADBEEF00C0FFEE", "18446744073709551615"])
def test_cli_with_a_high_seed_and_restarts_is_the_python_solve(tmp_path, seed):
    f = tmp_path / "current.json"
    f.write_text(README_CURRENT)
    brokers, racks = ",".join(map(str, range(19))), ",".join("%d:%s" % (b, "b" if b % 2 else "a") for b in range(20))
    p = subprocess.run([CLI, "--assignment", str(f), "--brokers", brokers, "--racks", racks, "--rounds", "16",
                        "--round-size", "256", "--restarts", "3", "--seed", seed], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    doc, res = kao.AssignmentOptimizer(seed=int(seed, 0), rounds=16, round_size=256, restarts=3).optimize(
        README_CURRENT, brokers, racks)
    assert json.loads(p.stdout) == doc and res.feasible


def test_two_sessions_with_alternating_calls_follow_their_own_trajectories(ref_lib):
    """Two sessions of one problem (the same buffer sizes), one on the tensor-core default and one delta, from
    different bases and seeds: their calls of 3 rounds alternate across 2^32"""
    pb = SHAPES["cfg2_rm2"]()
    run_other_sessions(pb, ref_lib)
    r = ref_lib.Ref(pb)
    init = r.decode(*r.init_base())
    plan = {"a": (init, SEEDS["all_ones"], False), "b": (moved_base(pb, init, 6), SEEDS["restart1_of_0"], True)}
    state, sess = {}, {}
    for k, (start, s, delta) in plan.items():
        state[k] = r.encode(start)
        sess[k] = kao.Session(product(pb))
        sess[k].set_base(start)
    first = WRAP - 5
    for call in range(4):
        for k, (start, s, delta) in plan.items():
            _, want = r.search(*state[k], s, round_at(first, 3 * call), 3, SIZE)
            got = (sess[k].search_delta if delta else sess[k].search)(s, round_at(first, 3 * call), 3, SIZE)[0]
            assert_keys(got, want, (k, call))
    for k in plan:
        check_base(sess[k], pb, r, *state[k], k)
        sess[k].close()


# ---- four host threads ------------------------------------------------------------------------------------------------
def _thread_problems():
    """name -> (problem, solve options): column-major, delta, topic rows, fixed rows with the LP bound"""
    cm = product(SHAPES["cfg2_rm2"]())
    tpb = SHAPES["cfg3_small"]()
    tpb.topics = [("t%d" % (p % 5), p) for p in range(tpb.P)]
    kt = product(tpb)
    fx = F.random_mask(cm, 0xF1, share=0.5)
    common = dict(rounds=12, round_size=1024, restarts=2)
    return {"column_major": (cm, dict(common, seed=SEEDS["all_ones"])),
            "delta": (product(SHAPES["cfg3_small"]()), dict(common, seed=SEEDS["high_word"], delta=True)),
            "topics": (kt, dict(common, seed=SEEDS["goldens_low"], topics=kao.topic_rows(kt))),
            "fixed_lp": (_fixed(cm, fx), dict(common, seed=SEEDS["2^32"], tight_bound=True, lp_bound=True))}


def test_four_threads_solving_at_once_get_the_serial_results():
    """kao_solve from four host threads at once (as /submit on a ThreadingHTTPServer does); the kernels all go to the
    legacy default stream, so the device work serialises while the host work interleaves"""
    probs = _thread_problems()
    fields = ("objective", "violation", "moves", "feasible", "key", "n_candidates", "rounds", "objective_bound", "optimal")
    serial = {k: kopt.solve(pb, **kw) for k, (pb, kw) in probs.items()}
    out, errors = {}, []
    go = threading.Barrier(len(probs), timeout=20)

    def work(k):
        try:
            go.wait()
            out[k] = kopt.solve(probs[k][0], **probs[k][1])
        except Exception as e:              # reported below, on the test's thread
            errors.append((k, repr(e)))

    threads = [threading.Thread(target=work, args=(k,), daemon=True) for k in probs]
    for t in threads:
        t.start()
    for t in threads:
        t.join(60)
    assert not any(t.is_alive() for t in threads) and not errors, errors
    for k in probs:
        for f in fields:
            assert getattr(out[k], f) == getattr(serial[k], f), (k, f)
        assert np.array_equal(out[k].replicas, serial[k].replicas), k
    assert serial["fixed_lp"].objective_bound > 0
