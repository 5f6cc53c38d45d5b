"""The shared-memory search kernel (search_persistent_kernel, csrc/kao_kernels.cuh) over long walks: every plain shape
of up to 8,160 partitions, every runner (row-major, each column-major schedule, delta), from the initial base and
from damaged ones.  Inside one launch each winner patches state that only lives in shared memory (the row-major base
and its one-hot plane, the transposed, term, rack-field and shortfall planes, the count of invalid leaders, the
displaced lists); a patch that is wrong for one plane, one operation slot or one kind of winner only shows after
enough winners of that kind, so the walks are long (48 rounds of 1,024 candidates in two launches) or many (400
rounds of 4 candidates, each winner the best of three candidates and the identity).  Keys and final bases are held
to the restatement (oracle/kao_ref.c) and the exact model; after a walk a fresh session on the walked base must score
candidates as the walked session does, with the row-major per-round kernel reading the displaced lists the search
left in HBM.  The per-round entry points (kao_round_launch / kao_round_apply, kao_profile_rounds) run on the same
session between searches, and the round patience stops at is checked against its definition."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import optimizer as kopt
from kafka_assignment_optimizer_b200 import tuning
from oracle import model as m
from oracle import ref as oracle_ref
from problems import (C7_SHAPES, LAYOUT_SHAPES, SHAPES, emptied_base, moved_base, patience_stop,
                      with_saturating_violation)
from test_gpu_large_layouts import assert_keys, empty_rows
from test_gpu_layout_matrix import saturated_problem

pytestmark = pytest.mark.gpu

# shapes the named tables leave out: the compile-time 32-word form, the run-time word count above 32, the largest
# column-major row count, and saturated bases on the column-major evaluator (every saturated shape of problems.py
# is row-major only)
SMEM_EXTRA = {
    "cfg3": lambda: m.synthetic_problem(1000, 64, 8, 3),
    "p1100": lambda: m.synthetic_problem(1100, 64, 8, 3, remove=2),
    "cm_max": lambda: m.synthetic_problem(8160, 32, 4, 2, remove=1),
    "saturated_problem": lambda: saturated_problem(oracle_ref)[0],
    "sat_cm_cfg2": lambda: with_saturating_violation(LAYOUT_SHAPES["widecm_cfg2"]()),
    "sat_cm_cfg3_small": lambda: with_saturating_violation(LAYOUT_SHAPES["widecm_cfg3_small"]()),
}
ALL = {**SHAPES, **LAYOUT_SHAPES, **C7_SHAPES, **SMEM_EXTRA}
SATURATED = {"sat_cfg2", "sat_rack5_w4", "saturated_problem", "sat_cm_cfg2", "sat_cm_cfg3_small"}
ROUND = {"max_rows": 256, "w2_rows6000": 256, "cm_max": 256}     # the restatement scores every candidate in O(P)
KEYS = {"max_rows": 1024, "w2_rows6000": 1024, "cm_max": 1024}   # candidates of a rebuild check round
WALK, PROBE = 48, 400                                           # rounds of the long walk (two calls), the probe walk


def product(pb):
    return kao.Problem.from_fields(pb)


def t_words(P):
    """Partition words per slot of the column-major planes (kao_device.cuh: t_words of the padded row count)"""
    n = (P + 255) // 256 * 256 >> 5
    return (n + 31) & ~31 if n > 32 else n


def delta_fits(sess):
    try:
        sess.candidate_keys_delta(1, 0, 2, 0, 1)
    except kao.KaoError as e:
        assert "do not fit" in str(e), e
        return False
    return True


def runners(pb):
    """(name, column_major, schedule, delta) of every session configuration this shape runs: the row-major full
    search, each built column-major schedule where the layout allows it, the delta search where it fits"""
    sess = kao.Session(product(pb))
    out = [("row_major", False, None, False)]
    if sess.set_evaluator(True):
        for s in tuning.SCHEDULES:
            assert sess.set_schedule(*s), s
            out.append((tuning.schedule_name(s), True, s, False))
    if delta_fits(sess):
        out.append(("delta", False, None, True))
    sess.close()
    return out


def open_runner(pb, runner):
    _, cm, sched, _ = runner
    sess = kao.Session(product(pb))
    assert sess.set_evaluator(cm)
    if sched is not None:
        assert sess.set_schedule(*sched)
    return sess


def search(sess, runner, *args):
    return (sess.search_delta if runner[3] else sess.search)(*args)[0]


def bases(pb, r, name):
    reps = r.decode(*r.init_base())
    if name in SATURATED:
        return {"initial": reps}
    return {"initial": reps, "moved": moved_base(pb, reps, 6), "emptied": emptied_base(pb, reps, 5)}


def check_base(sess, pb, r, bits, ld, what):
    reps, v, o, moves = sess.get_base()
    assert (reps == r.decode(bits, ld)).all(), what
    assert (v, o) == r.evaluate(bits, ld) == m.evaluate(pb, reps), what
    assert moves == m.replica_moves(pb, reps), what
    return reps


# ---- long and probe walks, then a rebuilt session ---------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(ALL))
def test_long_and_probe_walks_from_every_base(ref_lib, name):
    pb = ALL[name]()
    assert pb.P <= 8160
    r = ref_lib.Ref(pb)
    run = runners(pb)
    size, ksize = ROUND.get(name, 1024), KEYS.get(name, 4096)
    if name.startswith("sat_cm"):
        assert any(cm for _, cm, _, _ in run), "a saturated base on the column-major evaluator"
    for what, start in bases(pb, r, name).items():
        seed = 0x5EED0 + len(what)
        # the restatement's walks, once for every runner
        bits, ld = r.encode(start)
        _, want_long = r.search(bits, ld, seed, 0, WALK, size)
        walked = (bits, ld)
        want_rebuild = {rnd: r.candidate_keys(bits, ld, seed, rnd, ksize, 0, ksize) for rnd in (WALK, WALK + 3)}
        pbits, pld = r.encode(start)
        _, want_probe = r.search(pbits, pld, seed ^ 0x77, 0, PROBE, 4)
        if name in SATURATED:                            # a saturated winner first
            assert r.unpack_key(want_long[0])[0] == (1 << (39 - r.obj_bits)) - 1
        for runner in run:
            tag = (what, runner[0])
            # long walk: two calls, the second restages the base, lists and planes from HBM
            sess = open_runner(pb, runner)
            sess.set_base(start)
            got = np.concatenate([search(sess, runner, seed, 0, WALK // 2, size),
                                  search(sess, runner, seed, WALK // 2, WALK - WALK // 2, size)])
            assert_keys(got, want_long, tag + ("long walk",))
            reps = check_base(sess, pb, r, *walked, tag + ("long walk",))
            if what == "emptied":
                assert empty_rows(reps) > 0             # leaders 0xFF: the invalid-leader count stays above 0
            # rebuild check: a fresh session on the walked base; the walked session's row-major keys come from the
            # per-round kernel on the displaced lists the search left in HBM
            fresh = open_runner(pb, runner)
            fresh.set_base(reps)
            for rnd, want in want_rebuild.items():
                for who, s in (("walked", sess), ("fresh", fresh)):
                    assert_keys(s.candidate_keys(seed, rnd, ksize, 0, ksize), want, tag + (who, rnd))
                    assert_keys(s.candidate_keys_delta(seed, rnd, ksize, 0, ksize), want, tag + (who, "delta", rnd))
            assert sess.set_evaluator(False)
            for rnd, want in want_rebuild.items():
                assert_keys(sess.candidate_keys(seed, rnd, ksize, 0, ksize), want, tag + ("walked row-major", rnd))
            fresh.close()
            sess.close()
            # probe walk: 400 rounds of three candidates and the identity, in one call
            sess = open_runner(pb, runner)
            sess.set_base(start)
            assert_keys(search(sess, runner, seed ^ 0x77, 0, PROBE, 4), want_probe, tag + ("probe walk",))
            check_base(sess, pb, r, pbits, pld, tag + ("probe walk",))
            sess.close()


# ---- every entry point on one session ------------------------------------------------------------------------------
@pytest.mark.parametrize("base", ["initial", "moved"])
@pytest.mark.parametrize("name", ["cfg2_rm2", "cfg3_small", "cfg3", "p1100", "w4_s16", "rf_up", "ragged"])
def test_entry_points_in_turn_on_one_session(ref_lib, name, base):
    """search, search_delta, round_launch / round_apply, search with each full evaluator, profile_rounds and search
    again on one session, with consecutive rounds of one seed: each per-round entry point reads the displaced lists the
    search before it left in HBM"""
    import torch

    pb = ALL[name]()
    r = ref_lib.Ref(pb)
    reps = r.decode(*r.init_base())
    start = reps if base == "initial" else moved_base(pb, reps, 6)
    bits, ld = r.encode(start)
    seed, size, first = 0xE17, 1024, 0
    sess = kao.Session(product(pb))
    sess.set_base(start)

    def step(n, call, what):
        """the session's call over the next n rounds (its keys, or None), then the restatement over the same rounds"""
        nonlocal first
        got = call(first, n)
        _, want = r.search(bits, ld, seed, first, n, size)
        if got is not None:
            assert_keys(got, want, what)
        first += n
        check_base(sess, pb, r, bits, ld, what)

    def rounds_by_shards(f, n):
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

    step(10, lambda f, n: sess.search(seed, f, n, size)[0], "1 search")
    step(10, lambda f, n: sess.search_delta(seed, f, n, size)[0], "2 search_delta")
    step(10, rounds_by_shards, "3 round_launch / round_apply")
    assert sess.set_evaluator(False)
    step(10, lambda f, n: sess.search(seed, f, n, size)[0], "4 row-major search")
    if sess.set_evaluator(True):
        assert sess.set_schedule(4, 0x22, 1024)
        step(10, lambda f, n: sess.search(seed, f, n, size)[0], "5 column-major search (4, 0x22, 1024)")
    step(5, lambda f, n: sess.profile_rounds(seed, f, n, size) and None, "6 profile_rounds")    # times, no keys
    step(10, lambda f, n: sess.search(seed, f, n, size)[0], "7 search")
    sess.close()


# ---- patience against its definition -------------------------------------------------------------------------------
def restatement_until_stop(r, bits, ld, seed, n, cap, size, chunk=100):
    keys = np.zeros(0, np.uint64)
    while len(keys) < cap:
        _, k = r.search(bits, ld, seed, len(keys), min(chunk, cap - len(keys)), size)
        keys = np.concatenate([keys, k])
        if patience_stop(keys, n) < len(keys):
            break
    stop = patience_stop(keys, n)
    return stop, keys[:stop]


@pytest.mark.parametrize("name", ["cfg2_rm2", "cfg3_small", "ragged", "widecm_cfg2", "planes8_w1", "sat_cm_cfg2"])
def test_patience_stops_where_its_definition_says(ref_lib, name):
    pb = ALL[name]()
    r = ref_lib.Ref(pb)
    reps = r.decode(*r.init_base())
    start = moved_base(pb, reps, 6)
    seed, size, cap = 0x9A7, 512, 2000
    for n in (5, 20):
        stop, want = restatement_until_stop(r, *r.encode(start), seed, n, cap, size)
        assert 0 < stop < cap, (n, stop)
        for runner in runners(pb):
            sess = open_runner(pb, runner)
            sess.set_base(start)
            sess.set_patience(n)
            got = search(sess, runner, seed, 0, cap, size)
            assert sess.last_rounds() == stop, (runner[0], n, sess.last_rounds(), stop)
            assert_keys(got[:stop], want, (runner[0], n))
            assert (got[stop:] == kopt.KEY_NONE).all(), runner[0]
            sess.close()
        stop0, _ = restatement_until_stop(r, *r.init_base(), seed, n, cap, size)
        res = kopt.solve(product(pb), seed=seed, rounds=cap, round_size=size, patience=n)
        assert res.rounds == stop0, (n, res.rounds, stop0)


# ---- what the matrix reaches ---------------------------------------------------------------------------------------
def test_the_walk_matrix_reaches_every_column_major_form(ref_lib):
    """Fails when an edit to the shape tables drops one of the kernel forms the walks above exist for"""
    reached = set()
    for name, f in sorted(ALL.items()):
        pb = f()
        sess = kao.Session(product(pb))
        cm = sess.set_evaluator(True)
        if cm:
            w, nw = sess.stats()["words_per_row"], t_words(pb.P)
            reached |= {"cm W=%d" % w, "cm 32 words" if nw == 32 else "cm run-time words"}
            if nw > 32:
                reached.add("cm run-time words above 32")
            if pb.P == 8160:
                reached.add("cm 8160 rows")
            if name.startswith("planes8_"):
                reached.add("8 term planes")
            if all(sess.set_schedule(*s) for s in tuning.SCHEDULES):
                reached.add("all schedules")
            if name not in SATURATED:
                r = ref_lib.Ref(pb)
                _, ld = r.encode(bases(pb, r, name)["emptied"])
                if (ld == 0xFF).any():
                    reached.add("cm invalid leaders")
        if name in SATURATED:
            r = ref_lib.Ref(pb)
            if r.evaluate(*r.init_base())[0] > (1 << (39 - r.obj_bits)) - 1:
                reached.add("saturated " + ("column-major" if cm else "row-major"))
        sess.close()
    want = {"cm W=1", "cm W=2", "cm 32 words", "cm run-time words", "cm run-time words above 32", "cm 8160 rows",
            "8 term planes", "all schedules", "cm invalid leaders", "saturated column-major", "saturated row-major"}
    assert want <= reached, sorted(want - reached)
