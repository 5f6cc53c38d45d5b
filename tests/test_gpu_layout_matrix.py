"""GPU parity on the evaluator layouts of tests/problems.py: LAYOUT_SHAPES (whole-word rack fields, general C7
bounds in wide rows, 12-bit packed entries, dense tables at every row width, weights above 12 bits, eight term
planes, saturated violation fields), column counts at the per-lane counter limit of 8192 padded rows, and a
delta search that starts from a saturated base.  Every call goes through the C ABI of libkao.so; the checkers
are the restatement (oracle/kao_ref.c) and the exact model (oracle/model.py)."""
import dataclasses

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import LAYOUT_SHAPES, with_12bit_weights

pytestmark = pytest.mark.gpu


def product(pb):
    return kao.Problem.from_fields(pb)


def evaluators(sess):
    """The full evaluators this session can run: row-major, and column-major where the layout allows it."""
    return [False] + ([True] if sess.set_evaluator(True) else [])


@pytest.mark.parametrize("name", sorted(LAYOUT_SHAPES))
def test_layout_keys_and_searches_vs_restatement(ref_lib, name):
    """candidate_keys (each full evaluator), candidate_keys_delta, search (each full evaluator) and
    search_delta against the restatement; the base a search ends on evaluates like the exact model."""
    pb = LAYOUT_SHAPES[name]()
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    sess = kao.Session(product(pb))
    for rnd, size, lo, n in [(1, 4096, 0, 4096), (6, 8192, 8192 - 500, 500)]:
        want = r.candidate_keys(bits, ld, 0x1A7, rnd, size, lo, n)
        for cm in evaluators(sess):
            assert sess.set_evaluator(cm)
            got = sess.candidate_keys(0x1A7, rnd, size, lo, n)
            bad = np.flatnonzero(want != got)
            assert bad.size == 0, (cm, rnd, int(bad[0]), r.unpack_key(want[bad[0]]), r.unpack_key(got[bad[0]]))
        assert (sess.candidate_keys_delta(0x1A7, rnd, size, lo, n) == want).all()
    runs = [("full", cm) for cm in evaluators(sess)] + [("delta", False)]
    sess.close()
    _, want = r.search(bits, ld, 0x51, 0, 6, 2000)
    for mode, cm in runs:
        sess = kao.Session(product(pb))
        assert sess.set_evaluator(cm)
        got, _ = (sess.search_delta if mode == "delta" else sess.search)(0x51, 0, 6, 2000)
        assert (got == want).all(), (mode, cm)
        reps, v, o, moves = sess.get_base()
        assert (reps == r.decode(bits, ld)).all()
        assert (v, o) == m.evaluate(pb, reps) and moves == m.replica_moves(pb, reps)
        sess.close()


@pytest.mark.parametrize("name", sorted(LAYOUT_SHAPES))
def test_layout_explicit_evaluation_and_solve(name):
    """kao_eval on random, short-row and duplicate-broker assignments equals the exact model; kao_solve's answer
    evaluates as it says."""
    pb = LAYOUT_SHAPES[name]()
    rng = np.random.RandomState(5)
    cands = np.stack([np.stack([rng.choice(pb.B, size=pb.RF, replace=False) for _ in range(pb.P)]) for _ in range(9)])
    cands = cands.astype(np.int32)
    cands[1::3, rng.randint(pb.P), -1] = -1
    if pb.RF > 1:
        cands[2::3, 0, 1] = cands[2::3, 0, 0]
    v, o = kopt.evaluate(product(pb), cands)
    assert [(int(a), int(b)) for a, b in zip(v, o)] == [m.evaluate(pb, c) for c in cands]
    res = kopt.solve(product(pb), seed=7, rounds=24, round_size=2048)
    assert (res.violation, res.objective) == m.evaluate(pb, res.replicas)
    assert res.moves == m.replica_moves(pb, res.replicas)


# ---- column counts at the per-lane counter limit -------------------------------------------------
# A lane of the row-major evaluator takes 4 consecutive rows of every 128-row tile: at 8192 padded rows
# (P 7937..8160) the first lanes hold up to 256 real rows, one more than five high counter planes count.
def concentrated_bases(P):
    return {"every partition on brokers 0 and 1": np.tile(np.array([0, 1], np.int32), (P, 1)),
            "every partition led from broker 0": np.stack([[0, 1 + p % 14] for p in range(P)]).astype(np.int32)}


@pytest.mark.parametrize("P", [8065, 8068, 8100, 8160])
def test_column_counts_at_the_per_lane_counter_limit(ref_lib, P):
    pb = m.synthetic_problem(P, 16, 4, 2, remove=1)
    r = ref_lib.Ref(pb)
    bases = concentrated_bases(P)
    v, o = kopt.evaluate(product(pb), np.stack(list(bases.values())))
    sess = kao.Session(product(pb))
    for i, (what, reps) in enumerate(bases.items()):
        want_eval = m.evaluate(pb, reps)
        assert (int(v[i]), int(o[i])) == want_eval, what
        bits, ld = r.encode(reps)
        sess.set_base(reps)
        assert sess.get_base()[1:3] == want_eval, what
        want = r.candidate_keys(bits, ld, 0x8160, 4, 1024, 0, 1024)
        for cm in evaluators(sess):
            assert sess.set_evaluator(cm)
            assert (sess.candidate_keys(0x8160, 4, 1024, 0, 1024) == want).all(), (what, cm)
        assert (sess.candidate_keys_delta(0x8160, 4, 1024, 0, 1024) == want).all(), what
        _, want = r.search(bits, ld, 0xC0C0, 0, 3, 1024)
        for search in ("search", "search_delta"):           # row-major evaluator selected: full and delta search
            assert sess.set_evaluator(False)
            sess.set_base(reps)
            assert (getattr(sess, search)(0xC0C0, 0, 3, 1024)[0] == want).all(), (what, search)
            assert (sess.get_base()[0] == r.decode(bits, ld)).all()
    sess.close()


# ---- delta search from a saturated base ----------------------------------------------------------
def saturated_problem(ref_lib, excess=7):
    """12-bit packed entries on config 2 with replica lower bounds raised on three brokers until the initial base's violation is the
    violation field's cap + excess: round 0's winner is a saturated key, the later ones are not."""
    pb = with_12bit_weights(m.synthetic_problem(256, 32, 4, 3, remove=2), 41)
    r = ref_lib.Ref(pb)
    reps = r.decode(*r.init_base())
    cap = (1 << (39 - r.obj_bits)) - 1
    need = cap + excess - m.evaluate(pb, reps)[0]
    cnt = np.bincount(reps[reps >= 0], minlength=pb.B)
    lo = pb.rep_lo.copy()
    for b in range(3):                        # below its lower bound a broker adds lo - count to the violation
        start = max(int(cnt[b]), int(lo[b]))
        add = min(need, 65535 - start)
        lo[b] = start + add
        need -= add
    assert need == 0
    return dataclasses.replace(pb, rep_lo=lo, rep_hi=np.maximum(pb.rep_hi, lo)), cap


def test_delta_search_leaves_a_saturated_base_like_the_full_search(ref_lib):
    """The delta kernel re-evaluates its base in full after a saturated winning key; its trajectory out of
    saturation equals the restatement's and the full-evaluation search's, and so does the round patience
    stops it at."""
    pb, cap = saturated_problem(ref_lib)
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    assert r.evaluate(bits, ld)[0] > cap
    _, want = r.search(bits, ld, 0x5A7, 0, 10, 2000)
    viols = [r.unpack_key(k)[0] for k in want]
    assert viols[0] == cap and max(viols[1:]) < cap, viols           # a saturated winner, then none
    for search in ("search", "search_delta"):
        sess = kao.Session(product(pb))
        got, _ = getattr(sess, search)(0x5A7, 0, 10, 2000)
        assert (got == want).all(), search
        reps, v, o, _ = sess.get_base()
        assert (reps == r.decode(bits, ld)).all() and (v, o) == m.evaluate(pb, reps)
        sess.close()
    stops = {}
    for search in ("search", "search_delta"):
        sess = kao.Session(product(pb))
        sess.set_patience(2)
        got, _ = getattr(sess, search)(0x5A7, 0, 200, 2000)
        stops[search] = sess.last_rounds()
        assert 0 < stops[search] < 200
        assert (got[:stops[search]] == r.search(*r.init_base(), 0x5A7, 0, stops[search], 2000)[1]).all(), search
        sess.close()
    assert stops["search"] == stops["search_delta"]
