"""Evaluator layouts beyond the default weights and bounds, on the engine's own device code under the warp
emulator (tests/emu): whole-word rack fields, general C7 bounds in wide rows, packed entries with 12-bit
weights, dense tables at every row width, weights above 12 bits, eight term planes, saturated violation
fields (tests/problems.py: LAYOUT_SHAPES), and column counts at the per-lane counter limit of 8192 padded
rows.  Every key, evaluation and trajectory is checked against the restatement (oracle/kao_ref.c) and the
exact model (oracle/model.py)."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from oracle import model as m
from problems import LAYOUT_SHAPES, SHAPES


@pytest.fixture(scope="module")
def emu():
    import emu as emu_mod

    emu_mod.lib()
    return emu_mod


def product(pb):
    return kao.Problem.from_fields(pb)


def random_assignments(pb, rng, n):
    """Random replica lists; every third one has a short row (C1), every third + 1 a duplicate broker."""
    out = []
    for i in range(n):
        reps = np.stack([rng.choice(pb.B, size=pb.RF, replace=False) for _ in range(pb.P)]).astype(np.int32)
        if i % 3 == 1:
            reps[rng.randint(pb.P), -1] = -1
        if i % 3 == 2 and pb.RF > 1:
            p = rng.randint(pb.P)
            reps[p, 1] = reps[p, 0]
        out.append(reps)
    return out


@pytest.mark.parametrize("name", sorted(LAYOUT_SHAPES))
def test_layout_keys_evaluations_and_trajectories(emu, ref_lib, name):
    """Row-major, column-major (where the layout allows it: forms 1, 5 and 6) and delta keys equal the
    restatement's, from the initial base and from a random one; explicit evaluations equal the exact model;
    a 3-round search walks the restatement's trajectory."""
    pb = LAYOUT_SHAPES[name]()
    r = ref_lib.Ref(pb)
    sess = emu.EmuSession(product(pb))
    assert sess.config()["W"] == r.W
    forms = [0] + ([1, 5, 6] if sess.set_evaluator(1) else [])
    rng = np.random.RandomState(17)
    bits, ld = r.init_base()
    for it, reps in enumerate([None] + random_assignments(pb, rng, 2)):
        if reps is not None:
            sess.set_base(reps)
            bits, ld = r.encode(reps)
        got_reps, v, o, _ = sess.get_base()           # the identity candidate's key: a violation field may saturate
        assert (got_reps == r.decode(bits, ld)).all() and r.evaluate(bits, ld) == m.evaluate(pb, got_reps)
        assert (v, o) == r.unpack_key(r.pack_key(*m.evaluate(pb, got_reps), 0))[:2]
        for rnd, size, lo, n in [(1 + it, 4096, 4096 - 40, 40), (9, 256, 0, 40)]:
            want = r.candidate_keys(bits, ld, 0x1A7 + it, rnd, size, lo, n)
            for form in forms:
                assert sess.set_evaluator(form)
                got = sess.candidate_keys(0x1A7 + it, rnd, size, lo, n)
                bad = np.flatnonzero(want != got)
                assert bad.size == 0, (form, rnd, int(bad[0]), r.unpack_key(want[bad[0]]), r.unpack_key(got[bad[0]]))
            delta = sess.candidate_keys(0x1A7 + it, rnd, size, lo, n, delta=True)
            assert (delta == want).all(), ("delta", rnd, r.unpack_key(want[0]), r.unpack_key(delta[0]))
    cands = random_assignments(pb, rng, 6)
    v, o = sess.evaluate(np.stack(cands))
    for i, reps in enumerate(cands):
        assert (int(v[i]), int(o[i])) == m.evaluate(pb, reps), i
    bits, ld = r.init_base()
    sess.set_base(r.decode(bits, ld))
    _, want = r.search(bits, ld, 0xBEEF, 0, 3, 300)
    for form in forms[-1:]:                           # the last form: row-major, or a column-major one
        assert sess.set_evaluator(form)
        assert (sess.search(0xBEEF, 0, 3, 300) == want).all()
    assert (sess.get_base()[0] == r.decode(bits, ld)).all()
    sess.close()


def test_layout_regimes_are_what_their_names_say(emu):
    """Eight term planes with the widest cost field, and violations beyond the violation field."""
    from kafka_assignment_optimizer_b200.optimizer import key_obj_bits

    pb = LAYOUT_SHAPES["planes8_w1"]()
    assert key_obj_bits(product(pb)) == 24
    assert len(np.unique(pb.wF[pb.wF > 0])) + len(np.unique((pb.wL.astype(int) - pb.wF)[pb.wL > pb.wF])) == 8
    for name in ("sat_cfg2", "sat_rack5_w4"):
        pb = LAYOUT_SHAPES[name]()
        sess = emu.EmuSession(product(pb))
        assert sess.evaluate(sess.get_base()[0][None])[0][0] > (1 << (39 - key_obj_bits(product(pb)))) - 1, name
        sess.close()


# ---- column counts at the per-lane counter limit -------------------------------------------------
# A lane of the row-major evaluator takes 4 consecutive rows of every 128-row tile: at 8192 padded rows
# (P 7937..8160) the first lanes hold up to 256 real rows, one more than five high counter planes count.
@pytest.mark.parametrize("P", [8065, 8068, 8100, 8160])
def test_column_counts_at_the_per_lane_counter_limit(emu, ref_lib, P):
    pb = m.synthetic_problem(P, 16, 4, 2, remove=1)
    r = ref_lib.Ref(pb)
    sess = emu.EmuSession(product(pb))
    bases = {"every partition on brokers 0 and 1": np.tile(np.array([0, 1], np.int32), (P, 1)),
             "every partition led from broker 0": np.stack([[0, 1 + p % 14] for p in range(P)]).astype(np.int32)}
    v, o = sess.evaluate(np.stack(list(bases.values())))
    for i, (what, reps) in enumerate(bases.items()):
        want_eval = m.evaluate(pb, reps)
        assert (int(v[i]), int(o[i])) == want_eval, what
        bits, ld = r.encode(reps)
        assert r.evaluate(bits, ld) == want_eval
        sess.set_base(reps)
        want = r.candidate_keys(bits, ld, 0x8160, 4, 512, 0, 4)
        for form in (0, 1):
            assert sess.set_evaluator(form)
            assert sess.get_base()[1:3] == want_eval, (what, form)
            assert (sess.candidate_keys(0x8160, 4, 512, 0, 4) == want).all(), (what, form)
        assert (sess.candidate_keys(0x8160, 4, 512, 0, 4, delta=True) == want).all(), what
    sess.close()


# ---- coverage guard --------------------------------------------------------------------------------
def objective_form(cfg):
    return "planes" if cfg["obj"] else ("dense" if cfg["dense"] else "entries")


def impossible(W, rack, form, evaluator):
    """Why a (row width, rack form, objective form, evaluator) tuple cannot occur, or None."""
    if form == "planes" and W > 2:
        return "mask planes are built for rows of up to 64 slots only"
    if evaluator == "column-major" and W > 2:
        return "the column-major evaluator covers rows of up to 64 slots"
    if evaluator == "column-major" and rack != 3:
        return "the column-major evaluator covers 8-slot rack fields with at most one replica per rack"
    return None


def test_named_shapes_reach_every_dispatched_configuration(emu):
    """Every (W, rack form, objective form, evaluator) the engine can dispatch is reached by a named shape.
    The objective forms of the instantiated objective encodings are mask planes, packed entries and the dense
    table (a run-time flag of the entries encoding); the evaluator is the row-major one, or the column-major
    one where the session accepts it.  Counter depths are not part of the tuple: the counter-limit test above
    covers the second one.  A configuration dispatch gains fails here until a shape reaches it."""
    possible = set()
    for W, _nph, rack, obj in emu.dispatch_configs():
        for form in (["planes"] if obj else ["entries", "dense"]):
            for evaluator in ("row-major", "column-major"):
                if impossible(W, rack, form, evaluator) is None:
                    possible.add((W, rack, form, evaluator))
    reached = set()
    for f in list(SHAPES.values()) + list(LAYOUT_SHAPES.values()):
        sess = emu.EmuSession(product(f()))
        c = sess.config()
        reached.add((c["W"], c["rack"], objective_form(c), "row-major"))
        if sess.set_evaluator(1):
            reached.add((c["W"], c["rack"], objective_form(c), "column-major"))
        sess.close()
    assert not {t for t in reached if impossible(*t)}, "a shape reached a tuple listed as impossible"
    assert sorted(possible - reached) == [], "dispatched configurations no named shape reaches"
    assert reached == possible
