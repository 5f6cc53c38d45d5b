"""Replication factors 5 to 8 and RF = B - 1, without a GPU (problems.RF_SHAPES).  Every other shape of the suite that
runs on the shared-memory kernels has RF <= 4, while the engine depends on RF in places only larger factors reach:
the row pass compares bit-sliced counts with four slices of RF (bit 3 is set at RF 8 only), the tensor-core body
sums shortfalls max(0, RF - n) over planes of weight 2^k (a shortfall of 4 or more needs RF >= 5), default weights
need RFcur + 1 term planes (8 at RFcur 7, the column-major limit, and 9 at RFcur 8), the initial base completes rows by
up to five replicas or drops the tail, and at RF = B - 1 REPLACE has exactly one broker the row does not use.

The engine's device code compiled for the host (tests/emu) is held bit for bit to the restatement (oracle/kao_ref.c)
and the exact model (oracle/model.py) from the initial base, from damaged bases (rows emptied or cut short: RF 7
and RF 8 shortfalls up to RF), from a base whose every row leads from another replica and, with C7 0..1, from a base
of well-formed rows, which the column-major row pass must never charge one by one; the replication and topic forms
of the HBM-base code at RF 8; and, on instances small enough for HiGHS, the restatement's search, the flow bound, the
Lagrangian LP bound, leader-only rebalancing and the CLI's LP text at RF 8 and RF = B - 1."""
import json
import os
import subprocess

import numpy as np
import pytest
from scipy.optimize import Bounds, LinearConstraint, milp

import kafka_assignment_optimizer_b200 as kao
import lp_exact
import lp_ref
import rf_ref
import topics_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from kafka_assignment_optimizer_b200.optimizer import key_obj_bits
from oracle import model as m
from problems import (RF_EXACT_SHAPES, RF_SHAPES, emptied_base, mixed_rows, moved_base, one_per_rack_base,
                      reordered_base, term_planes)
from test_bound import relaxation_optima
from test_gpu_large_layouts import assert_keys
from test_layout_matrix import objective_form, random_assignments
from test_leaders_cpu import _check as check_leaders, with_topics
from test_lp_bound import lp_relaxation
from test_lp_text import parse_lp

SMEM = sorted(n for n, f in RF_SHAPES.items() if not n.startswith("big_"))
SIZE = 256                          # candidates of a key round; the last one is the identity
WALK = (4, 256)                     # rounds x candidates of a walk, the patched state checked after every round
CLI = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "kafka_assignment_optimizer_b200",
                   "kao-cli")

# name -> (RF, B, C7 bounds, W, row-major rack form, objective form, column-major, term planes)
# rack forms (EvalCfg): 0 general C7 bounds, 3 8-slot fields 0..1, 4 16-slot fields 0..1, 5 whole-word fields 0..1
CLASSES = {
    "rf7_cm": (7, 62, (0, 1), 2, 3, "planes", True, 4),
    "rf7_cur7": (7, 64, (0, 1), 2, 3, "planes", True, 8),
    "rf7_cur8": (7, 64, (0, 1), 2, 3, "planes", False, 9),
    "rf8_r8": (8, 64, (1, 1), 2, 0, "planes", False, 9),
    "rf8_cm": (8, 62, (0, 1), 2, 3, "planes", True, 4),
    "rf8_b9": (8, 9, (8, 8), 1, 0, "planes", False, 9),
    "rf8_r3_b9": (8, 9, (2, 3), 1, 0, "planes", False, 6),
    "rf2_b3": (2, 3, (1, 1), 1, 0, "planes", False, 3),
    "rf2_b3_r3": (2, 3, (0, 1), 1, 3, "planes", True, 3),
    "rf8_w8": (8, 221, (0, 1), 8, 4, "dense", False, 9),
    "rf5_w8": (5, 118, (0, 1), 8, 5, "dense", False, 6),
    "rf8_w12": (8, 64, (1, 1), 2, 0, "entries", False, None),
}
# the HBM path: (RF, B, C7 bounds, W, term planes, most weighted cells of a partition)
LARGE = {"big_rf8": (8, 64, (1, 1), 2, 4, 3), "big_rf8_b9": (8, 9, (8, 8), 1, 9, 8)}


@pytest.fixture(scope="module")
def emu():
    import emu as emu_mod

    emu_mod.lib()
    return emu_mod


def product(pb):
    return kao.Problem.from_fields(pb)


def shortfall(pb, reps):
    return pb.RF - (reps >= 0).sum(1)


def bases(pb, r):
    """the initial base, two damaged ones, the initial base with another replica leading every row and, with C7 0..1,
    a base of well-formed rows (RF replicas in RF racks)"""
    reps = r.decode(*r.init_base())
    out = {"initial": reps, "moved": moved_base(pb, reps, 6), "emptied": emptied_base(pb, reps, 5),
           "reordered": reordered_base(reps)}
    if (pb.ppr_lo, pb.ppr_hi) == (0, 1):
        out["one_per_rack"] = one_per_rack_base(pb)
    return out


def sessions(emu, pb):
    """name -> emulated session of every full evaluator the shape runs: row-major, column-major (popcount form 1) and
    the tensor-core body of the default schedule where the layout allows them"""
    out = {"row_major": emu.EmuSession(product(pb))}
    cm = emu.EmuSession(product(pb))
    if cm.set_evaluator(1):
        out["column_major"] = cm
        out["mma"] = emu.MmaSession(product(pb), 0x300)
    else:
        cm.close()
    return out


# ---- what each shape is for -------------------------------------------------------------------------------------------
def test_rf_shapes_reach_their_classes(emu, ref_lib):
    """Each RF_SHAPES entry is in the layout class it was added for, so that an edit cannot quietly move it out"""
    assert set(CLASSES) | set(LARGE) == set(RF_SHAPES)
    for name, (RF, B, c7, W, rack, form, cm, planes) in CLASSES.items():
        pb = RF_SHAPES[name]()
        assert (pb.RF, pb.B, (pb.ppr_lo, pb.ppr_hi)) == (RF, B, c7), name
        assert pb.P <= 8160 and term_planes(pb) == planes, name
        sess = emu.EmuSession(product(pb))
        c = sess.config()
        assert (c["W"], c["rack"], objective_form(c)) == (W, rack, form), (name, c)
        assert sess.set_evaluator(1) == cm, name
        sess.close()
    for name, (RF, B, c7, W, planes, cells) in LARGE.items():
        pb = RF_SHAPES[name]()
        assert pb.P > 8160 and (pb.RF, pb.B, (pb.ppr_lo, pb.ppr_hi)) == (RF, B, c7), name
        assert ref_lib.Ref(pb).W == W and term_planes(pb) == planes, name
        assert ((pb.wF | pb.wL) > 0).sum(1).max() == cells, name       # above four: the dense table
    # RF = B - 1: one broker the row does not use
    assert {n for n, f in RF_SHAPES.items() if f().RF == f().B - 1} == {"rf8_b9", "rf8_r3_b9", "rf2_b3", "rf2_b3_r3",
                                                                       "big_rf8_b9"}
    # the widest weights at RF 8: a 24-bit cost field, the narrowest violation field
    assert key_obj_bits(product(RF_SHAPES["rf8_w12"]())) == 24
    # the initial base completes rows by five replicas (3 -> 8) and drops the tail of eight (8 -> 7)
    for name, RFcur in (("rf8_cm", 3), ("rf7_cur8", 8)):
        pb = RF_SHAPES[name]()
        r = ref_lib.Ref(pb)
        reps = r.decode(*r.init_base())
        assert pb.cur.shape[1] == RFcur and ((reps >= 0).sum(1) == pb.RF).all(), name
        if RFcur == 8:                                  # the first seven kept, led from the first
            assert (reps[:, 0] == pb.cur[:, 0]).all()
            assert all(set(reps[p]) == set(pb.cur[p, :7]) for p in range(pb.P))
    # damaged RF 7 and RF 8 bases on the column-major evaluator have rows short by 4 or more (the S_2 shortfall plane)
    # and rows short by all RF (z = 0: RF 8 is bit 3 of z); the one-per-rack bases are well formed
    for name in ("rf7_cm", "rf7_cur7", "rf8_cm"):
        pb = RF_SHAPES[name]()
        b = bases(pb, ref_lib.Ref(pb))
        assert shortfall(pb, b["emptied"]).max() == pb.RF, name
        assert (shortfall(pb, b["one_per_rack"]) == 0).all(), name
        assert all(len(set(pb.rack_of[row])) == pb.RF for row in b["one_per_rack"]), name


# ---- keys and walks on the shared-memory kernels' code -----------------------------------------------------------------
@pytest.mark.parametrize("name", SMEM)
def test_emulated_keys_from_every_base(emu, ref_lib, name):
    """A free and a cycle round, the identity candidate included, on every full evaluator, the delta keys and the
    tensor-core body's sorted batches; get_base after set_base equals the restatement and the model"""
    pb = RF_SHAPES[name]()
    r = ref_lib.Ref(pb)
    runs = sessions(emu, pb)
    for what, b in bases(pb, r).items():
        bits, ld = r.encode(b)
        want_eval = m.evaluate(pb, r.decode(bits, ld))
        for who, sess in runs.items():
            sess.set_base(b)
            reps, v, o, moves = sess.get_base()
            assert (reps == r.decode(bits, ld)).all() and r.evaluate(bits, ld) == want_eval, (what, who)
            assert (v, o) == r.unpack_key(r.pack_key(*want_eval, 0))[:2], (what, who)
            assert moves == m.replica_moves(pb, reps), (what, who)
        emu.rows_charged_one_by_one()
        for rnd in (4, 7):
            want = r.candidate_keys(bits, ld, 0x7F8, rnd, SIZE, 0, SIZE)
            assert r.unpack_key(want[-1])[:2] == r.unpack_key(r.pack_key(*want_eval, 0))[:2]
            for who, sess in runs.items():
                assert_keys(sess.candidate_keys(0x7F8, rnd, SIZE, 0, SIZE), want, (what, who, rnd))
            assert_keys(runs["row_major"].candidate_keys(0x7F8, rnd, SIZE, 0, SIZE, delta=True), want,
                        (what, "delta", rnd))
            if "mma" in runs:
                assert_keys(runs["mma"].sorted_keys(0x7F8, rnd, SIZE, 0, SIZE, 2, 16, 8192), want, (what, "sorted", rnd))
        if "column_major" in runs and what == "emptied":
            assert emu.rows_charged_one_by_one() > 0           # rows short by up to RF, charged one by one
        if "column_major" in runs and what == "one_per_rack":
            assert emu.rows_charged_one_by_one() == 0          # a well-formed row never is
    for sess in runs.values():
        sess.close()


@pytest.mark.parametrize("name", SMEM)
def test_emulated_walks_from_every_base(emu, ref_lib, name):
    """4 rounds of 256 on every full evaluator, one round a call, the state every winner patches (planes, one-hot plane,
    count of invalid leaders, displaced lists) checked against the state rebuilt from the base after each; the walked
    base is the restatement's and scores as the model says"""
    pb = RF_SHAPES[name]()
    r = ref_lib.Ref(pb)
    rounds, size = WALK
    runs = sessions(emu, pb)
    for what, start in bases(pb, r).items():
        seed = 0x5EED + len(what)
        bits, ld = r.encode(start)
        _, want = r.search(bits, ld, seed, 0, rounds, size)
        for who, sess in runs.items():
            sess.set_base(start)
            for rnd in range(rounds):
                assert_keys(sess.search(seed, rnd, 1, size), want[rnd:rnd + 1], (what, who, rnd))
                rc, at, msg = sess.check_state()
                assert rc == 0, (what, who, rnd, rc, at, msg)
            end, v, o, _ = sess.get_base()
            assert (end == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == m.evaluate(pb, end), (what, who)
    for sess in runs.values():
        sess.close()


@pytest.mark.parametrize("name", SMEM)
def test_evaluations_equal_the_model(emu, name):
    """kao_eval and get_base on random assignments, rows cut short and brokers named twice"""
    pb = RF_SHAPES[name]()
    sess = emu.EmuSession(product(pb))
    cands = random_assignments(pb, np.random.RandomState(23), 6)
    v, o = sess.evaluate(np.stack(cands))
    for i, reps in enumerate(cands):
        assert (int(v[i]), int(o[i])) == m.evaluate(pb, reps), i
        sess.set_base(reps)
        got, gv, go, moves = sess.get_base()
        assert (gv, go) == m.evaluate(pb, got) and moves == m.replica_moves(pb, got), i
    sess.close()


# ---- per-partition replication and topic rows at RF 8 --------------------------------------------------------------------
@pytest.mark.parametrize("name", ["rf8_r8", "rf8_b9"])
def test_emulated_replication_and_topic_sessions_at_rf8(emu, name):
    """rf[p] over 1..min(8, B - 1) with mixed C7 forms, and five interleaved topics: get_base and the delta keys of a
    free and a cycle round from the initial and the damaged bases, and a 24-round walk, against tests/rf_ref and
    tests/topics_ref"""
    pb = RF_SHAPES[name]()
    kp = product(pb)
    rr = mixed_rows(kp, 0x58)
    assert {1, min(8, pb.B - 1)} <= set(rr.rf.tolist())
    tpb = RF_SHAPES[name]()
    tpb.topics = [("t%d" % (p % 5), p) for p in range(pb.P)]
    tr = kao.topic_rows(product(tpb))
    runs = {"replication": (emu.EmuSession(kp, replication=rr), rf_ref.RRef(kp, rr),
                            lambda reps: rf_ref.evaluate(kp, rr, reps)),
            "topics": (emu.EmuSession(tpb, topics=tr), topics_ref.TRef(tpb, tr),
                       lambda reps: topics_ref.evaluate(tpb, tr, reps))}
    for who, (sess, r, evaluate) in runs.items():
        init = r.decode(*r.init_base())
        for what, b in (("initial", init), ("moved", moved_base(pb, init, 6)), ("emptied", emptied_base(pb, init, 5))):
            sess.set_base(b)
            bits, ld = r.encode(b)
            got, v, o, _ = sess.get_base()
            assert (got == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == evaluate(got), (who, what)
            for rnd in (4, 7):
                assert_keys(sess.candidate_keys(0xB16, rnd, 1024, 0, 1024, delta=True),
                            r.candidate_keys(bits, ld, 0xB16, rnd, 1024, 0, 1024), (who, what, rnd))
            sess.set_base(b)
            _, want = r.search(bits, ld, 0x5EED, 0, 24, 256)
            assert_keys(sess.search(0x5EED, 0, 24, 256), want, (who, what, "walk"))
            end, v, o, _ = sess.get_base()
            assert (end == r.decode(bits, ld)).all() and (v, o) == evaluate(end), (who, what)
        sess.close()


# ---- against HiGHS -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(RF_EXACT_SHAPES))
def test_restatement_search_reaches_the_exact_optimum(ref_lib, name):
    pb = RF_EXACT_SHAPES[name]()
    sol = m.solve_exact(pb)
    assert sol.status == "optimal"
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    _, keys = r.search(bits, ld, 0x5EED, 0, 300, 4096)
    assert r.unpack_key(keys[-1])[:2] == (0, sol.objective)
    assert m.evaluate(pb, r.decode(bits, ld)) == (0, sol.objective)


@pytest.mark.parametrize("name", sorted(RF_EXACT_SHAPES))
def test_flow_bound_and_lp_bound_bracket_the_optimum(name):
    """kao_objective_bound is min(cheap bound, the flow relaxations' optima) and at least the optimum; the Lagrangian
    LP bound's restatement is at least the optimum and the LP relaxation, and L at its multipliers floors to it"""
    pb = RF_EXACT_SHAPES[name]()
    sol = m.solve_exact(pb)
    kp = product(pb)
    cheap = kao.objective_bound(kp)
    tight = kao.objective_bound(kp, sol.replicas)
    assert sol.objective <= tight <= cheap
    assert tight == min(cheap, relaxation_optima(pb))
    bound, its, u = lp_ref.lp_bound(pb, sol.objective, kopt.LP_ITERATIONS)
    assert 1 <= its <= kopt.LP_ITERATIONS and (np.abs(u) <= lp_exact.U).all()
    assert lp_exact.lagrangian_fixed(pb, u) >> lp_exact.F == bound
    assert bound >= sol.objective and bound >= int(np.floor(lp_relaxation(pb) + 1e-6))


@pytest.mark.parametrize("name", sorted(RF_EXACT_SHAPES))
@pytest.mark.parametrize("topics", [False, True])
def test_leaders_only_is_the_exact_optimum(name, topics):
    opb = RF_EXACT_SHAPES[name]()
    if topics:
        opb = with_topics(opb, 3, 8)
    check_leaders(opb, kao.topic_rows(product(opb)) if topics else None)


@pytest.mark.parametrize("name", ["rf8_b9_p12", "rf8_b10"])
def test_emitted_lp_at_rf8_solves_to_the_model_optimum(tmp_path, name):
    """kao-cli --rf 8 --emit-lp on the shape's current assignment, parsed back and solved with HiGHS"""
    import __graft_entry__ as g

    if not os.path.exists(CLI):
        g.build()
    pb = RF_EXACT_SHAPES[name]()
    rows = [[int(b) for b in row if b >= 0] for row in pb.cur]
    f = tmp_path / "current.json"
    f.write_text(json.dumps({"version": 1, "partitions": [{"topic": "t", "partition": p, "replicas": row}
                                                          for p, row in enumerate(rows)]}))
    racks = ",".join("%d:r%d" % (b, pb.rack_of[b]) for b in range(pb.B))
    text = subprocess.check_output([CLI, "--assignment", str(f), "--brokers", ",".join(map(str, range(pb.B))),
                                    "--racks", racks, "--rf", "8", "--emit-lp"], text=True)
    names, c, A, lo, hi = parse_lp(text)
    assert len(names) == 2 * pb.P * pb.B
    res = milp(-c, constraints=LinearConstraint(A, lo, hi), integrality=np.ones(len(names)), bounds=Bounds(0, 1))
    assert res.status == 0 and round(-res.fun) == m.solve_exact(pb).objective
