"""Fixed partitions (docs/MODEL.md §12) without a GPU: the engine's host reduction (reduce_fixed, compiled for the host
by tests/emu) scored by the emulated sessions of the same library, plus V0 / O0, is the restricted program of
tests/fixed_ref.py; kao_objective_bound_fixed brackets the HiGHS restricted optimum; every refusal is KAO_E_ARG before
any CUDA call; `kao-cli --emit-lp --topics-to-move` writes the restricted program; the Python codec and /submit pick
the searched rows by the CLI's rule."""
import ctypes as C
import dataclasses
import json
import os
import subprocess

import numpy as np
import pytest
from scipy.optimize import Bounds, LinearConstraint, milp

import emu
import fixed_ref as F
import kafka_assignment_optimizer_b200 as kao
from emu import EmuSession
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import SHAPES, SLOT255_SHAPES, moved_base
from test_lp_text import parse_lp
from test_replication_cpu import BOUND_INSTANCES, readme_mixed, readme_mixed_document, seeded_mixed
from test_topics_cpu import interleaved_topics, readme_three_topics, sixteen_topics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "kao-cli")
RACKS = {b: ("b" if b % 2 else "a") for b in range(20)}
PLAIN = ["readme", "readme_tb", "cfg2", "cfg2_rm2", "cfg3_small", "w4_s16", "w8_s16", "s32", "s64_r1", "rf_up",
         "rf_down", "dense_small", "tiny", "ragged", "rf1", "all_slots", "max_rows"]


def _full(pb, red, reduced):
    out = emu.expand(pb, np.isin(np.arange(pb.P), red.searched, invert=True), reduced)
    assert np.array_equal(out, F.expand(pb, red, reduced))
    return out


def _check(opb, fx, tr=None, rr=None, seeds=(0, 1)):
    """reduce_fixed against the restatement, then the emulated reduced session + V0 / O0 against the restricted program
    at the reduced problem's initial base and at moved bases"""
    pb = kao.Problem.from_fields(opb)
    red = emu.reduce(pb, fx, tr, rr)
    want = F.reduce(pb, fx, tr, rr)
    assert (red.V0, red.O0) == (want.V0, want.O0) and np.array_equal(red.searched, want.searched)
    for k in ("cur", "wF", "wL", "rep_lo", "rep_hi", "ldr_lo", "ldr_hi", "rack_lo", "rack_hi"):
        assert np.array_equal(getattr(red.pb, k), getattr(want.pb, k)), k
    for a, b in ((red.replication, want.replication), (red.topics, want.topics)):
        if a is not None:
            for k in ("rf", "ppr_lo", "ppr_hi") if a is red.replication else ("topic_of", "rep_lo", "rep_hi", "ldr_lo", "ldr_hi"):
                assert np.array_equal(getattr(a, k), getattr(b, k)), k
    s = EmuSession(red.pb, replication=red.replication, topics=red.topics)
    base = s.get_base()[0]
    for reps in [base] + [moved_base(red.pb, base, seed) for seed in seeds]:
        s.set_base(reps)
        got, v, o, _ = s.get_base()
        full = _full(pb, red, got)
        assert (v + red.V0, o + red.O0) == F.evaluate(opb, fx, full, tr, rr)
    s.close()
    return red


@pytest.mark.parametrize("name", PLAIN)
@pytest.mark.parametrize("seed", [0, 1])
def test_reduced_session_is_the_restricted_program(name, seed):
    opb = SHAPES[name]()
    fx = F.random_mask(opb, seed, share=0.3 + 0.4 * seed)
    _check(opb, fx)


@pytest.mark.parametrize("name", ["s255_r32", "s255_r4", "s255_r16_dense"])
def test_slot255(name):
    opb = SLOT255_SHAPES[name]()
    _check(opb, F.random_mask(opb, 3))


def test_fixed_load_above_rep_hi():
    """f_b > rep_hi_b: the fixed rows alone exceed C3 / C4 / C6 on some brokers and racks, V0 > 0"""
    opb = SHAPES["cfg2"]()
    opb = dataclasses.replace(opb, rep_lo=np.zeros(opb.B, np.int32), rep_hi=np.full(opb.B, 5, np.int32),
                              ldr_lo=np.zeros(opb.B, np.int32), ldr_hi=np.full(opb.B, 2, np.int32),
                              rack_hi=np.full(opb.R, 100, np.int32), rack_lo=np.zeros(opb.R, np.int32))
    fx = F.random_mask(opb, 4, share=0.8)
    f, fl, fr, *_ = F.fixed_load(opb, fx)
    assert (f > 5).any() and (fl > 2).any() and (fr > 100).any()
    red = _check(opb, fx)
    assert red.V0 > 0 and (red.pb.rep_hi == 0).any()


@pytest.mark.parametrize("make", [readme_three_topics, sixteen_topics, interleaved_topics])
@pytest.mark.parametrize("seed", [0, 1])
def test_topics(make, seed):
    opb, tr = make()
    fx = F.random_mask(opb, seed, tr=tr)
    assert fx.any() and not fx.all()
    _check(opb, fx, tr=tr)


@pytest.mark.parametrize("name", sorted(BOUND_INSTANCES))
def test_replication_rows(name):
    pb = BOUND_INSTANCES[name]()
    fx = F.random_mask(pb, 5, share=0.5)
    _check(pb, fx, rr=pb.replication)


def test_topics_above_the_shared_memory_limit():
    """a fixed topic's cells over 256 brokers, 9,000 partitions, reduced below 8,160"""
    from problems import SLOT255_TOPIC_SHAPES

    opb = SLOT255_TOPIC_SHAPES["sized_big"]()
    tr = kao.topic_rows(kao.Problem.from_fields(opb))
    fx = F.random_mask(opb, 6, share=0.6, tr=tr)
    red = _check(opb, fx, tr=tr, seeds=(0,))
    assert red.pb.P < opb.P


# ------------------------------------------------------------------------------------------- bounds
def _bound(pb, fixed, replicas=None, rr=None):
    out = C.c_int64()
    fx = np.ascontiguousarray(fixed, np.uint8) if fixed is not None else None
    reps = None if replicas is None else np.ascontiguousarray(replicas, np.int32)
    rc = kopt.load_library().kao_objective_bound_fixed(
        kopt._CProblem(pb).ref(), kopt._CReplication(rr).ref(), None if fx is None else C.c_void_p(fx.ctypes.data),
        None if reps is None else C.c_void_p(reps.ctypes.data), C.byref(out))
    assert rc == 0, kopt.load_library().kao_last_error()
    return out.value


BOUND_SHAPES = ["readme", "readme_tb", "tiny", "dense_small", "dense_unique", "dense_unique2", "rf1", "one_partition"]


@pytest.mark.parametrize("name", BOUND_SHAPES + sorted(BOUND_INSTANCES))
def test_bounds_bracket_the_restricted_optimum(name):
    opb = SHAPES[name]() if name in SHAPES else BOUND_INSTANCES[name]()
    pb = kao.Problem.from_fields(opb)
    rr = pb.replication
    for seed in (0, 1, 2):
        fx = F.random_mask(pb, seed)
        sol = F.solve_exact(opb, fx, rr=rr)
        if sol.status != "optimal":
            continue
        cheap, flow = _bound(pb, fx, None, rr), _bound(pb, fx, sol.replicas, rr)
        assert sol.objective <= flow <= cheap
        assert kao.objective_bound(dataclasses.replace(pb, fixed=fx), sol.replicas) == flow
    zero = np.zeros(pb.P, bool)
    feas = (m.solve_exact(opb).replicas if rr is None else None)
    for reps in (None, feas):
        plain = kao.objective_bound(pb, reps)
        assert _bound(pb, zero, reps, rr) == plain == _bound(pb, None, reps, rr)


# ------------------------------------------------------------------------------------------- refusals
def _solve_rc(pb, fixed, tr=None, rr=None):
    lib = kopt.load_library()
    reps = np.full((pb.P, pb.RF), -1, np.int32)
    opt = kopt._KaoOptions(1, 4, 64, 0, 0, 1, 0)
    res = kopt._KaoResult()
    res.replicas = reps.ctypes.data
    fx = np.ascontiguousarray(fixed, np.uint8)
    rc = lib.kao_solve_fixed(kopt._CProblem(pb).ref(), kopt._CTopics(tr).ref(), kopt._CReplication(rr).ref(),
                             C.c_void_p(fx.ctypes.data), C.byref(opt), C.byref(res))
    out = C.c_int64()
    rcb = lib.kao_objective_bound_fixed(kopt._CProblem(pb).ref(), kopt._CReplication(rr).ref(),
                                        C.c_void_p(fx.ctypes.data), None, C.byref(out))
    return rc, (rcb if tr is None else rc), lib.kao_last_error().decode()


def _with_row(pb, p, row):
    cur = np.full((pb.P, max(pb.cur.shape[1], len(row))), -1, np.int32)
    cur[:, :pb.cur.shape[1]] = pb.cur
    cur[p] = -1
    cur[p, :len(row)] = row
    return dataclasses.replace(pb, cur=cur)


def test_refusals_without_a_gpu():
    pb = kao.Problem.from_fields(m.readme_problem())
    one = np.zeros(pb.P, bool)
    one[3] = True
    cases = {
        "empty": (_with_row(pb, 3, [-1, -1]), one),
        "after -1": (_with_row(pb, 3, [-1, 4]), one),
        "after -1 (second)": (_with_row(pb, 3, [2, -1, 4]), one),
        "twice": (_with_row(pb, 3, [2, 2]), one),
        "more than RF": (_with_row(pb, 3, [2, 3, 4]), one),
        "not a dense index": (_with_row(pb, 3, [2, 19]), one),
        "all fixed": (pb, np.ones(pb.P, bool)),
    }
    for what, (q, fx) in cases.items():
        rc, rcb, msg = _solve_rc(q, fx)
        assert rc == -1 and rcb == -1, (what, rc, rcb, msg)
        assert "fixed partitions" in msg, (what, msg)
    # a topic partly fixed, with topic rows (without them the same mask is accepted by the reduction)
    opb, tr = readme_three_topics()
    tp = kao.Problem.from_fields(opb)
    fx = np.asarray(tr.topic_of) == 1                      # topic b: no replica on the leaving broker 19
    fx[np.flatnonzero(fx)[0]] = False
    rc, _, msg = _solve_rc(tp, fx, tr)
    assert rc == -1 and "partly fixed" in msg
    emu.reduce(tp, fx)
    # what kao_solve_replication refuses is still refused first
    rc, rcb, msg = _solve_rc(dataclasses.replace(pb, ppr_lo=64, ppr_hi=64), one)
    assert rc == -1 and rcb == -1 and "per-partition-per-rack" in msg
    # the Python paths that take no mask refuse a problem with one
    fxpb = dataclasses.replace(pb, fixed=one)
    for call in (lambda: kao.Session(fxpb), lambda: kopt.evaluate(fxpb, np.zeros((pb.P, pb.RF), np.int32)),
                 lambda: kao.lp_bound(fxpb, np.zeros((pb.P, pb.RF), np.int32))):
        with pytest.raises(ValueError, match="fixed rows"):
            call()


# ------------------------------------------------------------------------------------------- CLI and codec
def _document(rows, topics):
    return {"version": 1, "partitions": [{"topic": t, "partition": q, "replicas": r} for r, (t, q) in zip(rows, topics)]}


@pytest.fixture
def cli(tmp_path):
    import __graft_entry__ as g

    if not os.path.exists(CLI):
        g.build()
    rows, topics = readme_mixed_document()
    f = tmp_path / "current.json"
    f.write_text(json.dumps(_document(rows, topics)))

    def run(move, *extra):
        t = tmp_path / "topics-to-move.json"
        t.write_text(json.dumps({"topics": [{"topic": n} for n in move], "version": 1}))
        return subprocess.run([CLI, "--assignment", str(f), "--brokers", ",".join(map(str, range(19))),
                               "--racks", ",".join("%d:%s" % (b, RACKS[b]) for b in range(20)),
                               "--topics-to-move", str(t)] + list(extra), capture_output=True, text=True)
    return run


def _codec(move, **kw):
    rows, topics = kao.problem.parse_assignment_json(json.dumps(_document(*readme_mixed_document())))
    return kao.build_problem(rows, range(19), RACKS, kw.pop("rf", None), topics, topics_to_move=move, **kw)


@pytest.mark.parametrize("extra", [("--rf", "3"), ("--rf", "3", "--topic-balance"), ("--keep-rf",),
                                   ("--keep-rf", "--topic-balance")])
@pytest.mark.parametrize("move", [["a3"], ["b1"], ["a3", "b1"]])
def test_emitted_restricted_program_is_the_models(cli, extra, move):
    out = cli(move, "--emit-lp", *extra)
    assert out.returncode == 0, out.stderr
    head = out.stdout.splitlines()[0]
    assert head.startswith("// Fixed partitions:")
    O0 = int(head.rsplit("=", 1)[1])
    names, c, A, lo, hi = parse_lp(out.stdout)
    res = milp(-c, constraints=LinearConstraint(A, lo, hi), integrality=np.ones(len(names)), bounds=Bounds(0, 1))
    kw = {"keep_rf": True} if "--keep-rf" in extra else {"rf": 3}
    pb = _codec(move, **kw)
    tr = kao.topic_rows(pb) if "--topic-balance" in extra else None
    sol = F.solve_exact(pb, pb.fixed, tr=tr, rr=pb.replication)
    assert (res.status == 0) == (sol.status == "optimal")
    if sol.status == "optimal":
        assert round(-res.fun) + O0 == sol.objective
    # the variables are the searched rows' only
    searched = set(np.flatnonzero(~pb.fixed))
    assert {int(n.split("p")[-1].split("_")[0]) for n in names} == searched
    assert F.fixed_load(pb, pb.fixed)[3] == O0


def test_cli_refuses_unknown_and_fixed_names(cli):
    out = cli(["nope"], "--emit-lp")
    assert out.returncode == 1 and "no topic named nope" in out.stderr
    out = cli(["a3"], "--emit-lp", "--topic-rf", "b1:1")
    assert out.returncode == 1 and "fixed partitions" in out.stderr
    assert cli(["a3"], "--emit-lp", "--topic-rf", "a3:2").returncode == 0


def test_codec_searches_partitions_on_leaving_brokers():
    pb = _codec(["a3"], rf=3)
    rows, topics = kao.problem.parse_assignment_json(json.dumps(_document(*readme_mixed_document())))
    for p, ((t, q), reps) in enumerate(zip(topics, rows)):
        assert pb.fixed[p] == (t != "a3" and 19 not in reps), (t, q, reps)
    assert not pb.fixed[[p for p, r in enumerate(rows) if 19 in r]].any()
    with pytest.raises(ValueError, match="does not contain"):
        _codec(["nope"], rf=3)
    with pytest.raises(ValueError, match="fixed"):
        _codec(["a3"], topic_rf={"b1": 1})
    doc = kao.problem.reassignment_json(pb, np.zeros((pb.P, pb.RF), np.int32))
    assert [(e["topic"], e["partition"]) for e in doc["partitions"]] == \
        [tq for tq, f in zip(topics, pb.fixed) if not f]
    assert kao.problem.parse_topics_to_move('{"topics":[{"topic":"a3"},{"topic":"b1"}],"version":1}') == ["a3", "b1"]


def test_submit_passes_topics_to_move_only_when_asked():
    from kafka_assignment_optimizer_b200 import service

    seen = []

    def solver(pb, **kw):
        seen.append(pb)
        return kopt.SolveResult(np.zeros((pb.P, pb.RF), np.int32), 0, 0, 0, True, 0, 0, 0, 0.0, 0.0)

    rows, topics = readme_mixed_document()
    body = {"assignment": _document(rows, topics), "brokers": ",".join(map(str, range(19))), "racks": RACKS, "rf": 3}
    plain = service.handle_submit(body, solver)
    moved = service.handle_submit(dict(body, topics_to_move=["b1"]), solver)
    assert seen[0].fixed is None and len(plain["reassignment"]["partitions"]) == len(rows)
    # b1's three partitions and the one x.y.z.t partition on broker 19, which is leaving
    got = [(e["topic"], e["partition"]) for e in moved["reassignment"]["partitions"]]
    assert got == [("b1", 0), ("b1", 1), ("b1", 2), ("x.y.z.t", 1)]
    service.handle_submit(dict(body, topics_to_move=["b1"], keep_rf=True), solver)
    assert seen[2].fixed is not None and seen[2].replication is not None


def test_cli_refuses_rows_and_topics_the_solve_would_refuse(cli, tmp_path):
    # --topic-balance: x.y.z.t's partition 1 sits on the leaving broker 19, so that topic would be partly fixed
    out = cli(["a3"], "--rf", "3", "--topic-balance")
    assert out.returncode == 1 and "topic x.y.z.t is partly fixed" in out.stderr and out.stdout == ""
    assert cli(["a3", "x.y.z.t"], "--rf", "3", "--topic-balance", "--emit-lp").returncode == 0
    # --emit-lp checks the kept rows as the solve does: a broker twice, more than RF replicas, no replica
    rows, topics = readme_mixed_document()
    for bad, extra, msg in (([2, 2], (), "lists a broker twice"), ([2, 3], ("--rf", "1"), "has more than RF = 1"),
                            ([], (), "has no replica")):
        doc = _document(rows + [bad], topics + [("c", 0)])
        f = tmp_path / "bad.json"
        f.write_text(json.dumps(doc))
        t = tmp_path / "move.json"
        t.write_text(json.dumps({"topics": [{"topic": "a3"}], "version": 1}))
        out = subprocess.run([CLI, "--assignment", str(f), "--brokers", ",".join(map(str, range(19))),
                              "--racks", ",".join("%d:%s" % (b, RACKS[b]) for b in range(20)), "--topics-to-move", str(t),
                              "--emit-lp"] + list(extra), capture_output=True, text=True)
        assert out.returncode == 1 and "partition c-0 is kept but " + msg in out.stderr, out.stderr


def test_python_solve_names_partly_fixed_topics():
    pb = _codec(["a3"], rf=3)
    with pytest.raises(ValueError, match="partly fixed.*x.y.z.t"):
        kopt.solve(pb, topic_balance=True)
