"""Leader-only rebalancing (kao_solve_leaders, docs/MODEL.md §13) without a GPU: the flow's (violation, objective) is
the lexicographic optimum HiGHS finds for the program of tests/leaders_ref.py, and what exhaustive enumeration finds on
small instances; every row keeps its replicas and their order; every refusal is KAO_E_ARG with its message; the CLI
writes only the changed leaders, refuses the options that move data or search, and its --emit-lp text solves to the
same objective; /submit passes "leaders_only" through."""
import ctypes as C
import dataclasses
import json
import os
import subprocess

import numpy as np
import pytest
from scipy.optimize import Bounds, LinearConstraint, milp

import kafka_assignment_optimizer_b200 as kao
import leaders_ref as L
import topics_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import SLOT255_SHAPES
from test_lp_text import parse_lp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "kao-cli")


def piled(P, B, R, RF, hot, seed, extra_brokers=0, lengths=None):
    """Replicas drawn at random, the leader of every row on one of the `hot` lowest brokers (leadership piled up after
    restarts); `lengths`: row lengths drawn from it; `extra_brokers` empty brokers added to the target list"""
    rng = np.random.RandomState(seed)
    current = []
    for _ in range(P):
        n = RF if lengths is None else int(rng.choice(lengths))
        lead = int(rng.randint(hot))
        current.append([lead] + [int(b) for b in rng.choice([b for b in range(B) if b != lead], n - 1, replace=False)])
    racks = {b: "r%02d" % (b % R) for b in range(B + extra_brokers)}
    return m.build_problem(current, list(range(B + extra_brokers)), racks, RF)


def with_topics(pb, T, seed):
    rng = np.random.RandomState(seed)
    pb.topics = [("t%02d" % t, p) for p, t in enumerate(rng.randint(T, size=pb.P))]
    return pb


SHAPES = {
    "readme": lambda: m.readme_problem(),
    "cfg2_piled": lambda: piled(256, 32, 4, 3, 4, 1),
    "cfg3_piled": lambda: piled(400, 64, 8, 3, 8, 2),
    "empty_broker": lambda: piled(120, 12, 3, 3, 2, 3, extra_brokers=1),
    "mixed_lengths": lambda: piled(150, 16, 4, 4, 3, 4, lengths=[1, 2, 3, 4]),
    "slot255": lambda: SLOT255_SHAPES["s255_r32"](),
    "slot255_r4": lambda: SLOT255_SHAPES["s255_r4"](),
}
TOPIC_SHAPES = {
    "t3x20": lambda: with_topics(piled(60, 12, 3, 3, 2, 5), 3, 5),
    "t16x256": lambda: with_topics(piled(256, 32, 4, 3, 4, 6), 16, 6),
    "t16x256_slot255": lambda: with_topics(SLOT255_SHAPES["s255_r16"](), 16, 7),
}


def _lib_solve(pb, tr=None, fixed=None):
    """kao_solve_leaders through the C ABI: (rc, result, fixed_violation, replicas [P, RF])"""
    reps = np.full((pb.P, pb.RF), -7, np.int32)
    res = kopt._KaoResult()
    res.replicas = reps.ctypes.data
    fv = C.c_int64(-1)
    fx = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
    rc = kopt.load_library().kao_solve_leaders(kopt._CProblem(pb).ref(), kopt._CTopics(tr).ref(),
                                               None if fx is None else C.c_void_p(fx.ctypes.data), C.byref(res), C.byref(fv))
    return rc, res, fv.value, reps


def _check(opb, tr=None, fixed=None):
    pb = kao.Problem.from_fields(opb)
    rc, res, fv, reps = _lib_solve(pb, tr, fixed)
    assert rc in (0, 1), kopt.load_library().kao_last_error()
    # rows keep their replicas and the order of the others; unchanged leaders give cur's list
    for p, row in enumerate(L.rows(pb)):
        got = [int(b) for b in reps[p] if b >= 0]
        assert (reps[p, len(got):] == -1).all() and got[0] in row and got[1:] == [b for b in row if b != got[0]]
        if fixed is not None and fixed[p]:
            assert got == row
    assert res.moves == 0 and res.n_candidates == 0 and res.rounds_run == 0 and m.replica_moves(opb, reps) == 0
    # the violation as the model scores the assignment, its fixed part, and the exact lexicographic optimum
    whole = m.evaluate(opb, reps)
    if tr is not None:
        whole = (whole[0] + topics_ref.topic_violation(opb, tr, reps), whole[1])
    assert (res.violation, res.objective) == whole
    assert fv == L.fixed_part(pb, tr)
    v, obj, _ = L.solve_exact(pb, tr, fixed)
    assert (res.violation - fv, res.objective) == (v, obj)
    assert res.objective_bound == res.objective and res.optimal == res.feasible == (res.violation == 0)
    assert rc == (0 if res.violation == 0 else 1)
    # the same input gives the same lists
    assert np.array_equal(_lib_solve(pb, tr, fixed)[3], reps)
    return res, fv, reps


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_plain_shapes_are_the_exact_optimum(name):
    res, fv, _ = _check(SHAPES[name]())
    if name == "empty_broker" or name.startswith("slot255"):
        assert res.violation > fv                          # the new broker's C4 lower bound cannot be met


@pytest.mark.parametrize("name", sorted(TOPIC_SHAPES))
def test_topic_shapes_are_the_exact_optimum(name):
    opb = TOPIC_SHAPES[name]()
    _check(opb, kao.topic_rows(kao.Problem.from_fields(opb)))


@pytest.mark.parametrize("name", ["cfg2_piled", "mixed_lengths", "slot255", "t16x256"])
@pytest.mark.parametrize("seed", [0, 1])
def test_fixed_masks(name, seed):
    opb = {**SHAPES, **TOPIC_SHAPES}[name]()
    tr = kao.topic_rows(kao.Problem.from_fields(opb)) if name in TOPIC_SHAPES else None
    fixed = np.random.RandomState(seed).random_sample(opb.P) < 0.3 + 0.4 * seed
    _check(opb, tr, fixed)


@pytest.mark.parametrize("seed", range(6))
def test_small_instances_match_enumeration(seed):
    rng = np.random.RandomState(seed)
    opb = piled(9, 6, 2, 3, 2, 10 + seed, lengths=[2, 3])
    opb = dataclasses.replace(opb, wL=(opb.wL + rng.randint(0, 3, size=opb.wL.shape) * (opb.wF > 0)).astype(np.uint16))
    tr = kao.topic_rows(kao.Problem.from_fields(with_topics(opb, 2, seed))) if seed % 2 else None
    fixed = rng.random_sample(opb.P) < 0.2 if seed >= 4 else None
    assert np.prod([len(r) for r in L.rows(opb)]) <= 10 ** 5
    res, fv, _ = _check(opb, tr, fixed)
    assert (res.violation - fv, res.objective) == L.enumerate_all(opb, tr, fixed)


def _with_row(pb, p, row):
    cur = np.full((pb.P, max(pb.cur.shape[1], len(row))), -1, np.int32)
    cur[:, :pb.cur.shape[1]] = pb.cur
    cur[p] = -1
    cur[p, :len(row)] = row
    return dataclasses.replace(pb, cur=cur)


def test_refusals_are_arguments_errors():
    pb = kao.Problem.from_fields(m.readme_problem())           # 19 brokers, RF 2
    tr = kao.topic_rows(pb)
    cases = {
        "outside the target list": (_with_row(pb, 3, [-1, 4]), None, "partition 3 has a replica on a broker outside"),
        "outside, second entry": (_with_row(pb, 3, [2, -1, 4]), None, "partition 3 has a replica on a broker outside"),
        "not a dense index": (_with_row(pb, 3, [2, 19]), None, "partition 3 names broker 19, not a dense index"),
        "twice": (_with_row(pb, 3, [2, 2]), None, "partition 3 names broker 2 twice"),
        "empty": (_with_row(pb, 3, [-1, -1]), None, "partition 3 has no replica"),
        "longer than RF": (_with_row(pb, 3, [2, 3, 4]), None, "partition 3 has 3 replicas, more than RF = 2"),
        "topic out of range": (pb, dataclasses.replace(tr, topic_of=np.full(pb.P, 1, np.int32)), "topic rows: topic_of[0] = 1"),
        "topic lo too high": (pb, dataclasses.replace(tr, ldr_lo=np.array([11], np.int32), ldr_hi=np.array([11], np.int32)),
                              "topic rows: topic 0: lo exceeds"),
        "problem": (dataclasses.replace(pb, RF=19), None, "RF must be 1..8"),
    }
    for what, (q, t, msg) in cases.items():
        rc, res, fv, reps = _lib_solve(q, t)
        err = kopt.load_library().kao_last_error().decode()
        assert rc == -1 and msg in err, (what, rc, err)
        assert (reps == -7).all() and fv == -1, what         # nothing written
    with pytest.raises(ValueError, match="replication"):
        kao.solve_leaders(dataclasses.replace(pb, replication=kao.ReplicationRows(*[np.full(pb.P, 2, np.int32)] * 3)))


def test_python_binding_is_the_abi():
    opb = TOPIC_SHAPES["t3x20"]()
    pb = kao.Problem.from_fields(opb)
    fixed = np.arange(pb.P) % 3 == 0
    for tb in (False, True):
        got = kao.solve_leaders(dataclasses.replace(pb, fixed=fixed), topic_balance=tb)
        rc, res, fv, reps = _lib_solve(pb, kao.topic_rows(pb) if tb else None, fixed)
        assert np.array_equal(got.replicas, reps) and (got.violation, got.objective, got.fixed_violation) == \
            (res.violation, res.objective, fv) and got.feasible == (rc == 0) and got.moves == 0


# ------------------------------------------------------------------------------------------- CLI
RACKS = {b: "r%d" % (b % 3) for b in range(13)}


def _document(opb):
    return {"version": 1, "partitions": [{"topic": t, "partition": q, "replicas": [int(b) for b in opb.cur[p] if b >= 0]}
                                         for p, (t, q) in enumerate(opb.topics)]}


@pytest.fixture
def cli(tmp_path):
    import __graft_entry__ as g

    if not os.path.exists(CLI):
        g.build()
    opb = with_topics(piled(60, 12, 3, 3, 2, 5), 3, 5)
    doc = _document(opb)
    f = tmp_path / "current.json"
    f.write_text(json.dumps(doc))

    def run(*extra, brokers=range(12)):
        return subprocess.run([CLI, "--assignment", str(f), "--brokers", ",".join(map(str, brokers)),
                               "--racks", ",".join("%d:%s" % (b, RACKS[b]) for b in range(13)), "--leaders-only"] +
                              list(extra), capture_output=True, text=True)
    run.doc = doc
    run.tmp = tmp_path
    return run


def _codec(doc, move=None):
    rows, topics = kao.problem.parse_assignment_json(json.dumps(doc))
    return kao.build_problem(rows, range(12), RACKS, max(len(r) for r in rows), topics, topics_to_move=move)


@pytest.mark.parametrize("topic_balance", [False, True])
@pytest.mark.parametrize("move", [None, ["t01"]])
def test_cli_lists_only_changed_leaders(cli, topic_balance, move):
    extra = ["--stats"] + (["--topic-balance"] if topic_balance else [])
    if move:
        t = cli.tmp / "move.json"
        t.write_text(json.dumps({"topics": [{"topic": n} for n in move], "version": 1}))
        extra += ["--topics-to-move", str(t)]
    out = cli(*extra)
    assert out.returncode in (0, 3), out.stderr
    pb = _codec(cli.doc, move)
    want = kao.solve_leaders(pb, topic_balance=topic_balance)
    cur = {(e["topic"], e["partition"]): e["replicas"] for e in cli.doc["partitions"]}
    got = json.loads(out.stdout)["partitions"]
    changed = [(t, q) for p, (t, q) in enumerate(pb.topics) if want.replicas[p, 0] != pb.cur[p, 0]]
    assert [(e["topic"], e["partition"]) for e in got] == changed and changed
    for e in got:
        old = cur[(e["topic"], e["partition"])]
        assert e["replicas"][0] != old[0] and e["replicas"][1:] == [b for b in old if b != e["replicas"][0]]
        assert not move or e["topic"] == move[0]
    assert ("fixed_violation %d, leaders_changed %d," % (want.fixed_violation, len(changed))) in out.stderr
    assert ("violation %d," % want.violation) in out.stderr and "replica moves 0" in out.stderr


REFUSED = [("--rf", "3"), ("--keep-rf",), ("--topic-rf", "t00:2"), ("--delta",), ("--row-major",), ("--column-major",),
           ("--gpus", "1"), ("--restarts", "2"), ("--lp-certificate",), ("--certificate",)]


@pytest.mark.parametrize("flag", REFUSED, ids=[f[0] for f in REFUSED])
def test_cli_refuses_search_and_movement_options(cli, flag):
    out = cli(*flag)
    assert out.returncode == 2 and ("--leaders-only cannot be combined with %s" % flag[0]) in out.stderr and out.stdout == ""


def test_cli_refuses_rows_it_cannot_keep(cli):
    out = cli(brokers=range(11))                           # broker 11 leaves: its replicas would have to move
    assert out.returncode == 1 and "has a replica on broker 11, which is not in --brokers" in out.stderr


@pytest.mark.parametrize("topic_balance", [False, True])
def test_emitted_leader_program_solves_to_the_objective(cli, topic_balance):
    extra = ["--topic-balance"] if topic_balance else []
    text = cli("--emit-lp", *extra).stdout
    head = text.splitlines()[0]
    assert head.startswith("// Leaders only:")
    W0 = int(head.rsplit("=", 1)[1])
    names, c, A, lo, hi = parse_lp(text)
    assert all(n.endswith("_l") for n in names)
    pb = _codec(cli.doc)
    assert len(names) == sum(len(r) for r in L.rows(pb))
    res = milp(-c, constraints=LinearConstraint(A, lo, hi), integrality=np.ones(len(names)), bounds=Bounds(0, 1))
    want = kao.solve_leaders(pb, topic_balance=topic_balance)
    free = want.violation - want.fixed_violation
    assert (res.status == 0) == (free == 0)
    if free == 0:
        assert round(-res.fun) + W0 == want.objective


def test_emitted_program_with_an_empty_broker_is_infeasible(cli):
    text = cli("--emit-lp", brokers=range(13)).stdout     # broker 12 holds nothing: C4 lo = 60 // 13 = 4 unreachable
    assert "0 t1b" in text
    names, c, A, lo, hi = parse_lp(text)
    res = milp(-c, constraints=LinearConstraint(A, lo, hi), integrality=np.ones(len(names)), bounds=Bounds(0, 1))
    assert res.status == 2


# ------------------------------------------------------------------------------------------- /submit
def test_submit_leaders_only():
    from kafka_assignment_optimizer_b200 import service

    opb = with_topics(piled(60, 12, 3, 3, 2, 5), 3, 5)
    body = {"assignment": _document(opb), "brokers": ",".join(map(str, range(12))), "racks": RACKS, "leaders_only": True}

    def solver(pb, **kw):
        raise AssertionError("a leader-only request runs no search")

    out = service.handle_submit(body, solver)
    pb = _codec(body["assignment"])
    want = kao.solve_leaders(pb)
    assert out["moves"] == 0 and out["fixed_violation"] == want.fixed_violation and out["violation"] == want.violation
    assert out["objective"] == out["objective_bound"] == want.objective and out["feasible"] == out["proven_optimal"]
    changed = {(t, q) for p, (t, q) in enumerate(pb.topics) if want.replicas[p, 0] != pb.cur[p, 0]}
    assert {(e["topic"], e["partition"]) for e in out["reassignment"]["partitions"]} == changed
    tb = service.handle_submit(dict(body, topic_balance=True, topics_to_move=["t02"]), solver)
    want = kao.solve_leaders(_codec(body["assignment"], ["t02"]), topic_balance=True)
    assert tb["violation"] == want.violation and tb["objective"] == want.objective
    assert {e["topic"] for e in tb["reassignment"]["partitions"]} <= {"t02"}
    assert service.handle_submit(dict(body, rf=3), solver)["moves"] == 0         # rf equal to the rows' is accepted
    for bad in ({"keep_rf": True}, {"topic_rf": {"t00": 2}}, {"rf": 2}, {"brokers": ",".join(map(str, range(11)))}):
        with pytest.raises(ValueError):
            service.handle_submit(dict(body, **bad), solver)
