"""Per-partition replication rows (docs/MODEL.md §11) at the front ends, without a GPU: `kao-cli --keep-rf / --topic-rf
--emit-lp` writes each partition's C1 / C7 rows and solves (HiGHS) to the model's optimum, with and without
--topic-balance; without the new options the CLI's text on a mixed document is what it was before them; the Python
codec and /submit build per-partition rows only when asked and refuse what they cannot answer."""
import hashlib
import json
import os
import re
import subprocess

import numpy as np
import pytest
from scipy.optimize import Bounds, LinearConstraint, milp

import kafka_assignment_optimizer_b200 as kao
import rf_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from test_lp_text import parse_lp
from test_replication_cpu import RACKS, readme_mixed_document

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "kao-cli")
BROKERS = list(range(19))

# sha256 of `kao-cli --emit-lp [extra]` on the mixed document, from the CLI as it was before --keep-rf / --topic-rf
BEFORE = {(): "921f6c03504c45f990b0ea45b60d1969d9a457d542824ecb880a5bb67a706a98",
          ("--topic-balance",): "ba64d3ca2dd87bd7a45cbd2eff2e61f48e8fccdbb85ae689e0de48b8fd18f762",
          ("--rf", "2"): "06cb312ce692a763e9188b833163a0a78fc5d27077fd16e524a2f78fd9966d48"}


def _doc():
    rows, topics = readme_mixed_document()
    return {"version": 1, "partitions": [{"topic": t, "partition": q, "replicas": r} for r, (t, q) in zip(rows, topics)]}


@pytest.fixture
def cli(tmp_path):
    import __graft_entry__ as g

    if not os.path.exists(CLI):
        g.build()
    f = tmp_path / "current.json"
    f.write_text(json.dumps(_doc()))
    args = [CLI, "--assignment", str(f), "--brokers", ",".join(map(str, BROKERS)),
            "--racks", ",".join("%d:%s" % (b, RACKS[b]) for b in range(20))]
    return lambda *extra: subprocess.run(args + list(extra), capture_output=True, text=True)


def _codec(**kw):
    """the problem the codec builds from the same document (rows in (topic, partition) order, as kao-cli sorts them)"""
    rows, topics = kao.problem.parse_assignment_json(json.dumps(_doc()))
    return kao.build_problem(rows, BROKERS, RACKS, kw.pop("rf", None), topics, **kw)


def _c1_rows(text):
    block = text.split("// Constrain on replication factor for every partition\n")[1].split("\n\n")[0]
    return [int(re.search(r" = (\d+);$", line).group(1)) for line in block.splitlines()]


def _highs(text):
    names, c, A, lo, hi = parse_lp(text)
    res = milp(-c, constraints=LinearConstraint(A, lo, hi), integrality=np.ones(len(names)), bounds=Bounds(0, 1))
    assert res.status == 0
    return round(-res.fun)


def test_without_the_new_options_the_text_is_unchanged(cli):
    for extra, digest in BEFORE.items():
        out = cli("--emit-lp", *extra)
        assert out.returncode == 0 and hashlib.sha256(out.stdout.encode()).hexdigest() == digest, extra
    assert _codec(rf=3).replication is None and _codec(rf=3).RF == 3


@pytest.mark.parametrize("topic_balance", [False, True])
def test_keep_rf_program_is_the_models(cli, topic_balance):
    pb = _codec(keep_rf=True)
    rr = pb.replication
    extra = ["--topic-balance"] if topic_balance else []
    text = cli("--emit-lp", "--keep-rf", *extra).stdout
    assert _c1_rows(text) == rr.rf.tolist() == [3] * 4 + [1] * 3 + [2] * 10        # a3, b1, x.y.z.t
    tr = kao.topic_rows(pb) if topic_balance else None
    assert _highs(text) == rf_ref.solve_exact(pb, rr, tr).objective
    if topic_balance:
        assert "// Constraint on min/max replicas of topic x.y.z.t per broker" in text


def test_topic_rf_program_is_the_models(cli):
    pb = _codec(topic_rf={"x.y.z.t": 3, "a3": 2})
    text = cli("--emit-lp", "--topic-rf", "x.y.z.t:3,a3:2").stdout
    assert _c1_rows(text) == pb.replication.rf.tolist() == [2] * 4 + [1] * 3 + [3] * 10
    assert _highs(text) == rf_ref.solve_exact(pb, pb.replication).objective
    # --rf N for the unnamed topics
    pb2 = _codec(rf=2, topic_rf={"b1": 1})
    assert _c1_rows(cli("--emit-lp", "--rf", "2", "--topic-rf", "b1:1").stdout) == pb2.replication.rf.tolist() == \
        [2] * 4 + [1] * 3 + [2] * 10


def test_unknown_topic_names_are_refused(cli):
    out = cli("--emit-lp", "--topic-rf", "x.y.z.T:3")
    assert out.returncode == 1 and "no topic named x.y.z.T" in out.stderr
    with pytest.raises(ValueError, match="x.y.z.T"):
        _codec(topic_rf={"x.y.z.T": 3})


def test_python_paths_without_per_partition_rows_refuse_them():
    pb = _codec(keep_rf=True)
    reps = np.zeros((pb.P, pb.RF), np.int32)
    with pytest.raises(ValueError, match="per-partition"):
        kopt.evaluate(pb, reps)
    with pytest.raises(ValueError, match="per-partition"):
        kopt.lp_bound(pb, reps)


def test_submit_passes_per_partition_rows_only_when_asked():
    from kafka_assignment_optimizer_b200 import service

    seen = []

    def solver(pb, **kw):
        seen.append((pb, kw))
        return kopt.SolveResult(np.zeros((pb.P, pb.RF), np.int32), 0, 0, 0, True, 0, 0, 0, 0.0, 0.0)

    body = {"assignment": _doc(), "brokers": ",".join(map(str, BROKERS)), "racks": RACKS}
    service.handle_submit(body, solver)
    service.handle_submit(dict(body, keep_rf=True), solver)
    service.handle_submit(dict(body, topic_rf={"x.y.z.t": 3}, rf=2), solver)
    assert seen[0][0].replication is None and seen[0][0].RF == 3
    assert seen[1][0].replication.rf.tolist() == [3] * 4 + [1] * 3 + [2] * 10
    assert seen[2][0].replication.rf.tolist() == [2] * 4 + [2] * 3 + [3] * 10
    assert all(kw == seen[0][1] for _, kw in seen)
    with pytest.raises(ValueError):
        service.handle_submit(dict(body, topic_rf={"nope": 2}), solver)
