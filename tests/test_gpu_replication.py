"""Per-partition replication rows (docs/MODEL.md §11) on the GPU: kao_create_replication sessions against the
restatement (tests/rf_ref) below and above 8,160 rows, at every row width, with padding slots, dense weights and topic
rows; uniform rows against a plain session's delta search; kao_solve_replication against HiGHS."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import rf_ref
from test_replication_cpu import changed_rf, readme_mixed, uniform

pytestmark = pytest.mark.gpu
SEED = 0x5EED


def mixed(P, B0, R, remove=1, dense=False):
    """A synthetic cluster at RF 3 whose partitions keep 3, 2 or 1 replicas (every 7th RF 1, every 4th RF 2)."""
    pb = kao.synthetic_problem(P, B0, R, 3, remove=remove)
    p = np.arange(P)
    rf = np.where(p % 7 == 0, 1, np.where(p % 4 == 0, 2, 3)).astype(np.int32)
    pb.replication = kao.ReplicationRows(rf, (rf // R).astype(np.int32), (-(-rf // R)).astype(np.int32))
    if dense:
        pb.wF[:, :6] += 1                              # six weighted brokers per row: the dense table
    return pb


SHAPES = {
    "readme_mixed": (lambda: readme_mixed(), False, 4096),
    "changed_rf": (lambda: changed_rf(), True, 4096),
    "w1": (lambda: mixed(500, 20, 2), False, 4096),
    "w2_padding_topics": (lambda: mixed(700, 30, 3, remove=2), True, 4096),
    "w4": (lambda: mixed(1200, 96, 12), False, 4096),
    "w8_topics": (lambda: mixed(1000, 200, 25), True, 2048),
    "dense": (lambda: mixed(900, 30, 3, dense=True), False, 4096),
    "large_topics": (lambda: mixed(9000, 60, 3), True, 1024),
    "large": (lambda: mixed(8500, 64, 8), False, 1024),
}


def setup(name):
    make, topics, rs = SHAPES[name]
    pb = make()
    tr = kao.topic_rows(pb) if topics else None
    return pb, tr, rs, kao.Session(pb, device=0, topics=tr), rf_ref.RRef(pb, pb.replication, tr)


def damaged(pb, r):
    """The initial base with rows longer and shorter than their rf[p], and replicas moved"""
    reps = r.decode(*r.init_base())
    rng = np.random.RandomState(11)
    for p in rng.choice(pb.P, size=min(pb.P, 40), replace=False):
        k = int((reps[p] >= 0).sum())
        if p % 3 == 0 and k < pb.RF:                    # longer than rf[p]
            reps[p, k] = next(b for b in range(pb.B) if b not in reps[p])
        elif p % 3 == 1 and k > 1:                      # shorter
            reps[p, k - 1] = -1
        else:                                           # a replica moved
            reps[p, 0] = next(b for b in rng.permutation(pb.B) if b not in reps[p])
    return reps


@pytest.mark.parametrize("name", list(SHAPES))
def test_keys_trajectory_and_base_equal_the_restatement(name):
    pb, tr, rs, s, r = setup(name)
    with pytest.raises(kao.KaoError, match="per-partition replication factors"):
        s.set_evaluator(False)                                      # the HBM-base path, delta evaluation only
    bits, ld = r.init_base()
    reps, viol, obj, _ = s.get_base()
    assert (reps == r.decode(bits, ld)).all() and (viol, obj) == r.evaluate(bits, ld)
    assert ((reps >= 0).sum(axis=1) == pb.replication.rf).all()
    for base in ("initial", "damaged"):
        if base == "damaged":
            d = damaged(pb, r)
            s.set_base(d)
            bits, ld = r.encode(d)
            got = s.get_base()
            assert (got[0] == r.decode(bits, ld)).all() and got[1:3] == r.evaluate(bits, ld)
        for rnd in (0, 1):                                          # a free round and a cycle round
            want = r.candidate_keys(bits, ld, SEED, rnd, rs, 0, rs)
            assert (s.candidate_keys_delta(SEED, rnd, rs, 0, rs) == want).all(), (name, base, rnd)
        keys, _ = s.search_delta(SEED, 0, 8, rs)
        _, want = r.search(bits, ld, SEED, 0, 8, rs)
        assert (keys == want).all(), (name, base)
        got = s.get_base()
        assert (got[0] == r.decode(bits, ld)).all() and got[1:3] == r.evaluate(bits, ld)
    s.close()


@pytest.mark.parametrize("name", ["w2_padding_topics", "w8_topics", "large"])
def test_uniform_rows_equal_a_plain_session(name):
    make, topics, rs = SHAPES[name]
    pb = make()
    tr = kao.topic_rows(pb) if topics else None
    pb.replication = None
    plain = kao.Session(pb, device=0, topics=tr)
    pb.replication = uniform(pb)
    rows = kao.Session(pb, device=0, topics=tr)
    for rnd in (0, 1):
        assert (rows.candidate_keys_delta(SEED, rnd, rs, 0, rs) == plain.candidate_keys_delta(SEED, rnd, rs, 0, rs)).all()
    a, _ = rows.search_delta(SEED, 0, 8, rs)
    b, _ = plain.search_delta(SEED, 0, 8, rs)
    assert (a == b).all() and (rows.get_base()[0] == plain.get_base()[0]).all()
    rows.close()
    plain.close()


@pytest.mark.parametrize("make", [readme_mixed, changed_rf])
def test_solve_reaches_the_highs_optimum(make):
    pb = make()
    sol = rf_ref.solve_exact(pb, pb.replication)
    res = kao.optimizer.solve(pb, rounds=400, round_size=4096, tight_bound=True)
    assert res.feasible and res.objective == sol.objective
    assert ((res.replicas >= 0).sum(axis=1) == pb.replication.rf).all()
    assert rf_ref.evaluate(pb, pb.replication, res.replicas) == (0, sol.objective)
    assert res.objective <= res.objective_bound and res.optimal == (res.objective == res.objective_bound)
    again = kao.optimizer.solve(pb, rounds=400, round_size=4096, restarts=3)
    spread = kao.optimizer.solve(pb, rounds=400, round_size=4096, restarts=3, spread_restarts=True)
    assert again.objective == sol.objective and (again.replicas == spread.replicas).all()
    import torch

    if torch.cuda.device_count() > 1:
        multi = kao.optimizer.solve(pb, rounds=400, round_size=4096, restarts=3, spread_restarts=True, n_gpus=2)
        assert (multi.replicas == again.replicas).all()


def test_optimizer_keeps_every_topic_rf():
    import json

    from test_replication_cpu import RACKS, readme_mixed_document

    rows, topics = readme_mixed_document()
    doc = {"version": 1, "partitions": [{"topic": t, "partition": q, "replicas": r} for r, (t, q) in zip(rows, topics)]}
    opt = kao.AssignmentOptimizer(rounds=400, round_size=4096)
    out, res = opt.optimize(json.dumps(doc), ",".join(map(str, range(19))), RACKS, keep_rf=True)
    assert res.feasible
    want = {(t, q): len(r) for r, (t, q) in zip(rows, topics)}
    assert all(len(e["replicas"]) == want[(e["topic"], e["partition"])] for e in out["partitions"])
    assert all(19 not in e["replicas"] for e in out["partitions"])


@pytest.mark.parametrize("extra", [["--keep-rf"], ["--keep-rf", "--topic-balance"], ["--topic-rf", "x.y.z.t:3,a3:2"]])
def test_cli_keeps_every_topic_rf(tmp_path, extra):
    import json
    import subprocess

    from test_replication_cli import CLI, _doc
    from test_replication_cpu import RACKS

    doc = _doc()
    f = tmp_path / "current.json"
    f.write_text(json.dumps(doc))
    out = subprocess.run([CLI, "--assignment", str(f), "--brokers", ",".join(map(str, range(19))),
                          "--racks", ",".join("%d:%s" % (b, RACKS[b]) for b in range(20)), "--rounds", "400",
                          "--round-size", "4096", "--certificate", "--stats"] + extra, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr                  # 0: a feasible reassignment (3: none found)
    want = {(e["topic"], e["partition"]): len(e["replicas"]) for e in doc["partitions"]}
    if extra[0] == "--topic-rf":
        want = {k: {"x.y.z.t": 3, "a3": 2}.get(k[0], v) for k, v in want.items()}
    got = json.loads(out.stdout)["partitions"]
    assert len(got) == len(want)
    for e in got:
        assert len(set(e["replicas"])) == len(e["replicas"]) == want[(e["topic"], e["partition"])], e
        assert 19 not in e["replicas"]
