"""Per-topic balance rows (docs/MODEL.md §10) without a GPU: the restatement's evaluation equals the model with topic
rows, its search reaches the HiGHS optimum of the program with topic rows, the codec and kao-cli build the default
bounds, `kao-cli --emit-lp --topic-balance` is that program, invalid kao_topics input is refused before any CUDA call,
and the topic kernels neither spill nor change the SASS of any kernel that existed before them."""
import ctypes as C
import dataclasses
import hashlib
import json
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.optimize import Bounds, LinearConstraint, milp

import kafka_assignment_optimizer_b200 as kao
import topics_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from test_lp_text import parse_lp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "csrc")
CLI = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "kao-cli")


def readme_three_topics():
    """The README topology, broker 19 removed, 20 partitions in topics of 10, 6 and 4 (RF 3: with RF 2 the rack totals
    of 40 replicas cannot be met)."""
    cur = [[p % 20, (p + 11) % 20, (p + 2) % 20] for p in range(20)]
    topics = [("a", p) for p in range(10)] + [("b", p) for p in range(6)] + [("c", p) for p in range(4)]
    pb = m.build_problem(cur, list(range(19)), {b: ("b" if b % 2 else "a") for b in range(20)}, 3, topics=topics)
    return pb, kao.topic_rows(kao.Problem.from_fields(pb))


def sixteen_topics():
    pb = m.synthetic_problem(256, 32, 4, 3, remove=1)
    pb.topics = [("t%02d" % (p // 16), p % 16) for p in range(256)]
    return pb, kao.topic_rows(kao.Problem.from_fields(pb))


def interleaved_topics():
    """30 topics whose partitions interleave (topic = row mod 30), 3 racks of 20: padding slots"""
    from conftest import make_problem

    pb = make_problem(700, [20, 20, 20], 3, seed=5, removed=2)
    pb.topics = [("t%d" % (p % 30), p) for p in range(700)]
    return pb, kao.topic_rows(kao.Problem.from_fields(pb))


@pytest.mark.parametrize("make", [readme_three_topics, sixteen_topics, interleaved_topics])
def test_restatement_evaluation_equals_the_model(ref_lib, make):
    pb, tr = make()
    r = topics_ref.TRef(pb, tr)
    rng = np.random.RandomState(7)
    generated = r.decode(*r.init_base())
    random = np.stack([rng.choice(pb.B, size=pb.RF, replace=False) for _ in range(pb.P)]).astype(np.int32)
    malformed = random.copy()
    malformed[0, :] = malformed[0, 0]                 # duplicates collapse
    malformed[1, 1:] = -1                             # a short row
    malformed[2, :] = -1                              # an empty row: no leader
    for reps in (generated, random, malformed):
        want = topics_ref.evaluate(pb, tr, reps)
        assert r.evaluate(*r.encode(reps)) == want
        assert want[0] - m.evaluate(pb, reps)[0] == topics_ref.topic_violation(pb, tr, reps)
    assert topics_ref.topic_violation(pb, tr, random) > 0


def test_restatement_without_binding_rows_is_the_oracle(ref_lib):
    pb, tr = sixteen_topics()
    n = np.bincount(tr.topic_of).astype(np.int32)
    loose = dataclasses.replace(tr, rep_lo=0 * n, rep_hi=n * pb.RF, ldr_lo=0 * n, ldr_hi=n)
    plain, r = ref_lib.Ref(pb), topics_ref.TRef(pb, loose)
    bits, ld = plain.init_base()
    for rnd in (0, 3):
        assert (r.candidate_keys(bits, ld, 0xB16, rnd, 512, 0, 512) == plain.candidate_keys(bits, ld, 0xB16, rnd, 512, 0, 512)).all()


def test_restatement_search_reaches_the_highs_optimum(ref_lib):
    """(The 256-partition, 16-topic instance is searched to its HiGHS optimum on the GPU: tests/test_gpu_topics.py.)"""
    pb, tr = readme_three_topics()
    sol = topics_ref.solve_exact(pb, tr)
    assert sol.status == "optimal" and sol.objective == 128
    assert m.solve_exact(pb).objective == 133               # the topic rows cost objective here
    r = topics_ref.TRef(pb, tr)
    bits, ld = r.init_base()
    r.search(bits, ld, 0x5EED, 0, 300, 4096)
    assert r.evaluate(bits, ld) == (0, sol.objective)
    assert topics_ref.evaluate(pb, tr, r.decode(bits, ld)) == (0, sol.objective)


def test_default_bounds_are_the_readme_rows():
    """For the README's one topic the default rows are its C3 / C4 (README.md:158-166): 20 replicas of t1 on 19
    brokers 1..2, 10 leaders 0..1."""
    tr = kao.topic_rows(kao.Problem.from_fields(m.readme_problem()))
    assert tr.T == 1 and (tr.topic_of == 0).all()
    assert (int(tr.rep_lo[0]), int(tr.rep_hi[0]), int(tr.ldr_lo[0]), int(tr.ldr_hi[0])) == (1, 2, 0, 1)
    pb, tr = readme_three_topics()
    assert tr.names == ["a", "b", "c"]
    assert tr.rep_lo.tolist() == [1, 0, 0] and tr.rep_hi.tolist() == [2, 1, 1]     # 30, 18, 12 replicas on 19 brokers
    assert tr.ldr_lo.tolist() == [0, 0, 0] and tr.ldr_hi.tolist() == [1, 1, 1]


def _document(pb):
    return json.dumps({"version": 1, "partitions": [
        {"topic": t, "partition": q, "replicas": [int(pb.broker_ids[b]) if b >= 0 else 19 for b in pb.cur[p]]}
        for p, (t, q) in enumerate(pb.topics)]})


def test_cli_emits_the_program_with_topic_rows(tmp_path):
    import __graft_entry__ as g

    if not os.path.exists(CLI):
        g.build()
    pb, tr = readme_three_topics()
    f = tmp_path / "current.json"
    f.write_text(_document(pb))
    args = [CLI, "--assignment", str(f), "--brokers", ",".join(map(str, range(19))),
            "--racks", ",".join("%d:%s" % (b, "b" if b % 2 else "a") for b in range(20))]
    plain = subprocess.check_output(args + ["--emit-lp"], text=True)
    text = subprocess.check_output(args + ["--emit-lp", "--topic-balance"], text=True)
    # every line of the program without topic rows stays; the topic rows come as README-style lines
    head, tail = plain.split("\n// All variables are binary")
    assert text.startswith(head) and text.endswith("\n// All variables are binary" + tail)
    assert text[len(head):].count("// Constraint on min/max") == 6
    assert "// Constraint on min/max replicas of topic b per broker" in text
    names, c, A, lo, hi = parse_lp(text)
    assert len(names) == 2 * 20 * 19
    res = milp(-c, constraints=LinearConstraint(A, lo, hi), integrality=np.ones(len(names)), bounds=Bounds(0, 1))
    assert res.status == 0 and round(-res.fun) == topics_ref.solve_exact(pb, tr).objective == 128
    # the 2 * T * B topic rows, each as a <= and a >= line, with the default bounds
    assert A.shape[0] - parse_lp(plain)[2].shape[0] == 2 * 2 * 3 * 19
    # the codec groups the document's rows the same way (topics in name order)
    rows, topics = kao.problem.parse_assignment_json(_document(pb))
    assert kao.topic_rows(kao.build_problem(rows, range(19), {b: "ab"[b % 2] for b in range(20)}, 3, topics)).names == ["a", "b", "c"]


def test_invalid_topic_rows_are_refused_without_a_gpu():
    pb = kao.Problem.from_fields(m.readme_problem())
    tr = kao.topic_rows(pb)
    lib = kopt.load_library()
    cp = kopt._CProblem(pb)

    def solve(t):
        reps = np.zeros((pb.P, pb.RF), np.int32)
        opt, res = kopt._KaoOptions(1, 2, 256, 0, 0, 1, 0), kopt._KaoResult()
        res.replicas = reps.ctypes.data
        rc = lib.kao_solve_topics(cp.ref(), kopt._CTopics(t).ref(), C.byref(opt), C.byref(res))
        return rc, lib.kao_last_error().decode()

    def create(t):
        h = C.c_void_p()
        rc = lib.kao_create_topics(cp.ref(), kopt._CTopics(t).ref(), C.c_int32(0), C.byref(h))
        return rc, lib.kao_last_error().decode()

    i32 = lambda *v: np.array(v, np.int32)
    bad = [dataclasses.replace(tr, topic_of=np.full(10, 1, np.int32)),                            # topic out of range
           dataclasses.replace(tr, topic_of=np.full(10, -1, np.int32)),
           dataclasses.replace(tr, rep_lo=i32(3), rep_hi=i32(2)),                                # lo > hi
           dataclasses.replace(tr, ldr_lo=i32(-1)),                                              # lo < 0
           dataclasses.replace(tr, rep_lo=i32(21), rep_hi=i32(30)),                              # more than 10 * RF
           dataclasses.replace(tr, ldr_lo=i32(11), ldr_hi=i32(11)),                              # more than 10
           kao.TopicRows(np.zeros(10, np.int32), i32(*[0] * 11), i32(*[2] * 11), i32(*[0] * 11), i32(*[1] * 11),
                         ["t"] * 11)]                                                            # T > P
    for t in bad:
        for call in (solve, create):
            rc, msg = call(t)
            assert rc == -1 and msg.startswith("topic rows:"), (t, rc, msg)


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) or "12.9" not in subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout:
        pytest.skip("pinned for nvcc 12.9")
    return nvcc


def test_topic_instantiations_do_not_spill():
    nvcc = _nvcc()
    with tempfile.TemporaryDirectory() as d:
        out = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
                              "-Xptxas", "-dlcm=cg", "-c", "-o", os.path.join(d, "k.o"), os.path.join(CSRC, "kao_large.cu")],
                             capture_output=True, text=True, check=True).stderr
    props = re.findall(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out)
    topic = [p for p in props if re.search(r"search_large_kernelILi\dELb1E|eval_large_base_kernel|topic_", p[0])]
    # search (kTopics, with and without per-partition rows), base evaluation (with and without them), count and
    # violation kernels, 4 widths
    assert len(topic) == 24
    assert all(p[2] == "0" and p[3] == "0" for p in topic), topic


def _sass(obj):
    text = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    res, name, ins = {}, None, []
    for line in text.splitlines() + ["Function : <end>"]:
        mt = re.match(r"\s*Function : (\S+)", line)
        if mt:
            if name:
                res[re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+", "_GLOBAL__N_", name)] = ins
            name, ins = mt.group(1), []
            continue
        mt = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if mt:
            ins.append(mt.group(1).strip())
    return res


def test_plain_and_topic_kernels_keep_their_pinned_sass():
    """Every kernel of the large-path and engine objects as the build before the topic rows made it, and the topic search
    kernels as the build before the per-partition rows made them: the plain search kernel became the kTopics = false
    instantiation, with TopicArgs appended after every parameter it had, and then every search kernel became the
    kRF = false instantiation, with the rftab pointer appended."""
    _nvcc()
    pin = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_parent_large_engine.json")))
    for obj, kernels in pin["objects"].items():
        path = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "_obj", obj)
        if not os.path.exists(path) or not shutil.which("cuobjdump"):
            pytest.skip("object files of the in-tree build or cuobjdump not available")
        now = _sass(path)
        for name, want in kernels.items():
            cur = re.sub(r"search_large_kernelILi(\d)EEEv(.*)$", r"search_large_kernelILi\1ELb0EEEv\g<2>9TopicArgs", name)
            cur = re.sub(r"search_large_kernelILi(\d)ELb(\d)EEEv(.*)$", r"search_large_kernelILi\1ELb\2ELb0EEEv\g<3>PKj", cur)
            ins = now[cur]
            assert (len(ins), hashlib.sha256("\n".join(ins).encode()).hexdigest()) == (want["instructions"], want["sha256"]), name


def test_submit_passes_topic_balance_only_when_asked():
    from kafka_assignment_optimizer_b200 import service

    seen = []

    def solver(pb, **kw):
        seen.append(kw)
        return kopt.SolveResult(np.zeros((pb.P, pb.RF), np.int32), 0, 0, 0, True, 0, 0, 0, 0.0, 0.0)

    pb, _ = readme_three_topics()
    body = {"assignment": json.loads(_document(pb)), "brokers": ",".join(map(str, range(19))),
            "racks": {b: "ab"[b % 2] for b in range(20)}, "rf": 3}
    service.handle_submit(body, solver)
    service.handle_submit(dict(body, topic_balance=True), solver)
    assert "topic_balance" not in seen[0] and seen[1]["topic_balance"] is True
