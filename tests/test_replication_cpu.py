"""Per-partition replication rows (docs/MODEL.md §11) without a GPU: the restatement's evaluation equals the model on
mixed-RF instances, its keys equal the oracle's with uniform rows, its search reaches the HiGHS optimum, the bounds
bracket that optimum, the codec keeps every topic's RF only when asked, invalid kao_replication input is refused
before any CUDA call, and the new kernels do not spill."""
import ctypes as C
import dataclasses
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import rf_ref
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from oracle import ref as oref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "csrc")
RACKS = {b: ("b" if b % 2 else "a") for b in range(20)}


def readme_mixed(topic_rf=None):
    """The README example (topic x.y.z.t, RF 2, broker 19 removed) plus an RF-3 topic of 4 partitions and an RF-1
    topic of 3 partitions on the same brokers; every topic keeps its RF (or takes topic_rf's)."""
    rows, topics = readme_mixed_document()
    return kao.build_problem(rows, range(19), RACKS, None, topics, keep_rf=topic_rf is None, topic_rf=topic_rf)


def readme_mixed_document():
    """(replica lists by Kafka broker id, (topic, partition) labels) of readme_mixed"""
    readme = [[7, 18], [8, 19], [9, 10], [0, 11], [1, 12], [2, 13], [3, 14], [4, 15], [5, 16], [6, 17]]
    three = [[(3 * p + 1) % 20, (3 * p + 6) % 20, (3 * p + 11) % 20] for p in range(4)]
    one = [[(5 * p + 2) % 20] for p in range(3)]
    rows = readme + three + one
    topics = [("x.y.z.t", p) for p in range(10)] + [("a3", p) for p in range(4)] + [("b1", p) for p in range(3)]
    return rows, topics


def changed_rf():
    """The same document with x.y.z.t raised to RF 3 and a3 lowered to RF 2 (b1 keeps RF 1)."""
    return readme_mixed({"x.y.z.t": 3, "a3": 2, "b1": 1})


def uniform(pb):
    return kao.ReplicationRows(np.full(pb.P, pb.RF, np.int32), np.full(pb.P, pb.ppr_lo, np.int32),
                               np.full(pb.P, pb.ppr_hi, np.int32))


def test_builder_keeps_every_topic_rf():
    pb = readme_mixed()
    assert pb.RF == 3 and pb.replication.rf.tolist() == [2] * 10 + [3] * 4 + [1] * 3
    assert pb.replication.ppr_lo.tolist() == [1] * 10 + [1] * 4 + [0] * 3
    assert pb.replication.ppr_hi.tolist() == [1] * 10 + [2] * 4 + [1] * 3
    tot = 20 + 12 + 3
    assert (pb.rep_lo == tot // 19).all() and (pb.rep_hi == -(-tot // 19)).all()
    assert changed_rf().replication.rf.tolist() == [3] * 10 + [2] * 4 + [1] * 3
    # one RF everywhere: the plain problem, no per-partition rows
    rows, topics = [[0, 1], [2, 3]], [("t", 0), ("t", 1)]
    plain = kao.build_problem(rows, range(6), {b: "r%d" % (b % 2) for b in range(6)}, 2, topics)
    kept = kao.build_problem(rows, range(6), {b: "r%d" % (b % 2) for b in range(6)}, None, topics, keep_rf=True)
    assert kept.replication is None and kept.RF == 2 and (kept.rep_lo == plain.rep_lo).all()
    # the topic rows follow the per-partition factors: x.y.z.t holds 20 replicas, a3 12, b1 3 on 19 brokers
    tr = kao.topic_rows(pb)
    assert tr.rep_lo.tolist() == [1, 0, 0] and tr.rep_hi.tolist() == [2, 1, 1]


@pytest.mark.parametrize("make", [readme_mixed, changed_rf])
def test_restatement_evaluation_equals_the_model(make):
    pb = make()
    rr = pb.replication
    rng = np.random.RandomState(3)
    for tr in (None, kao.topic_rows(pb)):
        r = rf_ref.RRef(pb, rr, tr)
        generated = r.decode(*r.init_base())
        random = np.stack([rng.choice(pb.B, size=pb.RF, replace=False) for _ in range(pb.P)]).astype(np.int32)
        damaged = random.copy()
        damaged[0, :] = damaged[0, 0]                 # duplicates collapse
        damaged[1, 1:] = -1                           # short
        damaged[2, :] = -1                            # empty: no leader
        damaged[15, 1:] = -1                          # the RF-1 topic at its own length
        for reps in (generated, random, damaged):
            assert r.evaluate(*r.encode(reps)) == rf_ref.evaluate(pb, rr, reps, tr)
    # the initial base keeps every row at its own RF
    r = rf_ref.RRef(pb, rr)
    gen = r.decode(*r.init_base())
    assert ((gen >= 0).sum(axis=1) == rr.rf).all()


def test_uniform_rows_are_the_oracle():
    for pb in (m.readme_problem(), m.synthetic_problem(256, 32, 4, 3, remove=1)):
        plain, r = oref.Ref(pb), rf_ref.RRef(pb, uniform(pb))
        bits, ld = plain.init_base()
        b2, l2 = r.init_base()
        assert (bits == b2).all() and (ld == l2).all()
        for rnd in (0, 3):
            assert (r.candidate_keys(bits, ld, 0xB16, rnd, 512, 0, 512) == plain.candidate_keys(bits, ld, 0xB16, rnd, 512, 0, 512)).all()


@pytest.mark.parametrize("make", [readme_mixed, changed_rf])
def test_restatement_search_reaches_the_highs_optimum(make):
    pb = make()
    sol = rf_ref.solve_exact(pb, pb.replication)
    assert sol.status == "optimal"
    assert ((sol.replicas >= 0).sum(axis=1) == pb.replication.rf).all()
    r = rf_ref.RRef(pb, pb.replication)
    bits, ld = r.init_base()
    r.search(bits, ld, 0x5EED, 0, 400, 4096)
    assert r.evaluate(bits, ld) == (0, sol.objective)
    assert rf_ref.evaluate(pb, pb.replication, r.decode(bits, ld)) == (0, sol.objective)


def _bound(pb, rr, replicas=None):
    out = C.c_int64()
    rp = None if rr is None else kopt._CReplication(rr).ref()
    reps = None if replicas is None else np.ascontiguousarray(replicas, np.int32)
    rc = kopt.load_library().kao_objective_bound_replication(kopt._CProblem(pb).ref(), rp,
                                                            None if reps is None else C.c_void_p(reps.ctypes.data),
                                                            C.byref(out))
    assert rc == 0, kopt.load_library().kao_last_error()
    return out.value


def seeded_mixed(seed, racks, topics, removed=0):
    """Brokers 0.. in racks of the given sizes (interleaved), the last `removed` of them leaving; topics: (partitions,
    rf) pairs, each partition on rf random brokers; every topic keeps its RF (build_problem(keep_rf=True))."""
    rng = np.random.RandomState(seed)
    rack = [r for i in range(max(racks)) for r in range(len(racks)) if i < racks[r]]
    B = len(rack)
    rows, labels = [], []
    for t, (n, rf) in enumerate(topics):
        rows += [[int(b) for b in rng.choice(B, size=rf, replace=False)] for _ in range(n)]
        labels += [("t%d" % t, q) for q in range(n)]
    return kao.build_problem(rows, range(B - removed), {b: "r%d" % rack[b] for b in range(B)}, None, labels,
                             keep_rf=True)


BOUND_INSTANCES = {
    "readme_mixed": readme_mixed,
    "changed_rf": changed_rf,
    "lo_above_0": lambda: seeded_mixed(1, [3, 3], [(4, 3), (3, 2), (2, 1)]),         # two racks: C7 1..2 / 1..1
    "one_rack": lambda: seeded_mixed(2, [5], [(3, 3), (4, 1), (2, 2)]),               # C7 lo = hi = rf[p]
    "rf1_partitions": lambda: seeded_mixed(3, [3, 3, 3], [(6, 1), (4, 3)], removed=1),
    "rf_b_minus_1": lambda: seeded_mixed(4, [2, 2], [(3, 3), (3, 1)]),                # four brokers, rf 3
    "three_factors": lambda: seeded_mixed(5, [3, 3, 2], [(3, 3), (4, 2), (3, 1)], removed=1),
    "unequal_racks": lambda: seeded_mixed(6, [4, 2, 3], [(5, 2), (3, 3), (2, 1)]),
}


@pytest.mark.parametrize("name", sorted(BOUND_INSTANCES))
def test_bounds_bracket_the_optimum(name):
    """kao_solve_replication certifies optimality when a result reaches the cheap bound: both bounds must lie at or
    above the HiGHS optimum on every instance"""
    pb = BOUND_INSTANCES[name]()
    assert pb.replication is not None
    sol = rf_ref.solve_exact(pb, pb.replication)
    assert sol.status == "optimal", sol.status
    cheap = _bound(pb, pb.replication)
    flow = _bound(pb, pb.replication, sol.replicas)
    assert sol.objective <= flow <= cheap
    assert kao.objective_bound(pb) == cheap and kao.objective_bound(pb, sol.replicas) == flow


def test_uniform_rows_give_the_plain_bound():
    for opb in (m.readme_problem(), m.synthetic_problem(256, 32, 4, 3, remove=1)):
        pb = kao.Problem.from_fields(opb)
        feas = m.solve_exact(opb).replicas if pb.P <= 20 else None
        for reps in (None, feas):
            assert _bound(pb, uniform(pb), reps) == _bound(pb, None, reps) == kao.objective_bound(pb, reps)


def test_invalid_replication_rows_are_refused_without_a_gpu():
    pb = readme_mixed()
    rr = pb.replication
    lib = kopt.load_library()
    cp = kopt._CProblem(pb)
    tr = kao.topic_rows(pb)

    def calls(r, t=None):
        ct = kopt._CTopics(t)
        cr = kopt._CReplication(r)
        reps = np.zeros((pb.P, pb.RF), np.int32)
        opt, res = kopt._KaoOptions(1, 2, 256, 0, 0, 1, 0), kopt._KaoResult()
        res.replicas = reps.ctypes.data
        h = C.c_void_p()
        out = []
        out.append((lib.kao_solve_replication(cp.ref(), ct.ref(), cr.ref(), C.byref(opt), C.byref(res)), lib.kao_last_error().decode()))
        out.append((lib.kao_create_replication(cp.ref(), ct.ref(), cr.ref(), C.c_int32(0), C.byref(h)), lib.kao_last_error().decode()))
        return out

    n = pb.P
    bad = [dataclasses.replace(rr, rf=np.where(np.arange(n) == 4, 0, rr.rf).astype(np.int32)),        # rf < 1
           dataclasses.replace(rr, rf=np.where(np.arange(n) == 4, 4, rr.rf).astype(np.int32)),        # rf > RF
           dataclasses.replace(rr, ppr_lo=np.where(np.arange(n) == 4, 2, rr.ppr_lo).astype(np.int32)),  # lo > hi
           dataclasses.replace(rr, ppr_hi=np.full(n, 128, np.int32)),                                 # hi > 127
           dataclasses.replace(rr, ppr_lo=np.full(n, -1, np.int32))]
    # lo > 63: four 8-slot racks' deficits would wrap the byte they are summed in (docs/MODEL.md §1)
    for lo in (64, 127):
        bad.append(dataclasses.replace(rr, ppr_lo=np.where(np.arange(n) == 4, lo, rr.ppr_lo).astype(np.int32),
                                       ppr_hi=np.where(np.arange(n) == 4, 127, rr.ppr_hi).astype(np.int32)))
    for r in bad:
        for rc, msg in calls(r):
            assert rc == -1 and msg.startswith("per-partition replication factors:"), (rc, msg)
    # the same limit on the problem's own C7, with and without per-partition rows
    h = C.c_void_p()
    for lo in (64, 127):
        cpl = kopt._CProblem(dataclasses.replace(pb, ppr_lo=lo, ppr_hi=127))
        rcs = [lib.kao_create(cpl.ref(), C.c_int32(0), C.byref(h)),
               lib.kao_create_replication(cpl.ref(), None, kopt._CReplication(rr).ref(), C.c_int32(0), C.byref(h))]
        msg = lib.kao_last_error().decode()
        assert rcs == [-1, -1] and msg.startswith("bad per-partition-per-rack bounds"), (rcs, msg)
    cpl = kopt._CProblem(dataclasses.replace(pb, ppr_lo=63, ppr_hi=127))
    assert lib.kao_key_obj_bits(cpl.ref()) > 0
    # a topic row whose lo exceeds the sum of its partitions' factors (b1: 3 replicas)
    t = dataclasses.replace(tr, rep_lo=np.array([0, 0, 4], np.int32), rep_hi=np.array([9, 9, 9], np.int32))
    for rc, msg in calls(rr, t):
        assert rc == -1 and msg.startswith("topic rows:") and "replication factors" in msg, (rc, msg)
    # rf above B - 1: 3 brokers, RF 3
    small = kao.build_problem([[0, 1, 2], [0, 1]], range(3), {0: "a", 1: "b", 2: "c"}, None,
                              [("t", 0), ("u", 0)], keep_rf=True)
    assert small.replication is not None
    cps = kopt._CProblem(small)
    out = C.c_int64()
    assert lib.kao_objective_bound_replication(cps.ref(), kopt._CReplication(small.replication).ref(), None, C.byref(out)) == -1
    # the LP bound is not offered with per-partition rows
    reps = np.zeros((pb.P, pb.RF), np.int32)
    opt, res = kopt._KaoOptions(1, 2, 256, 0, 0x1000, 1, 0), kopt._KaoResult()
    res.replicas = reps.ctypes.data
    rc = lib.kao_solve_replication(cp.ref(), None, kopt._CReplication(rr).ref(), C.byref(opt), C.byref(res))
    assert rc == -1 and "KAO_FLAG_LP_BOUND" in lib.kao_last_error().decode()


def test_replication_instantiations_do_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) or "12.9" not in subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout:
        pytest.skip("pinned for nvcc 12.9")
    with tempfile.TemporaryDirectory() as d:
        out = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v",
                              "-Xptxas", "-dlcm=cg", "-c", "-o", os.path.join(d, "k.o"), os.path.join(CSRC, "kao_large.cu")],
                             capture_output=True, text=True, check=True).stderr
    props = re.findall(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out)
    new = [p for p in props if re.search(r"search_large_kernelILi\dELb\dELb1E|eval_large_base_kernelILi\dELb1E", p[0])]
    assert len(new) == 12                                   # search (with and without topic rows) and eval, 4 widths
    assert all(p[2] == "0" and p[3] == "0" for p in new), new
