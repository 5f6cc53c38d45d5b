"""Instances of more than 8,160 partitions (the large path, DESIGN.md 7.1) on the host: the engine's validation
takes up to 65,280 partitions, the plain-C restatement and the model handle those sizes, and the JSON codecs carry a
many-topic `kafka-reassign-partitions --generate` document through unchanged."""
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

from kafka_assignment_optimizer_b200 import optimizer as kopt
from kafka_assignment_optimizer_b200 import problem as kprob
from oracle import model as m

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "kao-cli")


def _obj_bits(pb):
    lib = kopt.load_library()
    return lib.kao_key_obj_bits(kopt._CProblem(pb).ref()), lib.kao_last_error().decode()


@pytest.mark.parametrize("P", [8161, 65280])
def test_large_row_counts_pass_validation(P):
    bits, err = _obj_bits(m.synthetic_problem(P, 64, 8, 3, remove=1))
    assert bits > 0, err


def test_row_count_above_65280_is_refused_with_the_limit():
    bits, err = _obj_bits(m.synthetic_problem(65281, 64, 8, 3, remove=1))
    assert bits == -1 and "65280" in err


def test_restatement_and_model_at_65280_partitions(ref_lib):
    """The restatement's initial base, candidates and evaluation at the largest row count agree with the model."""
    pb = m.synthetic_problem(65280, 64, 8, 3, remove=1)
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    reps = r.decode(bits, ld)
    assert r.evaluate(bits, ld) == m.evaluate(pb, reps)
    keys = r.candidate_keys(bits, ld, 0x1A26E, 3, 64, 0, 64)
    best = int(keys.min())
    cb, cl = r.gen(bits, ld, 0x1A26E, 3, best & 0xFFFFFF, 64)
    v, o, _ = r.unpack_key(best)
    assert (v, o) == r.evaluate(cb, cl) == m.evaluate(pb, r.decode(cb, cl))
    # a partition id above 2^15 survives the round trip through the replica lists
    assert (r.encode(r.decode(cb, cl))[0] == cb).all()


def _generate_document(topics=240, parts=50, brokers=12, rf=3, seed=7):
    rng = np.random.RandomState(seed)
    doc = {"version": 1, "partitions": []}
    for t in range(topics):
        for p in range(parts):
            doc["partitions"].append({"topic": "topic-%03d" % t, "partition": p,
                                      "replicas": [int(b) for b in rng.choice(brokers, size=rf, replace=False)]})
    rng.shuffle(doc["partitions"])
    return doc


def test_many_topic_document_round_trips_through_the_python_codec():
    doc = _generate_document()
    rows, topics = kprob.parse_assignment_json(json.dumps(doc))
    assert len(rows) == 12000 > 8160
    pb = kprob.build_problem(rows, range(12), {b: "r%d" % (b % 3) for b in range(12)}, 3, topics)
    out = kprob.reassignment_json(pb, pb.cur)
    got = {(e["topic"], e["partition"]): e["replicas"] for e in out["partitions"]}
    want = {(e["topic"], e["partition"]): e["replicas"] for e in doc["partitions"]}
    assert len(out["partitions"]) == len(got) == len(want) and got == want


def test_many_topic_document_through_the_cli_lp(tmp_path):
    import __graft_entry__ as g

    if not os.path.exists(CLI):
        g.build()
    doc = _generate_document()
    f = tmp_path / "current.json"
    f.write_text(json.dumps(doc))
    racks = ",".join("%d:r%d" % (b, b % 3) for b in range(12))
    text = subprocess.check_output([CLI, "--assignment", str(f), "--brokers", ",".join(map(str, range(12))),
                                    "--racks", racks, "--emit-lp"], text=True)
    # rows in (topic, partition) order; every row appears once in the leader family, and its objective terms
    # name exactly the brokers of its replica list (the leader with weight 4)
    order = sorted(doc["partitions"], key=lambda e: (e["topic"], e["partition"]))
    objective = text.split(";", 1)[0]
    terms = {}
    for w, b, p, l in re.findall(r"(\d+) t1b(\d+)p(\d+)(_l)?", objective):
        terms.setdefault(int(p), {})[(int(b), bool(l))] = int(w)
    assert sorted(terms) == list(range(len(order)))
    for p, e in enumerate(order):
        assert {b for b, l in terms[p] if not l} == set(e["replicas"])
        assert terms[p][(e["replicas"][0], True)] == 4
    leader_rows = text.split("// Constraint on having one and only one leader per partition\n", 1)[1].split("\n\n", 1)[0]
    assert len(leader_rows.strip().split("\n")) == len(order)
