"""Clusters that use all 256 broker slots, without a GPU.  Slot 255 is then a real broker while several tables use the
byte 0xFF for "none" or "padding" (DESIGN.md 7.1).  MODEL §4's initial base written out in Python must equal the
restatements' and the engine host code's on every shape, including partitions led from slot 255 whose rows get
completed; the committed golden streams must still be what the restatement computes; and the topic rows of the
HBM-base kernels (csrc/kao_topics.cuh, compiled for the host by the emulator) must count the broker on slot 255 in
their evaluations, delta keys and walks, as the restatement does."""
import importlib.util
import json
import os

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import topics_ref
from emu import EmuSession
from oracle import model as m
from problems import (C7_SHAPES, HOME255_SHAPES, LARGE_SHAPES, LAYOUT_SHAPES, LEADER255_SHAPES, SHAPES, SLOT255_SHAPES,
                      SLOT255_TOPIC_SHAPES, emptied_base, home255_bases, moved_base, slots)
from test_topics_cpu import interleaved_topics, sixteen_topics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EVERY = {**SHAPES, **LAYOUT_SHAPES, **C7_SHAPES, **LARGE_SHAPES, **SLOT255_SHAPES, **LEADER255_SHAPES, **HOME255_SHAPES}


def model4_initial_base(pb):
    """docs/MODEL.md §4 as written: cur[p] restricted to the target brokers, order kept, leader = first survivor,
    replicas beyond RF dropped from the tail; then rows short of RF completed, partitions in ascending order, one
    replica at a time on the broker minimising (replicas of p in its rack, replicas placed on it so far, broker index).
    -> (leader broker per partition, -1 for none; replica set per partition)"""
    load = [0] * pb.B
    rows, leader = [], []
    for p in range(pb.P):
        row = []
        for b in pb.cur[p]:
            if 0 <= b < pb.B and b not in row and len(row) < pb.RF:
                row.append(int(b))
                load[b] += 1
        rows.append(row)
        leader.append(row[0] if row else -1)
    for p in range(pb.P):
        row = rows[p]
        while len(row) < min(pb.RF, pb.B):
            in_rack = np.bincount(pb.rack_of[row], minlength=pb.R) if row else np.zeros(pb.R, int)
            best = min((b for b in range(pb.B) if b not in row), key=lambda b: (in_rack[pb.rack_of[b]], load[b], b))
            row.append(best)
            load[best] += 1
            if leader[p] < 0:
                leader[p] = best
    return leader, [set(r) for r in rows]


def completed_from_255(pb):
    """partitions whose first survivor sits on slot 255 and whose row is completed by MODEL §4"""
    slot = slots(pb)
    out = []
    for p in range(pb.P):
        alive = list(dict.fromkeys(int(b) for b in pb.cur[p] if 0 <= b < pb.B))
        if alive and slot[alive[0]] == 255 and len(alive) < pb.RF:
            out.append(p)
    return out


def assert_model4(pb, reps, what):
    leader, rows = model4_initial_base(pb)
    for p in range(pb.P):
        got = [int(b) for b in reps[p] if b >= 0]
        assert (got[0] if got else -1, set(got)) == (leader[p], rows[p]), (what, p, got, leader[p], sorted(rows[p]))


@pytest.mark.parametrize("name", sorted(EVERY))
def test_initial_base_is_model_section_4(ref_lib, name):
    """The restatement (oracle/kao_ref.c), the per-partition-rows restatement with uniform rows (tests/rf_ref) and the
    engine's host code (kao_host.hpp initial_base, through the emulator) against MODEL §4 written out above"""
    import rf_ref

    pb = EVERY[name]()
    r = ref_lib.Ref(pb)
    assert_model4(pb, r.decode(*r.init_base()), "kao_ref")
    rf = np.full(pb.P, min(pb.RF, pb.B - 1), np.int32)
    rr = kao.ReplicationRows(rf, np.full(pb.P, pb.ppr_lo, np.int32), np.full(pb.P, pb.ppr_hi, np.int32))
    rref = rf_ref.RRef(pb, rr)
    assert_model4(pb, rref.decode(*rref.init_base()), "rf_ref")
    loose = kao.TopicRows(np.zeros(pb.P, np.int32), [0], [pb.P * pb.RF], [0], [pb.P], ["all"])
    sess = EmuSession(pb, topics=loose)
    assert_model4(pb, sess.get_base()[0], "host initial_base")
    sess.close()
    if name in LEADER255_SHAPES:
        assert len(completed_from_255(pb)) >= 2


def test_leader_on_slot_255_keeps_its_leadership(ref_lib):
    """The case that shows the difference: RF 2 -> 3 on 256 brokers, partitions 255 and 511 on [255, 0]"""
    pb = LEADER255_SHAPES["leader255_rf_up"]()
    assert completed_from_255(pb) == [255, 511]
    reps = ref_lib.Ref(pb).decode(*ref_lib.Ref(pb).init_base())
    assert reps[255, 0] == reps[511, 0] == 255
    assert completed_from_255(LEADER255_SHAPES["leader255_removed"]()) == [255, 515]


def test_golden_streams_are_what_the_restatement_computes(ref_lib):
    """tests/golden/streams.json regenerated in memory equals the committed file: no golden shape completes a row
    led from slot 255 (checked), so the initial bases and everything after them are unchanged"""
    for name in SHAPES:
        assert completed_from_255(SHAPES[name]()) == [], name
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(ROOT, "tests", "golden", "make_golden.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    with open(os.path.join(ROOT, "tests", "golden", "streams.json")) as f:
        assert json.loads(json.dumps(mg.streams())) == json.load(f)


def test_slot255_shapes_are_never_skipped(ref_lib):
    """Every 256-slot shape puts broker 255 on slot 255.  The grown-by-one walk shapes leave it empty; the home-255
    shapes give it home replicas, and the initial base of each has targeted bases whose displaced lists are made of
    home-255 partitions only (problems.home255_bases checks them); the initial-base shapes lead from slot 255."""
    for name, f in {**SLOT255_SHAPES, **SLOT255_TOPIC_SHAPES, **HOME255_SHAPES}.items():
        pb = f()
        slot = slots(pb)
        assert pb.B == 256 and sorted(slot) == list(range(256)) and slot[255] == 255, name
        on_255 = (slot[pb.cur[(pb.cur >= 0) & (pb.cur < pb.B)]] == 255).sum()
        assert (on_255 > 0) == (name in HOME255_SHAPES), name
    for name, f in HOME255_SHAPES.items():
        pb = f()
        r = ref_lib.Ref(pb)
        assert r.W == 8, name
        got = home255_bases(pb, r.decode(*r.init_base()))
        assert set(got) == ({"d255"} if name == "h255_rf_down" else {"d255", "dl255"}), name
    for name, f in LEADER255_SHAPES.items():
        pb = f()
        assert slots(pb)[255] == 255 and (slots(pb)[pb.cur[:, 0][pb.cur[:, 0] >= 0]] == 255).any(), name


def test_topic_shapes_bind_on_broker_255():
    """Every topic has n RF >= 256 replicas: its default C3t lower bound is at least 1, and the initial base leaves
    broker 255 empty, so every topic's row on broker 255 is violated"""
    for name, f in SLOT255_TOPIC_SHAPES.items():
        pb = f()
        tr = kao.topic_rows(kao.Problem.from_fields(pb))
        n = np.bincount(tr.topic_of)
        assert (n * pb.RF >= 256).all() and (tr.rep_lo >= 1).all(), name
        assert 50 <= n.min() and n.max() <= 600 or tr.T == 1, name


# ---- topic rows on the HBM-base kernels' code, compiled for the host ----------------------------------------------
def topic_cases():
    """(pb, topic rows) at W 1 / 2 / 4 / 8; the eight-word ones use every slot and bind on broker 255"""
    def with_topics(pb, label):
        pb.topics = label
        return pb, kao.topic_rows(kao.Problem.from_fields(pb))

    cases = {"w1_sixteen": sixteen_topics, "w4_interleaved": interleaved_topics,
             "w2_cfg3_small": lambda: with_topics(SHAPES["cfg3_small"](), [("t%d" % (p % 7), p) for p in range(200)])}
    for name in ("one_topic_r16", "sized_r32", "sized_r4"):
        cases["w8_" + name] = lambda n=name: (lambda pb: (pb, kao.topic_rows(kao.Problem.from_fields(pb))))(SLOT255_TOPIC_SHAPES[n]())
    return cases


TOPIC_CASES = topic_cases()


def keys_round(sess, r, bits, ld, seed, rnd, size, what):
    got = sess.candidate_keys(seed, rnd, size, 0, size, delta=True)
    want = r.candidate_keys(bits, ld, seed, rnd, size, 0, size)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (what, rnd, int(bad[0]), int(got[bad[0]]), int(want[bad[0]]))


@pytest.mark.parametrize("name", sorted(TOPIC_CASES))
def test_emulated_topic_sessions_equal_the_restatement(ref_lib, name):
    """get_base against the model with topic rows, delta keys of a free and a cycle round against the restatement from
    the initial, moved and emptied bases, and a 48-round walk (the counts patched winner by winner) against the
    restatement's, its final base against the model"""
    pb, tr = TOPIC_CASES[name]()
    r = topics_ref.TRef(pb, tr)
    reps = r.decode(*r.init_base())
    assert r.W == {"w1": 1, "w2": 2, "w4": 4, "w8": 8}[name[:2]]
    if name.startswith("w8"):
        assert topics_ref._topic_counts(pb, tr, reps)[0][:, 255].sum() == 0      # the new broker starts empty
    sess = EmuSession(pb, topics=tr)
    for what, b in (("initial", reps), ("moved", moved_base(pb, reps, 6)), ("emptied", emptied_base(pb, reps, 5))):
        sess.set_base(b)
        bits, ld = r.encode(b)
        got_reps, v, o, _ = sess.get_base()
        assert (got_reps == r.decode(bits, ld)).all(), what
        assert (v, o) == r.evaluate(bits, ld) == topics_ref.evaluate(pb, tr, got_reps), what
        for rnd in (4, 7):
            keys_round(sess, r, bits, ld, 0xB16, rnd, 1024, what)
    for what, start in (("initial", reps), ("moved", moved_base(pb, reps, 6))):
        sess.set_base(start)
        bits, ld = r.encode(start)
        _, want = r.search(bits, ld, 0x5EED, 0, 48, 256)
        got = sess.search(0x5EED, 0, 48, 256)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (what, "walk round", int(bad[0]))
        end, v, o, _ = sess.get_base()
        assert (end == r.decode(bits, ld)).all() and (v, o) == topics_ref.evaluate(pb, tr, end), what
        keys_round(sess, r, bits, ld, 0x5EED, 48, 1024, (what, "after the walk"))
    sess.close()
