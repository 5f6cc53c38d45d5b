"""Home replicas on slot 255, without a GPU: the engine's generator, displaced-list builders and evaluators compiled for
the host (tests/emu) on 256-broker clusters where broker 255 holds current replicas (problems.HOME255_SHAPES).  When
every slot is a broker the home byte 0xFF is slot 255 itself, so the guided operations and the displaced lists must
tell "slot 255" from "no home" as docs/MODEL.md §5.1 does.  From bases whose lists hold only partitions displaced from
slot 255 (problems.home255_bases), keys of a free and a cycle round and walks are held bit for bit to the restatement
(oracle/kao_ref.c), and the lists a walk patched to the lists rebuilt from its base."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from emu import EmuSession
from oracle import model as m
from problems import HOME255_SHAPES, home255_bases
from test_gpu_large_layouts import assert_keys, one_loose_topic

BIG = 8160
SIZE = 256                          # candidates per round of the key checks
WALK = (24, 128)                    # rounds x candidates of a walk
CHECK = 8                           # rounds between state checks of the row-major walk


def starts(pb, r):
    reps = r.decode(*r.init_base())
    return {"initial": reps, **home255_bases(pb, reps)}


@pytest.mark.parametrize("name", sorted(HOME255_SHAPES))
def test_emulated_keys_from_home255_bases(ref_lib, name):
    """Keys of a free round and a cycle round from the initial and the targeted bases: the row-major evaluator and the
    delta keys of a plain session (up to 8,160 partitions), and the HBM-base kernels' delta keys (a loose-topic session)"""
    pb = HOME255_SHAPES[name]()
    r = ref_lib.Ref(pb)
    sessions = {"hbm": EmuSession(pb, topics=one_loose_topic(pb))}
    if pb.P <= BIG:
        sessions["plain"] = EmuSession(kao.Problem.from_fields(pb))
    for what, b in starts(pb, r).items():
        bits, ld = r.encode(b)
        for rnd in (4, 7):
            want = r.candidate_keys(bits, ld, 0xB16, rnd, SIZE, 0, SIZE)
            for who, sess in sessions.items():
                sess.set_base(b)
                if who == "plain":
                    assert_keys(sess.candidate_keys(0xB16, rnd, SIZE, 0, SIZE), want, (what, who, rnd))
                assert_keys(sess.candidate_keys(0xB16, rnd, SIZE, 0, SIZE, delta=True), want, (what, who, "delta", rnd))
    for sess in sessions.values():
        sess.close()


@pytest.mark.parametrize("name", sorted(HOME255_SHAPES))
def test_emulated_walks_from_home255_bases(ref_lib, name):
    """Walks from the targeted bases against the restatement: the row-major search with its patched lists checked
    against the rebuilt ones every few rounds (up to 8,160 partitions), and the HBM-base search; the walked base
    equals the restatement's and the model's evaluation"""
    pb = HOME255_SHAPES[name]()
    r = ref_lib.Ref(pb)
    rounds, size = WALK
    for what, start in starts(pb, r).items():
        if what == "initial" and name != "h255_rf_down":
            continue                            # no displaced partition: the targeted bases are the cases
        seed = 0x5EED + len(what)
        bits, ld = r.encode(start)
        _, want = r.search(bits, ld, seed, 0, rounds, size)
        runs = {"hbm": EmuSession(pb, topics=one_loose_topic(pb))}
        if pb.P <= BIG:
            runs["row_major"] = EmuSession(kao.Problem.from_fields(pb))
        for who, sess in runs.items():
            sess.set_base(start)
            step = CHECK if who == "row_major" else rounds
            for first in range(0, rounds, step):
                assert_keys(sess.search(seed, first, step, size), want[first:first + step], (what, who, first))
                if who == "row_major":
                    rc, at, msg = sess.check_state()
                    assert rc == 0, (what, who, first + step - 1, rc, at, msg)
            end, v, o, _ = sess.get_base()
            assert (end == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == m.evaluate(pb, end), (what, who)
            sess.close()
