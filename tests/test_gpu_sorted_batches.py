"""The default tensor-core schedule (1, 0x300, 512) takes its batches from every CTA's candidates sorted by class
(csrc/kao_kernels.cuh, build_cand_list).  Keys, trajectories and bases must be the restatement's, bit for bit: tiny
rounds, sharded index ranges, cycle rounds, and CTA shares too large for the sorted list (walked unsorted)."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import tuning
from oracle import model as m
from problems import SHAPES

pytestmark = pytest.mark.gpu
SORTED = (1, 0x300, 512)
SEED = 0xC0FFEE
SHAPES_SORTED = {
    "cfg3": lambda: m.synthetic_problem(1000, 64, 8, 3),                 # the headline shape, 32 partition words
    "cfg2": SHAPES["cfg2"],                                              # one-word rows
    "p1100": lambda: m.synthetic_problem(1100, 64, 8, 3, remove=2),      # run-time word count, displaced partitions
}


def session(pb):
    sess = kao.Session(kao.Problem.from_fields(pb))
    assert sess.stats()["column_major"] and sess.set_schedule(*SORTED)
    return sess


def test_sorted_batches_are_the_default():
    assert tuning.DEFAULT_SCHEDULE == SORTED


@pytest.mark.parametrize("name", sorted(SHAPES_SORTED))
def test_candidate_keys_match_the_restatement(ref_lib, name):
    pb = SHAPES_SORTED[name]()
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    sess = session(pb)
    # (round, round size, first index, count): whole rounds, a cycle round, rounds smaller than a CTA's warps,
    # index ranges that do not start at 0 (one GPU's slice of a sharded round), the identity candidate alone
    for rnd, size, lo, n in [(2, 4096, 0, 4096), (3, 4096, 0, 4096), (1, 5, 0, 5), (2, 40, 0, 40),
                             (6, 8192, 1500, 1600), (7, 8192, 8000, 192), (2, 4096, 4095, 1)]:
        want = r.candidate_keys(bits, ld, SEED, rnd, size, lo, n)
        assert (sess.candidate_keys(SEED, rnd, size, lo, n) == want).all(), (rnd, size, lo, n)
    sess.close()


@pytest.mark.parametrize("name", sorted(SHAPES_SORTED))
def test_search_matches_the_restatement(ref_lib, name):
    pb = SHAPES_SORTED[name]()
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    sess = session(pb)
    keys, _ = sess.search(0x5EED, 0, 8, 4096)
    _, want = r.search(bits, ld, 0x5EED, 0, 8, 4096)             # the restatement's base becomes the winner's in place
    assert (keys == want).all()
    assert (sess.get_base()[0] == r.decode(bits, ld)).all()
    sess.close()


def test_share_beyond_the_list_matches_the_popcount_schedule():
    """A round of KAO_MAX_ROUND_SIZE candidates: every CTA's share (127,000 candidates) is larger than any list the
    shared memory holds.  Same keys as the popcount schedule, which does not sort."""
    pb = m.synthetic_problem(1000, 64, 8, 3)
    a, b = session(pb), kao.Session(kao.Problem.from_fields(pb))
    assert b.set_schedule(4, 0x22, 1024)
    size = 1 << 24
    for rnd in (2, 3):
        ka = a.candidate_keys(SEED, rnd, size, 0, size)
        kb = b.candidate_keys(SEED, rnd, size, 0, size)
        assert np.array_equal(ka, kb), rnd
    ka, _ = a.search(0x5EED, 0, 3, size)
    kb, _ = b.search(0x5EED, 0, 3, size)
    assert np.array_equal(ka, kb) and np.array_equal(a.get_base()[0], b.get_base()[0])
    a.close()
    b.close()
