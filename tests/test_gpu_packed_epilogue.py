"""The default tensor-core schedule (1, 0x300, 512) scores two candidates per instruction in its MMA epilogue (16 x 2
halfword pairs, csrc/kao_device_mma.cuh).  Keys, trajectories and bases must be the restatement's, bit for bit, with
bounds far above the column totals, bounds of 0, at the largest column-major row count, and, against the popcount
schedule (4, 0x22, 1024), in a round too large for the sorted list."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import tuning
from oracle import model as m
from problems import SHAPES
from test_packed_epilogue import with_extreme_bounds, with_random_bounds

pytestmark = pytest.mark.gpu
PACKED = (1, 0x300, 512)
POPCOUNT = (4, 0x22, 1024)
SEED = 0xC0FFEE
SHAPES_BOUNDS = {
    "cfg3_extreme": lambda: with_extreme_bounds(m.synthetic_problem(1000, 64, 8, 3)),          # 32 words, compile-time form
    "cfg2_extreme": lambda: with_extreme_bounds(SHAPES["cfg2"]()),                            # one-word rows
    "p1100_extreme": lambda: with_extreme_bounds(m.synthetic_problem(1100, 64, 8, 3, remove=2)),   # run-time word count
    "cfg3_random": lambda: with_random_bounds(m.synthetic_problem(1000, 64, 8, 3), 1),
    "max_extreme": lambda: with_extreme_bounds(m.synthetic_problem(8160, 32, 4, 2, remove=1)),   # 8,160 x 32 slots
}


def session(pb):
    sess = kao.Session(kao.Problem.from_fields(pb))
    assert sess.stats()["column_major"] and sess.set_schedule(*PACKED)
    return sess


def test_packed_epilogue_is_the_default():
    assert tuning.DEFAULT_SCHEDULE == PACKED


@pytest.mark.parametrize("name", sorted(SHAPES_BOUNDS))
def test_candidate_keys_and_search_match_the_restatement(ref_lib, name):
    pb = SHAPES_BOUNDS[name]()
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    sess = session(pb)
    for rnd, size, lo, n in [(2, 4096, 0, 4096), (3, 4096, 0, 4096), (1, 5, 0, 5), (6, 8192, 1500, 1600)]:
        want = r.candidate_keys(bits, ld, SEED, rnd, size, lo, n)
        assert (sess.candidate_keys(SEED, rnd, size, lo, n) == want).all(), (rnd, size, lo, n)
    keys, _ = sess.search(0x5EED, 0, 6, 4096)
    _, want = r.search(bits, ld, 0x5EED, 0, 6, 4096)
    assert (keys == want).all()
    assert (sess.get_base()[0] == r.decode(bits, ld)).all()
    sess.close()


def test_share_beyond_the_list_matches_the_popcount_schedule():
    """A round of KAO_MAX_ROUND_SIZE candidates (every CTA's share walks unsorted), with the edge bounds: same keys,
    trajectory and base as the popcount schedule."""
    pb = with_extreme_bounds(m.synthetic_problem(1000, 64, 8, 3))
    a, b = session(pb), kao.Session(kao.Problem.from_fields(pb))
    assert b.set_schedule(*POPCOUNT)
    size = 1 << 24
    for rnd in (2, 3):
        assert np.array_equal(a.candidate_keys(SEED, rnd, size, 0, size), b.candidate_keys(SEED, rnd, size, 0, size)), rnd
    ka, _ = a.search(0x5EED, 0, 3, size)
    kb, _ = b.search(0x5EED, 0, 3, size)
    assert np.array_equal(ka, kb) and np.array_equal(a.get_base()[0], b.get_base()[0])
    a.close()
    b.close()
