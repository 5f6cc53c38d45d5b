"""The sorted-batch body of the tensor-core schedules (pop 0x300, csrc/kao_kernels.cuh: build_cand_list and the batch loop)
restated under the warp emulator (tests/emu_sorted, on top of tests/emu_mma): every CTA sorts its share of a round by the class of the candidates'
control words (csrc/kao_device_mma.cuh, cand_class) and generates batches of 32 neighbours of that order.  Keys must be
the oracle restatement's, bit for bit, whichever lanes share a batch."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from oracle import model as m

SEED = 0xC0FFEE


@pytest.fixture(scope="module")
def srt():
    import emu_sorted

    emu_sorted.lib()
    return emu_sorted


@pytest.fixture(scope="module")
def cfg3(srt, ref_lib):
    pb = m.synthetic_problem(1000, 64, 8, 3)
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    sess = srt.SortedSession(kao.Problem.from_fields(pb))
    yield sess, r, bits, ld
    sess.close()


# (round, round_size, idx_lo, idx_hi, grid, warps, cap)
CASES = {
    "many_classes": (2, 4096, 0, 4096, 4, 16, 8192),
    "cycle_round": (3, 4096, 0, 4096, 4, 16, 8192),
    "round_below_warp_count": (5, 10, 0, 10, 2, 16, 8192),
    "share_above_capacity": (2, 4096, 0, 4096, 2, 16, 512),
    "idx_lo_not_zero": (6, 4096, 1500, 3100, 3, 16, 8192),
    "identity_only": (2, 4096, 4095, 4096, 4, 16, 8192),
    "one_candidate": (2, 4096, 77, 78, 4, 16, 8192),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_sorted_batches_give_the_restatement_keys(cfg3, name):
    sess, r, bits, ld = cfg3
    rnd, size, lo, hi, grid, warps, cap = CASES[name]
    want = r.candidate_keys(bits, ld, SEED, rnd, size, lo, hi - lo)
    assert (sess.sorted_keys(SEED, rnd, size, lo, hi, grid, warps, cap) == want).all()


@pytest.mark.parametrize("name", sorted(CASES))
def test_every_cta_sorts_exactly_its_share(srt, name):
    rnd, size, lo, hi, grid, warps, cap = CASES[name]
    seen = []
    for cta in range(grid):
        lst, cls, bounds, is_sorted = srt.cta_batches(SEED, rnd, size, lo, hi, grid, warps, cap, cta)
        share = [i for i in range(lo + cta * warps, hi, grid * warps) for i in range(i, min(i + warps, hi))]
        assert sorted(lst.tolist()) == share
        assert is_sorted == (len(share) <= cap)
        if is_sorted:
            assert (np.diff(cls.astype(np.int64)) >= 0).all()
        assert (np.diff(bounds.astype(np.int64)) <= 32).all() and (np.diff(bounds.astype(np.int64)) > 0).all()
        assert ((cls == 0) == (lst == size - 1)).all()                 # class 0: the identity candidate alone
        seen += share
    assert sorted(seen) == list(range(lo, hi))


def test_batches_mostly_share_one_class(srt):
    """The point of the sort: at the headline's CTA share a batch holds few classes (unsorted: about 20)."""
    lst, cls, bounds, is_sorted = srt.cta_batches(SEED, 2, 1 << 18, 0, 1 << 18, 132, 16, 8192, 0)
    assert is_sorted
    per_batch = [len(set(cls[a:b].tolist())) for a, b in zip(bounds[:-1], bounds[1:])]
    assert np.mean(per_batch) < 3
