"""The column-major evaluator with its sums on the tensor cores (csrc/kao_device_mma.cuh, schedules with pop 0x100)
under the warp emulator (tests/emu_mma on top of tests/emu): ldmatrix and the binary MMA are restated with their PTX
fragment layouts, and 32 candidates are generated, parked and evaluated together as one warp of the search kernel does it.
Keys and trajectories must be the restatement's, bit for bit."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from oracle import model as m
from problems import LAYOUT_SHAPES, SHAPES

SHAPES_MMA = {
    "cfg2": SHAPES["cfg2"],                                              # one-word rows, 8 partition words
    "cfg2_rm2": SHAPES["cfg2_rm2"],                                      # unequal racks
    "cfg3": lambda: m.synthetic_problem(1000, 64, 8, 3),                 # the headline shape: 32 words, compile-time form
    "rf4_w2": lambda: m.synthetic_problem(300, 40, 5, 4, remove=3),      # RF 4, padding slots
    "p1100": lambda: m.synthetic_problem(1100, 64, 8, 3, remove=2),      # 64 words (swizzled, run-time form)
}


@pytest.fixture(scope="module")
def emu():
    import emu as emu_mod

    emu_mod.lib()
    return emu_mod


@pytest.fixture(scope="module")
def mma():
    import emu_mma

    emu_mma.lib()
    return emu_mma


def product(pb):
    return kao.Problem.from_fields(pb)


def check(mma, ref_lib, pb, rounds=3, size=256, n=96):
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    sess = mma.MmaSession(product(pb))
    for rnd in (2, 3):                                                    # round 3: a cycle round
        want = r.candidate_keys(bits, ld, 0xC0FFEE, rnd, 1024, 1024 - n, n)
        assert (want == sess.candidate_keys(0xC0FFEE, rnd, 1024, 1024 - n, n)).all(), rnd
    _, want = r.search(bits, ld, 0x5EED, 0, rounds, size)
    assert (want == sess.search(0x5EED, 0, rounds, size)).all()
    assert (sess.get_base()[0] == r.decode(bits, ld)).all()
    sess.close()


@pytest.mark.parametrize("name", sorted(SHAPES_MMA))
def test_mma_body_matches_the_restatement(mma, ref_lib, name):
    check(mma, ref_lib, SHAPES_MMA[name]())


def test_mma_body_on_the_layout_shapes_it_covers(emu, mma, ref_lib):
    covered = []
    for name in sorted(LAYOUT_SHAPES):
        pb = LAYOUT_SHAPES[name]()
        sess = emu.EmuSession(product(pb))
        ok = sess.set_evaluator(1)                          # the column-major evaluator covers the layout
        sess.close()
        if ok:
            covered.append(name)
            check(mma, ref_lib, pb, rounds=3, size=128, n=64)
        else:
            with pytest.raises(ValueError):
                mma.MmaSession(product(pb))
    assert {"planes8_w1", "planes8_w2"} <= set(covered)


def test_mma_body_at_8160_partitions(mma, ref_lib):
    """256 words per slot (32 k-steps per tile), the largest row count."""
    check(mma, ref_lib, SHAPES["max_rows"](), rounds=1, size=64, n=32)


@pytest.mark.parametrize("name", ["cfg3", "cfg2_rm2"])
def test_mma_body_on_short_rows_and_invalid_leaders(emu, mma, ref_lib, name):
    """Short rows make the shortfall planes non-zero; a row whose first replica is missing and rows with a broker
    twice make leaders that are not one of the row's replicas.  Same keys as the restatement and as the popcount
    form of the column-major evaluator, and the base evaluates like the exact model."""
    pb = SHAPES_MMA[name]()
    r = ref_lib.Ref(pb)
    sess = mma.MmaSession(product(pb))
    pop = emu.EmuSession(product(pb))
    assert pop.set_evaluator(1)
    rng = np.random.RandomState(5)
    for it in range(3):
        reps = np.stack([rng.choice(pb.B, size=pb.RF, replace=False) for _ in range(pb.P)]).astype(np.int32)
        for _ in range(9):
            reps[rng.randint(pb.P), -1] = -1
        for _ in range(3):
            reps[rng.randint(pb.P), 0] = -1
        for _ in range(4):
            p = rng.randint(pb.P)
            reps[p, 1] = reps[p, 0]
        sess.set_base(reps)
        pop.set_base(reps)
        got_reps, v, o, _ = sess.get_base()
        assert (v, o) == m.evaluate(pb, got_reps)
        bits, ld = r.encode(reps)
        want = r.candidate_keys(bits, ld, 31 + it, it, 256, 0, 64)
        assert (want == sess.candidate_keys(31 + it, it, 256, 0, 64)).all(), it
        assert (want == pop.candidate_keys(31 + it, it, 256, 0, 64)).all(), it
        _, wk = r.search(bits, ld, 7 + it, 0, 3, 128)
        assert (wk == sess.search(7 + it, 0, 3, 128)).all(), it
        assert (sess.get_base()[0] == r.decode(bits, ld)).all()
    sess.close()
    pop.close()
