"""Per-partition replication rows (docs/MODEL.md §11) through the engine's own device code on the CPU: the kRF forms of
row_eval and delta_eval (kao_device.cuh) on the evaluator configuration of the HBM-base kernels (tests/emu), against
the restatement (tests/rf_ref) and the model.  Every layout class of rack field (8-slot racks in one to eight words,
with a rack count that is not a multiple of four, 16-, 32- and 64-slot racks), packed entries and dense tables, and
rows whose C7 forms differ from their neighbours' (docs/MODEL.md §1: ppr_lo <= 63, ppr_hi <= 127)."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import rf_ref
from conftest import make_problem
from oracle import model as m
from problems import C7_SHAPES, LAYOUT_SHAPES, SHAPES, emptied_base, mixed_rows, moved_base, off_rf_base

H100_SMS = 132           # the "second candidate of a thread" range of check_delta_keys (test_gpu_large_layouts.py)

RSHAPES = {
    "s8_r3_w1": SHAPES["rf_up"],                                    # R = 3: the nv mask of the last word
    "s8_r4_w1": SHAPES["cfg2"],                                     # four 8-slot racks in one word
    "s8_r5_w2": C7_SHAPES["c7_w2_s8_11"],
    "s8_r5_w2_dense": C7_SHAPES["c7_w2_s8_11_dense"],
    "s8_r12_w4": LAYOUT_SHAPES["rack3_w4"],
    "s8_r12_w4_dense": LAYOUT_SHAPES["dense_rack3_w4"],
    "s8_r20_w8": LAYOUT_SHAPES["rack3_w8"],
    "s16_w1": SHAPES["readme"],
    "s16_w4": SHAPES["w4_s16"],
    "s16_w8": LAYOUT_SHAPES["rack4_w8"],
    "s16_w8_dense": LAYOUT_SHAPES["dense_rack4_w8"],
    "s32_w2": SHAPES["s32"],
    "s32_w8": lambda: make_problem(60, [20] * 5, 3, seed=90),
    "s64_r1_w2": SHAPES["s64_r1"],
    "s64_r1_dense": LAYOUT_SHAPES["dense_s64_r1"],
    "s64_w8": LAYOUT_SHAPES["rack5_w8"],
    "ragged": SHAPES["ragged"],
    "rf_b_minus_1": lambda: make_problem(30, [2, 2], 3, seed=91),   # four brokers, RF 3: rf[p] up to B - 1
}


@pytest.fixture(scope="module")
def emu():
    import emu as emu_mod

    emu_mod.lib()
    return emu_mod


def setup(emu, name, seed=0x7F):
    kp = kao.Problem.from_fields(RSHAPES[name]())
    rr = mixed_rows(kp, seed)
    return kp, rr, emu.EmuSession(kp, replication=rr), rf_ref.RRef(kp, rr)


def assert_keys(got, want, what):
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (what, int(bad[0]), int(got[bad[0]]), int(want[bad[0]]))


def check_delta_keys(sess, r, bits, ld, size, what):
    """test_gpu_large_layouts.check_delta_keys on the CPU: a free and a cycle round; the smallest round, a full one, a
    sub-range; the first and last 256 of a round one candidate larger than a thread each on an H100"""
    n_two = H100_SMS * 512 + 1
    for rnd in (4, 7):
        for rs, lo, n in ((2, 0, 2), (size, 0, size), (size, size // 4, size // 3)):
            got = sess.candidate_keys(0xB16, rnd, rs, lo, n, delta=True)
            assert_keys(got, r.candidate_keys(bits, ld, 0xB16, rnd, rs, lo, n), (what, rnd, rs, lo))
        for lo in (0, n_two - 256):
            got = sess.candidate_keys(0xB16, rnd, n_two, lo, 256, delta=True)
            assert_keys(got, r.candidate_keys(bits, ld, 0xB16, rnd, n_two, lo, 256), (what, rnd, "two", lo))


def test_mixed_rows_mix_every_form():
    kp = kao.Problem.from_fields(RSHAPES["rf_b_minus_1"]())
    rr = mixed_rows(kp, 1)
    assert kp.B == 4 and set(rr.rf.tolist()) == {1, 2, 3}
    lohi = list(zip(rr.ppr_lo.tolist(), rr.ppr_hi.tolist()))
    assert not any(a == b == (63, 63) or a == b == (0, 0) for a, b in zip(lohi, lohi[1:]))
    assert (63, 63) in lohi and (0, 0) in lohi and any(h == 127 for _, h in lohi)
    assert (rr.ppr_lo <= rr.ppr_hi).all() and rr.ppr_lo.max() == 63


@pytest.mark.parametrize("name", sorted(RSHAPES))
def test_emulated_evaluation_and_keys_equal_the_restatement(emu, name):
    """get_base after set_base equals the restatement and the model, and the delta keys equal the restatement's, from
    the initial, a random, an off-rf (rows longer and shorter than rf[p]), an emptied and a moved base"""
    kp, rr, sess, r = setup(emu, name)
    cfg = sess.config()
    assert (cfg["W"], cfg["rack"], cfg["obj"]) == (r.W, 0, 0)      # LargeCfg<W>, whatever hi1 says
    bits, ld = r.init_base()
    init = r.decode(bits, ld)
    reps, v, o, _ = sess.get_base()
    assert (reps == init).all() and (v, o) == r.evaluate(bits, ld) == rf_ref.evaluate(kp, rr, reps)
    rng = np.random.RandomState(5)
    rand = np.stack([rng.choice(kp.B, size=kp.RF, replace=False) for _ in range(kp.P)]).astype(np.int32)
    bases = {"initial": init, "random": rand, "off_rf": off_rf_base(kp, init, 6),
             "emptied": emptied_base(kp, init, 5), "moved": moved_base(kp, init, 6)}
    lens = (bases["off_rf"] >= 0).sum(1)
    assert (lens > rr.rf).any() and (lens < rr.rf).any()
    for what, b in bases.items():
        sess.set_base(b)
        bits, ld = r.encode(b)
        got, v, o, _ = sess.get_base()
        assert (got == r.decode(bits, ld)).all(), what
        assert (v, o) == r.evaluate(bits, ld) == rf_ref.evaluate(kp, rr, got), what
        check_delta_keys(sess, r, bits, ld, 4096, what)
    sess.close()


@pytest.mark.parametrize("name", sorted(RSHAPES))
def test_emulated_walks_equal_the_restatement(emu, name):
    """48 rounds in two calls from the initial, an emptied and a moved base; the walked base evaluates as the model"""
    kp, rr, sess, r = setup(emu, name)
    init = r.decode(*r.init_base())
    for what, start in (("initial", init), ("emptied", emptied_base(kp, init, 5)), ("moved", moved_base(kp, init, 6))):
        sess.set_base(start)
        bits, ld = r.encode(start)
        for first, n in ((0, 24), (24, 24)):
            _, want = r.search(bits, ld, 0x5EED, first, n, 512)
            assert_keys(sess.search(0x5EED, first, n, 512), want, (what, first))
        reps, v, o, _ = sess.get_base()
        assert (reps == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld) == rf_ref.evaluate(kp, rr, reps)
    sess.close()


def uniform(pb):
    return kao.ReplicationRows(np.full(pb.P, pb.RF, np.int32), np.full(pb.P, pb.ppr_lo, np.int32),
                               np.full(pb.P, pb.ppr_hi, np.int32))


@pytest.mark.parametrize("name", sorted(n for n in {**SHAPES, **LAYOUT_SHAPES, **C7_SHAPES} if n != "max_rows"))
def test_uniform_rows_give_the_plain_delta_keys(emu, name):
    """With every row at RF and ppr_lo..ppr_hi, the kRF evaluator of the HBM kernels scores every candidate as the
    plain session's delta evaluator does (the shared-memory configuration: its own rack form and objective)"""
    kp = kao.Problem.from_fields({**SHAPES, **LAYOUT_SHAPES, **C7_SHAPES}[name]())
    try:
        plain = emu.EmuSession(kp)
    except ValueError:
        pytest.skip("no shared-memory plan")
    rows = emu.EmuSession(kp, replication=uniform(kp))
    init = plain.get_base()[0]
    assert (rows.get_base()[0] == init).all()
    for b in (init, moved_base(kp, init, 3)):
        plain.set_base(b)
        rows.set_base(b)
        for rnd in (4, 7):
            assert_keys(rows.candidate_keys(0xD317A, rnd, 1024, 0, 512, delta=True),
                        plain.candidate_keys(0xD317A, rnd, 1024, 0, 512, delta=True), rnd)
    plain.close()
    rows.close()


def test_lower_bound_63_on_four_empty_racks_is_exact(emu):
    """ppr_lo = 63 on a row with no replica in any of four 8-slot racks: 4 * 63 = 252 in one byte, no carry"""
    kp = kao.Problem.from_fields(SHAPES["cfg2"]())
    assert kp.R == 4
    rr = kao.ReplicationRows(np.ones(kp.P, np.int32), np.full(kp.P, 63, np.int32), np.full(kp.P, 63, np.int32))
    sess = emu.EmuSession(kp, replication=rr)
    r = rf_ref.RRef(kp, rr)
    reps = np.full((kp.P, kp.RF), -1, np.int32)
    reps[1:, 0] = np.arange(kp.P - 1) % kp.B                   # partition 0 empty, the others one replica each
    sess.set_base(reps)
    got, v, o, _ = sess.get_base()
    assert (v, o) == r.evaluate(*r.encode(reps)) == rf_ref.evaluate(kp, rr, got)
    assert rf_ref._row_terms(kp, reps, 0, 1, 63, 63) == 1 + 4 * 63
    sess.close()


@pytest.mark.parametrize("lo", [64, 127])
def test_emulated_sessions_refuse_lower_bounds_above_63(emu, lo):
    kp = kao.Problem.from_fields(SHAPES["cfg2"]())
    rr = kao.ReplicationRows(np.ones(kp.P, np.int32), np.zeros(kp.P, np.int32), np.full(kp.P, 127, np.int32))
    rr.ppr_lo[7] = lo
    with pytest.raises(ValueError, match="per-partition replication factors: partition 7"):
        emu.EmuSession(kp, replication=rr)
    kp.ppr_lo, kp.ppr_hi = lo, 127
    with pytest.raises(ValueError, match="bad per-partition-per-rack bounds"):
        emu.EmuSession(kp)
