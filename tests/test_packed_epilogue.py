"""The packed MMA epilogue (csrc/kao_device_mma.cuh, the sorted-batch schedule pop 0x300: two candidates per 16 x 2
instruction) under the warp emulator (tests/emu, pop 0x300).  Keys and trajectories must be the
restatement's, bit for bit, including bounds far above the column totals (clamped to P), bounds of 0, and the largest
column-major row count.  The host forms of the intrinsics are held to a plain-integer model first."""
import dataclasses

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from oracle import model as m
from problems import SHAPES

SHAPES_PACKED = {
    "cfg2": SHAPES["cfg2"],                                              # one-word rows, 8 partition words
    "cfg2_rm2": SHAPES["cfg2_rm2"],                                      # unequal racks
    "cfg3": lambda: m.synthetic_problem(1000, 64, 8, 3),                 # the headline shape: 32 words, compile-time form
    "rf4_w2": lambda: m.synthetic_problem(300, 40, 5, 4, remove=3),      # RF 4, padding slots
    "p1100": lambda: m.synthetic_problem(1100, 64, 8, 3, remove=2),      # 64 words (swizzled, run-time form)
}


def with_extreme_bounds(pb):
    """Per-broker bounds at the edges the epilogue clamps: lo = hi = 65,535 (far above any column total), hi = 0,
    lo = hi = P, lo just above P, hi just below P — for replicas and for leaders."""
    P = pb.P
    rl, rh, ll, lh = (np.array(x, np.int32).copy() for x in (pb.rep_lo, pb.rep_hi, pb.ldr_lo, pb.ldr_hi))
    for arr_lo, arr_hi, off in ((rl, rh, 0), (ll, lh, 5)):
        arr_lo[off + 0] = arr_hi[off + 0] = 65535
        arr_lo[off + 1] = arr_hi[off + 1] = 0
        arr_lo[off + 2] = arr_hi[off + 2] = P
        arr_lo[off + 3], arr_hi[off + 3] = P + 1, 65535
        arr_lo[off + 4], arr_hi[off + 4] = 0, max(P - 1, 0)
    return dataclasses.replace(pb, rep_lo=rl, rep_hi=rh, ldr_lo=ll, ldr_hi=lh)


def with_random_bounds(pb, seed):
    """Every broker's bounds drawn from 0, P - 1, P, P + 1, 65,535 and uniform values, with lo <= hi."""
    rng = np.random.RandomState(seed)
    P = pb.P

    def draw():
        pool = np.array([0, max(P - 1, 0), P, P + 1, 65535] + list(rng.randint(0, 65536, 3)) + list(rng.randint(0, P + 1, 3)))
        a, b = rng.choice(pool, 2)
        return min(a, b), max(a, b)

    rl, rh, ll, lh = (np.zeros(pb.B, np.int32) for _ in range(4))
    for b in range(pb.B):
        rl[b], rh[b] = draw()
        ll[b], lh[b] = draw()
    return dataclasses.replace(pb, rep_lo=rl, rep_hi=rh, ldr_lo=ll, ldr_hi=lh)


@pytest.fixture(scope="module")
def packed():
    import emu

    emu.lib()
    return emu


def check(packed, ref_lib, pb, rounds=3, size=256, n=96):
    r = ref_lib.Ref(pb)
    bits, ld = r.init_base()
    sess = packed.MmaSession(kao.Problem.from_fields(pb), 0x300)
    for rnd in (2, 3):                                                    # round 3: a cycle round
        want = r.candidate_keys(bits, ld, 0xC0FFEE, rnd, 1024, 1024 - n, n)
        assert (want == sess.candidate_keys(0xC0FFEE, rnd, 1024, 1024 - n, n)).all(), rnd
    _, want = r.search(bits, ld, 0x5EED, 0, rounds, size)
    assert (want == sess.search(0x5EED, 0, rounds, size)).all()
    assert (sess.get_base()[0] == r.decode(bits, ld)).all()
    sess.close()


# ---- the host intrinsics against a plain-integer model
EDGE_HALVES = np.array([0, 1, 2, 0x7FFE, 0x7FFF, 0x8000, 0x8001, 8160, 8161, 0xFFFE, 0xFFFF], np.uint32)


def operands(seed=3, n=4096):
    rng = np.random.RandomState(seed)
    halves = np.concatenate([EDGE_HALVES, rng.randint(0, 1 << 16, 64).astype(np.uint32)])
    lo_a, hi_a, lo_b, hi_b = (rng.choice(halves, n) for _ in range(4))
    edge = np.array(np.meshgrid(EDGE_HALVES, EDGE_HALVES)).reshape(2, -1)      # every pair of edge halves, both halves
    lo_a = np.concatenate([lo_a, edge[0]]); hi_a = np.concatenate([hi_a, edge[1]])
    lo_b = np.concatenate([lo_b, edge[1]]); hi_b = np.concatenate([hi_b, edge[0]])
    return (lo_a | hi_a << 16).astype(np.uint32), (lo_b | hi_b << 16).astype(np.uint32)


def halves(x):
    return x & 0xFFFF, x >> 16


@pytest.mark.parametrize("op,fn", [("vmaxu2", np.maximum), ("vminu2", np.minimum)])
def test_host_16x2_max_min_match_the_integer_model(packed, op, fn):
    a, b = operands()
    (al, ah), (bl, bh) = halves(a.astype(np.int64)), halves(b.astype(np.int64))
    want = (fn(al, bl) | fn(ah, bh) << 16).astype(np.uint32)
    assert (packed.simd(op, a, b) == want).all()


@pytest.mark.parametrize("sel", [0x5410, 0x4140, 0x4342, 0x1010, 0x3232])
def test_host_byte_perm_matches_the_integer_model(packed, sel):
    """The selectors the packed epilogue uses: pair two halfwords, spread two bytes, broadcast a halfword."""
    a, b = operands(seed=4)
    pool = a.astype(np.uint64) | b.astype(np.uint64) << 32
    want = np.zeros_like(a)
    for i in range(4):
        byte = (pool >> np.uint64(8 * ((sel >> (4 * i)) & 7))) & np.uint64(0xFF)
        want |= (byte.astype(np.uint32) << (8 * i)).astype(np.uint32)
    assert (packed.simd("byte_perm", a, b, sel) == want).all()


# ---- the packed body against the restatement
@pytest.mark.parametrize("name", sorted(SHAPES_PACKED))
def test_packed_body_matches_the_restatement(packed, ref_lib, name):
    check(packed, ref_lib, SHAPES_PACKED[name]())


@pytest.mark.parametrize("name", ["cfg2", "cfg3", "p1100"])
def test_packed_body_on_extreme_bounds(packed, ref_lib, name):
    check(packed, ref_lib, with_extreme_bounds(SHAPES_PACKED[name]()))


@pytest.mark.parametrize("seed", [1, 2])
def test_packed_body_on_random_bounds(packed, ref_lib, seed):
    check(packed, ref_lib, with_random_bounds(SHAPES_PACKED["cfg3"](), seed), rounds=2, size=128, n=64)


def test_packed_body_at_the_largest_column_major_shape(packed, ref_lib):
    """8,160 partitions on 32 slots (256 words per slot, the largest column totals), with the edge bounds."""
    pb = with_extreme_bounds(m.synthetic_problem(8160, 32, 4, 2, remove=1))
    check(packed, ref_lib, pb, rounds=1, size=64, n=32)
