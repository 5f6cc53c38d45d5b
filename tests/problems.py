"""Named problem shapes shared by the CPU and GPU tests (name -> oracle Problem factory).
Together they cover every layout class of the engine: W = 1/2/4/8 words per row, slot fields of
8/16/32/64 brokers per rack, unequal racks with padding slots, removed brokers, RF raised and
lowered, C7 lower bound > 0, and dense (tie-broken) weight tables."""
import dataclasses

import numpy as np

from oracle import model as m

from conftest import make_problem

SHAPES = {
    "readme": lambda: m.readme_problem(),                                       # W1 S16, README.md:27-63
    "readme_tb": lambda: m.with_tiebreak(m.readme_problem()),                   # dense weights
    "cfg2": lambda: m.synthetic_problem(256, 32, 4, 3),                         # W1 S8
    "cfg2_rm2": lambda: m.synthetic_problem(256, 32, 4, 3, remove=2),           # unequal racks
    "cfg3_small": lambda: m.synthetic_problem(200, 64, 8, 3, remove=2),         # W2 S8
    "w4_s16": lambda: make_problem(150, [12, 11, 12, 10, 12, 12, 9, 12], 3, seed=1, removed=3),
    "w8_s16": lambda: make_problem(300, [16] * 16, 3, seed=2, removed=5),       # cfg5 layout
    "s32": lambda: make_problem(120, [20, 19], 2, seed=3, removed=1),           # W2, whole-word racks
    "s64_r1": lambda: make_problem(90, [40], 3, seed=4),                        # one rack of 40: C7 lo = hi = 3
    "rf_up": lambda: make_problem(100, [6, 6, 6], 4, RFcur=2, seed=5),          # RF raised, ppr [1,2]
    "rf_down": lambda: make_problem(100, [8, 8, 8, 8], 2, RFcur=4, seed=6),     # RF lowered
    "dense_small": lambda: make_problem(24, [4, 4, 4], 3, seed=7, tiebreak=True),
    # unique optimum (checked with the exact model in the test): round robin, one broker removed,
    # weights scaled + seeded random per-cell preference
    "dense_unique": lambda: m.with_random_tiebreak(m.synthetic_problem(20, 12, 4, 3, 1), 0),
    "dense_unique2": lambda: m.with_random_tiebreak(m.synthetic_problem(12, 9, 3, 2, 1), 1),
    "dense_unique3": lambda: m.with_random_tiebreak(m.synthetic_problem(12, 9, 3, 2, 1), 0),
    "dense_unique4": lambda: m.with_random_tiebreak(m.synthetic_problem(20, 12, 4, 3, 1), 2),
    "tiny": lambda: make_problem(3, [2, 2], 2, seed=8),
    # edge cases: ragged current assignment (1..4 replicas per partition, some entirely on removed
    # brokers), RF 1, a single partition, the largest row count, every one of the 256 slots in use
    "ragged": lambda: ragged_problem(),
    "rf1": lambda: make_problem(40, [3, 3, 3], 1, seed=9, removed=1),
    "one_partition": lambda: make_problem(1, [2, 2, 2], 3, seed=10),
    "max_rows": lambda: m.synthetic_problem(8160, 16, 4, 2, remove=1),
    "all_slots": lambda: m.synthetic_problem(64, 256, 16, 3),
    # two-word rows too many for mask planes + one-hot plane in shared memory: the engine falls back
    # to packed weight entries (same keys)
    "w2_rows6000": lambda: m.synthetic_problem(6000, 64, 8, 3, remove=1),
}

# Layouts and weight / bound regimes the shapes above leave out; together with them they reach every evaluator
# configuration the engine dispatches (tests/test_layout_matrix.py checks that)
LAYOUT_SHAPES = {
    # whole-word rack fields with at most one replica per rack (ppr 0..1): one or two words per rack, racks of
    # 64 slots, one 32-slot rack in a one-word row; 16-slot racks in narrow rows, 8- and 16-slot racks in wide rows
    "rack5_w4": lambda: make_problem(120, [20, 20, 20], 2, seed=21),
    "rack5_w8": lambda: make_problem(90, [40, 40, 40], 2, seed=22),
    "rack5_w8_r4": lambda: make_problem(80, [33] * 4, 3, seed=23, removed=2),
    "rack5_w1": lambda: dataclasses.replace(make_problem(60, [20], 1, seed=24), ppr_lo=0),
    "rack5_w2": lambda: make_problem(70, [24, 24], 1, seed=25),
    "rack4_w1": lambda: make_problem(70, [12, 12], 1, seed=26),
    "rack4_w2": lambda: make_problem(80, [12, 12, 12], 2, seed=27),
    "rack3_w4": lambda: make_problem(90, [6] * 12, 3, seed=28),
    "rack3_w8": lambda: make_problem(90, [5] * 20, 3, seed=29, removed=2),
    "rack4_w8": lambda: make_problem(90, [10] * 10, 3, seed=30),
    # general C7 bounds (ppr 1..1) in four- and eight-word rows
    "ppr11_w4": lambda: make_problem(100, [20, 20, 20], 3, seed=31),
    "ppr11_w8": lambda: make_problem(100, [40, 40, 40], 3, seed=32),
    # exactly eight term planes of the column-major evaluator, the widest cost field (key_obj_bits 24)
    "planes8_w1": lambda: with_weight_classes(m.synthetic_problem(700, 32, 4, 3), [1000, 2000, 3000, 3500], [1, 7, 300, 595]),
    "planes8_w2": lambda: with_weight_classes(SHAPES["cfg3_small"](), [1000, 2000, 3000, 3500], [1, 7, 300, 595]),
    # violation fields that saturate: per-broker replica lower bounds near 65,535
    "sat_cfg2": lambda: with_saturating_bounds(with_12bit_weights(m.synthetic_problem(256, 32, 4, 3), 50)),
    "sat_rack5_w4": lambda: with_saturating_bounds(with_12bit_weights(LAYOUT_SHAPES["rack5_w4"](), 51)),
}


def with_12bit_weights(pb, seed):
    """Packed entries with all 12 bits in use: seeded follower and leader weights in 1..4095 drawn independently
    per current placement (a leader may weigh less than a follower), 4095 present in both."""
    rng = np.random.RandomState(seed)
    p, b = np.nonzero(pb.wF | pb.wL)
    wF, wL = np.zeros(pb.wF.shape, np.int64), np.zeros(pb.wL.shape, np.int64)
    wF[p, b], wL[p, b] = rng.randint(1, 4096, size=p.size), rng.randint(1, 4096, size=p.size)
    wF[p[0], b[0]] = wL[p[-1], b[-1]] = 4095
    return with_weights(pb, wF, wL)


def with_dense_weights(pb, seed):
    """A dense weight table: seeded weights 0..300 on every (partition, broker) cell."""
    rng = np.random.RandomState(seed)
    return with_weights(pb, rng.randint(0, 301, size=pb.wF.shape), rng.randint(0, 301, size=pb.wL.shape))


def with_wide_weights(pb, seed):
    """Seeded weights of 4096..9000 (followers) and 0..9000 (leaders) on the current placements: above the 12-bit
    fields of packed entries, so only the dense table holds them."""
    rng = np.random.RandomState(seed)
    p, b = np.nonzero(pb.wF | pb.wL)
    wF, wL = np.zeros(pb.wF.shape, np.int64), np.zeros(pb.wL.shape, np.int64)
    wF[p, b], wL[p, b] = rng.randint(4096, 9001, size=p.size), rng.randint(0, 9001, size=p.size)
    return with_weights(pb, wF, wL)


def with_weight_classes(pb, follower, bonus):
    """Partition p's i-th current replica weighs follower[(p + i) % len(follower)], its preferred replica leads
    with bonus[p % len(bonus)] on top: len(follower) + len(bonus) term planes, each class at most once per
    partition (RF <= len(follower))."""
    wF, wL = np.zeros(pb.wF.shape, np.int64), np.zeros(pb.wL.shape, np.int64)
    for p in range(pb.P):
        for i, b in enumerate(pb.cur[p]):
            if b >= 0:
                wF[p, b] = follower[(p + i) % len(follower)]
                wL[p, b] = wF[p, b] + (bonus[p % len(bonus)] if i == 0 else 0)
    return with_weights(pb, wF, wL)


def with_weights(pb, wF, wL):
    return dataclasses.replace(pb, wF=wF.astype(np.uint16), wL=wL.astype(np.uint16))


def with_saturating_bounds(pb, lo=65000):
    """Replica lower bounds near 65,535: violations exceed the violation field of a packed key."""
    return dataclasses.replace(pb, rep_lo=np.full(pb.B, lo, np.int32), rep_hi=np.full(pb.B, 65535, np.int32))


# weight regimes x the layouts they are applied to: 12-bit packed entries, dense tables, weights above 12 bits,
# weights above 12 bits in four classes (the column-major evaluator accepts them)
_REGIMES = {
    "w12": (with_12bit_weights, ["cfg2_rm2", "readme", "rack4_w1", "rack5_w1", "s32", "rack4_w2", "rack5_w2",
                                 "rack5_w4", "ppr11_w8"]),
    "dense": (with_dense_weights, ["rack4_w1", "s64_r1", "cfg3_small", "rack4_w2", "ppr11_w4", "rack3_w4", "w4_s16",
                                   "ppr11_w8", "rack3_w8", "rack4_w8"]),
    "wide": (with_wide_weights, ["rack5_w1", "rack5_w2", "rack5_w4", "rack5_w8"]),
    "widecm": (lambda pb, seed: with_weight_classes(pb, [4096, 5000, 6100], [700]), ["cfg2", "cfg3_small"]),
}
for _regime, (_f, _bases) in _REGIMES.items():
    for _i, _b in enumerate(_bases):
        LAYOUT_SHAPES["%s_%s" % (_regime, _b)] = (lambda f=_f, b=_b, seed=60 + _i: f({**SHAPES, **LAYOUT_SHAPES}[b](), seed))


def ragged_problem(P=60, seed=12):
    rng = np.random.RandomState(seed)
    B0, removed = 14, 3
    current = []
    for p in range(P):
        k = 1 + p % 4
        current.append(list(map(int, rng.choice(B0, size=k, replace=False))))
    for p in range(5, P, 997):
        current[p] = [12, 13]             # every replica on a broker that leaves the cluster
    current[6] = [11]
    racks = {b: "az%d" % (b % 3) for b in range(B0)}
    return m.build_problem(current, list(range(B0 - removed)), racks, 3)


# ---- the HBM-base search path (DESIGN.md 7.1): every topic session and every instance above 8,160 partitions
# Its evaluator is the general-bounds form at every rack width, so the C7 form (at most one replica per rack 0..1,
# exactly one 1..1, or a lower bound above 0 with RF > racks) is a layout axis of its own there.  Small shapes for the
# (row width, rack field, C7 form) combinations the shapes above leave out, each with packed entries and a dense table.
_C7_LAYOUTS = {
    "c7_w1_s8_lo": ([6, 6, 6], 4),          # C7 1..2
    "c7_w1_s16_lo": ([10, 10], 3),          # C7 1..2
    "c7_w1_word_11": ([20], 1),             # one rack of 20, RF 1: C7 1..1
    "c7_w1_word_lo": ([20], 2),             # C7 2..2
    "c7_w2_s8_11": ([6] * 5, 5),
    "c7_w2_s8_lo": ([6] * 5, 6),
    "c7_w2_s16_11": ([12, 12, 12], 3),
    "c7_w2_s16_lo": ([12, 12, 12], 4),
    "c7_w2_word_11": ([20, 20], 2),
    "c7_w4_s16_11": ([12] * 5, 5),
    "c7_w4_s16_lo": ([12] * 5, 6),
    "c7_w4_word_lo": ([20] * 3, 4),
    "c7_w8_word_lo": ([40] * 3, 4),
}
C7_SHAPES = {}
for _i, (_n, (_racks, _rf)) in enumerate(sorted(_C7_LAYOUTS.items())):
    # at most four current replicas: packed entries hold four weighted cells per partition
    C7_SHAPES[_n] = lambda r=_racks, rf=_rf, s=80 + _i: make_problem(50, r, rf, RFcur=min(rf, 4), seed=s, removed=1)
    C7_SHAPES[_n + "_dense"] = lambda r=_racks, rf=_rf, s=80 + _i: with_dense_weights(make_problem(50, r, rf, seed=s, removed=1), s)


def with_widest_cost_field(pb, seed):
    """Packed entries with the largest weight the 24-bit objective range allows (floor((2^24 - 1) / (P RF)), present
    once), seeded weights 1.. that on the current placements: key_obj_bits 24, the narrowest violation field.  Above
    4,096 partition replicas this is the widest a weight can be (12-bit weights exceed the objective range)."""
    top = 0xFFFFFF // (pb.P * pb.RF)
    rng = np.random.RandomState(seed)
    p, b = np.nonzero(pb.wF | pb.wL)
    wF, wL = np.zeros(pb.wF.shape, np.int64), np.zeros(pb.wL.shape, np.int64)
    wF[p, b], wL[p, b] = rng.randint(1, top + 1, size=p.size), rng.randint(1, top + 1, size=p.size)
    wL[p[0], b[0]] = top
    return with_weights(pb, wF, wL)


def with_saturating_violation(pb, excess=7):
    """Replica lower bounds raised, broker by broker, until the restatement's initial base violates the rows by the
    key's violation cap + excess: the first winner is a saturated key."""
    from oracle import ref

    r = ref.Ref(pb)
    reps = r.decode(*r.init_base())
    cap = (1 << (39 - r.obj_bits)) - 1
    need = cap + excess - m.evaluate(pb, reps)[0]
    cnt = np.bincount(reps[reps >= 0], minlength=pb.B)
    lo, hi = pb.rep_lo.copy(), pb.rep_hi.copy()
    for b in range(pb.B):
        # broker b's replica term becomes lo - count, its old term (over or under its bounds) plus what is added
        c = int(cnt[b])
        old = max(c - int(hi[b]), 0) + max(int(lo[b]) - c, 0)
        add = min(need, 65535 - c - old)
        lo[b] = c + old + add
        hi[b] = max(int(hi[b]), int(lo[b]))
        need -= add
    assert need == 0
    out = dataclasses.replace(pb, rep_lo=lo, rep_hi=hi)
    assert m.evaluate(out, reps)[0] == cap + excess
    return out


# Above 8,160 partitions only the HBM path runs: the layout edges of SHAPES at those row counts.  Weights above 12 bits
# have no shape here: P * RF * weight must stay below 2^24, so above 4,096 partition replicas no weight reaches 4,096.
LARGE_SHAPES = {
    "big_rf_up": lambda: make_problem(8200, [6, 6, 6], 4, RFcur=2, seed=71),                # RF raised, C7 1..2
    "big_rf_down": lambda: make_problem(8300, [8, 8, 8, 8], 2, RFcur=4, seed=72),           # four home slots a row
    "big_ragged": lambda: ragged_problem(8400, seed=73),                                    # 1..4 current replicas
    "big_rf1": lambda: make_problem(9000, [3, 3, 3], 1, seed=74, removed=1),
    "big_s64_r1": lambda: make_problem(8300, [40], 3, seed=75),                             # one rack: C7 3..3
    "big_ppr11_w8": lambda: make_problem(8200, [40, 40, 40], 3, seed=76),                   # eight-word rows, C7 1..1
    "big_obj24": lambda: with_widest_cost_field(make_problem(8500, [12, 12, 12, 12], 3, seed=77, removed=1), 78),
    "big_dense_w4": lambda: with_dense_weights(make_problem(8800, [12, 11, 12, 10, 12, 12, 9, 12], 3, seed=79,
                                                            removed=3), 80),
    "big_sat": lambda: with_saturating_violation(LARGE_SHAPES["big_obj24"]()),
}


def emptied_base(pb, reps, seed):
    """A damaged base with rows emptied (their leader byte stays 0xFF: the partitions led from a slot they do not
    hold), replicas moved to random brokers (duplicates collapse) and rows cut short; the damage scales with P."""
    rng = np.random.RandomState(seed)
    out = reps.copy()
    for p in rng.choice(pb.P, size=max(1, pb.P // 10), replace=False):
        out[p, rng.randint(pb.RF)] = rng.randint(pb.B)
    if pb.RF > 1:
        out[rng.choice(pb.P, size=max(1, pb.P // 30), replace=False), -1] = -1
    out[rng.choice(pb.P, size=max(1, pb.P // 50), replace=False), :] = -1
    return out


def moved_base(pb, reps, seed):
    """A damaged base with no row emptied: replicas moved in a quarter of the rows and rows cut short, so that many
    partitions miss a home broker or are led from elsewhere (long displaced lists)."""
    rng = np.random.RandomState(seed)
    out = reps.copy()
    for p in rng.choice(pb.P, size=max(1, pb.P // 4), replace=False):
        out[p, rng.randint(pb.RF)] = rng.randint(pb.B)
        if pb.RF > 1 and rng.randint(2):
            out[p, ::-1] = out[p].copy()          # another replica leads
    if pb.RF > 1:
        cut = rng.choice(pb.P, size=max(1, pb.P // 20), replace=False)
        out[cut, -1] = -1
    empty = (out < 0).all(1)
    out[empty] = reps[empty]                      # a short row that lost its last replica keeps it
    return out
