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


# ---- per-partition replication rows (docs/MODEL.md §11) ---------------------------------------------------------
# C7 forms of one row with rf replicas in R racks: (lo, hi)
C7_FORMS = {
    "floor_ceil": lambda rf, R, rng: (rf // R, -(-rf // R)),
    "zero": lambda rf, R, rng: (0, 0),                          # every replica is an excess
    "exact": lambda rf, R, rng: (rf, rf),                       # all of them in every rack
    "lo_more_racks": lambda rf, R, rng: (1 + rng.randint(2), 2 + rng.randint(3)),   # with R > rf every row misses
    "hi_above": lambda rf, R, rng: (0, rf + rng.randint(3)),
    "hi_127": lambda rf, R, rng: (rng.randint(3), 127),
    "lo_hi_63": lambda rf, R, rng: (63, 63),                    # the largest lower bound: 4 * 63 deficit in one byte
}


def mixed_rows(pb, seed):
    """Seeded per-partition rows: every tile of len(C7_FORMS) partitions takes each C7 form once, in an order of its
    own that never repeats the previous partition's form, with rf = 1, the row width RF (min(RF, B - 1)) or a random
    factor in between."""
    from kafka_assignment_optimizer_b200 import ReplicationRows

    rng = np.random.RandomState(seed)
    top = min(pb.RF, pb.B - 1)
    forms = list(C7_FORMS.values())
    order = []
    while len(order) < pb.P:
        tile = list(rng.permutation(len(forms)))
        if order and tile[0] == order[-1]:
            tile = tile[1:] + tile[:1]
        order += tile
    rf = np.array([(1, top, 1 + rng.randint(top))[rng.randint(3)] for _ in range(pb.P)], np.int32)
    lohi = np.array([forms[order[p]](int(rf[p]), pb.R, rng) for p in range(pb.P)], np.int32)
    return ReplicationRows(rf, lohi[:, 0].copy(), lohi[:, 1].copy())


def off_rf_base(pb, reps, seed):
    """A base of a replication session (rows of rf[p] replicas) with up to a ninth of the rows made longer (those
    shorter than RF), a ninth made shorter (those of two or more replicas), by one or two replicas each, and a ninth
    with their leader moved to another broker"""
    rng = np.random.RandomState(seed)
    out = reps.copy()
    n = max(1, pb.P // 9)
    k = (out >= 0).sum(1)
    for p in rng.permutation(np.flatnonzero(k < pb.RF))[:n]:       # longer
        free = [b for b in rng.permutation(pb.B) if b not in out[p]]
        for i in range(min(pb.RF - k[p], 1 + rng.randint(2), len(free))):
            out[p, k[p] + i] = free[i]
    for p in rng.permutation(np.flatnonzero(k > 1))[:n]:           # shorter
        out[p, max(1, k[p] - 1 - rng.randint(2)):] = -1
    for p in rng.choice(pb.P, size=n, replace=False):               # a replica moved
        free = [b for b in rng.permutation(pb.B) if b not in out[p]]
        out[p, 0] = free[0]
    return out


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


# ---- every one of the 256 slots a broker (docs/MODEL.md §2) -------------------------------------------------------
def slots(pb):
    """docs/MODEL.md §2: rack-major slots, S = pow2 >= max(8, largest rack) -> slot of every broker"""
    size = np.bincount(pb.rack_of, minlength=pb.R)
    S = 8
    while S < size.max():
        S <<= 1
    rank = np.array([int((pb.rack_of[:b] == pb.rack_of[b]).sum()) for b in range(pb.B)])
    return pb.rack_of.astype(int) * S + rank


# A cluster of 255 brokers grown by one: the current assignment uses brokers 0..254, the target list is 0..255 and
# broker b sits in rack b // (256 / racks), so broker 255 is the last of the last rack, on slot 255, with no home
# replica there (HOME255_SHAPES below put home replicas there).  Slot 255 is then a real broker while several tables
# use the byte 0xFF for "none" or "padding"; the new broker is empty, so every balance row that binds on it (C3 / C4,
# and the topic rows of the labellings below) reads its slot.
def grown_by_one(P, racks, RF=3, seed=0):
    rng = np.random.RandomState(seed)
    per = 256 // racks
    current = [list(map(int, rng.choice(255, size=RF, replace=False))) for _ in range(P)]
    return m.build_problem(current, list(range(256)), {b: "rack%02d" % (b // per) for b in range(256)}, RF)


SLOT255_SHAPES = {
    "s255_r32": lambda: grown_by_one(600, 32, seed=91),       # 32 racks of 8: 8-slot fields, KAO_MAX_RACKS
    "s255_r16": lambda: grown_by_one(600, 16, seed=92),
    "s255_r8": lambda: grown_by_one(500, 8, seed=93),         # 32-slot racks: one word each
    "s255_r4": lambda: grown_by_one(500, 4, seed=94),         # 64-slot racks: two words each
    "s255_r16_dense": lambda: with_dense_weights(grown_by_one(300, 16, seed=95), 95),
    "s255_big": lambda: grown_by_one(9000, 16, seed=96),      # the HBM path without topic rows
}


def one_topic(pb):
    """One topic over every partition: n RF >= 256 replicas, so its default rows bind on the empty broker 255"""
    pb.topics = [("all", p) for p in range(pb.P)]
    return pb


def topics_of_sizes(pb, seed, top=600):
    """Topics of 86..top partitions (seeded sizes, partitions interleaved by a seeded permutation), every one with
    n RF >= 256 replicas: with the default rows each topic binds on broker 255"""
    rng = np.random.RandomState(seed)
    sizes = []
    while sum(sizes) < pb.P:
        sizes.append(min(int(rng.randint(-(-256 // pb.RF), top + 1)), pb.P - sum(sizes)))
    if sizes[-1] * pb.RF < 256:                               # fold a short tail into the topic before it
        tail = sizes.pop()
        sizes[-1] += tail
    label = np.repeat(np.arange(len(sizes)), sizes)[rng.permutation(pb.P)]
    pb.topics = [("t%03d" % t, p) for p, t in enumerate(label)]
    return pb


# topic sessions with binding rows on broker 255, at and above 8,160 partitions
SLOT255_TOPIC_SHAPES = {
    "one_topic_r16": lambda: one_topic(SLOT255_SHAPES["s255_r16"]()),
    "sized_r32": lambda: topics_of_sizes(grown_by_one(1200, 32, seed=97), 97),
    "sized_r4": lambda: topics_of_sizes(SLOT255_SHAPES["s255_r4"](), 98, top=200),
    "sized_big": lambda: topics_of_sizes(SLOT255_SHAPES["s255_big"](), 99),
}


def leader_on_255_rf_up():
    """512 partitions on [p % 256, (p + 1) % 256], RF raised from 2 to 3, 256 brokers in 16 racks (broker b in rack
    b % 16, so broker 255 is on slot 255): partitions 255 and 511 are led from slot 255 and their rows get completed"""
    cur = [[p % 256, (p + 1) % 256] for p in range(512)]
    return m.build_problem(cur, list(range(256)), {b: "r%02d" % (b % 16) for b in range(256)}, 3)


def leader_on_255_removed():
    """260 brokers, the last four removed, 16 racks of 16 among the 256 that stay: rows [p, p + 1, p + 2] mod 260,
    so partitions 255 and 515 keep only their leader, on slot 255, and are completed"""
    cur = [[p % 260, (p + 1) % 260, (p + 2) % 260] for p in range(520)]
    return m.build_problem(cur, list(range(256)), {b: "r%02d" % (min(b, 255) // 16) for b in range(260)}, 3)


# initial-base checks: their current leaders sit on slot 255 and their rows get completed
LEADER255_SHAPES = {"leader255_rf_up": leader_on_255_rf_up, "leader255_removed": leader_on_255_removed}


# ---- home replicas on slot 255 (docs/MODEL.md §5.1) -------------------------------------------------------------------
# 256-broker clusters as they are met: broker 255 sits on slot 255 and holds current replicas, so it is a home slot of
# the partitions that have them.  When every slot is a broker the home byte 0xFF is slot 255 itself: the guided
# operations and the displaced lists must count it as the restatement does.
def full_cluster(P, racks, RF=3, seed=0):
    """A random current assignment over all 256 brokers; broker b in rack b // (256 / racks), so broker 255 is the last
    of the last rack, on slot 255"""
    rng = np.random.RandomState(seed)
    per = 256 // racks
    current = [list(map(int, rng.choice(256, size=RF, replace=False))) for _ in range(P)]
    return m.build_problem(current, list(range(256)), {b: "rack%02d" % (b // per) for b in range(256)}, RF)


def rf_down_onto_255(P, seed=0):
    """RF lowered from 4 to 3 in 16 racks of 16: every fifth partition has broker 255 fourth of four current replicas,
    the others three replicas on other brokers.  MODEL §4 drops the fourth, so the initial base's D is exactly the
    partitions whose one missing home is slot 255."""
    rng = np.random.RandomState(seed)
    current = []
    for p in range(P):
        row = list(map(int, rng.choice(255, size=3, replace=False)))
        current.append(row + [255] if p % 5 == 0 else row)
    return m.build_problem(current, list(range(256)), {b: "r%02d" % (b // 16) for b in range(256)}, 3)


HOME255_SHAPES = {
    "h255_r16_rr": lambda: m.synthetic_problem(1024, 256, 16, 3),      # config 5's layout: 16 racks of 16, round robin
    "h255_r32": lambda: full_cluster(600, 32, seed=110),               # 32 racks of 8
    "h255_r1": lambda: full_cluster(500, 1, seed=111),                 # one rack of 256: S = 256
    "h255_rf_down": lambda: rf_down_onto_255(600, seed=103),           # RF 4 -> 3, broker 255 fourth
    "h255_big": lambda: m.synthetic_problem(8200, 256, 16, 3, perturb=0.02, seed=5),    # the HBM path
}


def home_lists(pb, reps):
    """docs/MODEL.md §5.1 written out over replica lists (leader first, -1 padded): home[p] = the surviving brokers
    among the first four positions of cur[p]; home0[p] = cur[p][0] if it survives.  -> (D: partitions whose row lacks
    a home broker, DL: partitions that hold home0 but are led from another broker), both ascending"""
    D, DL = [], []
    for p in range(pb.P):
        row = [int(b) for b in reps[p] if b >= 0]
        home = {int(b) for b in pb.cur[p][:4] if 0 <= b < pb.B}
        if home - set(row):
            D.append(p)
        h0 = int(pb.cur[p][0])
        if 0 <= h0 < pb.B and h0 in row and row[0] != h0:
            DL.append(p)
    return D, DL


def home255_bases(pb, reps):
    """Bases that leave the guided operations no choice but slot 255, from a base `reps` with no displaced partition
    other than those missing only the broker on slot 255:
    - "d255": D is exactly the partitions whose only missing home is slot 255 (the broker there leaves every row that
      holds it as a non-leading home replica, for a broker no home list of that row names), DL is empty;
    - "dl255": DL is exactly the partitions whose home0 is slot 255 (each led from another of its replicas).
    Each list is checked with home_lists, so an edit to the construction cannot quietly empty it.  -> {name: base}"""
    b255 = int(np.flatnonzero(slots(pb) == 255)[0])
    D0, DL0 = home_lists(pb, reps)
    assert DL0 == [] and all(set(int(b) for b in pb.cur[p][:4] if 0 <= b < pb.B) - set(reps[p]) == {b255} for p in D0)
    out = {}
    d = reps.copy()
    for p in range(pb.P):
        row = list(d[p])
        if b255 in row[1:]:
            home = set(int(b) for b in pb.cur[p][:4])
            row[row.index(b255)] = next(b for b in range(pb.B) if b not in home and b not in row)
            d[p] = row
    D, DL = home_lists(pb, d)
    assert len(D) >= 3 and DL == [], (len(D), DL)
    assert all({int(b) for b in pb.cur[p][:4] if 0 <= b < pb.B} - set(d[p]) == {b255} for p in D)
    out["d255"] = d
    led = reps.copy()
    for p in range(pb.P):
        n = int((led[p] >= 0).sum())
        if int(pb.cur[p][0]) == b255 and led[p][0] == b255 and n > 1:
            led[p][:n] = np.roll(led[p][:n], -1)
    D, DL = home_lists(pb, led)
    want = [p for p in range(pb.P) if int(pb.cur[p][0]) == b255 and b255 in led[p] and led[p][0] != b255]
    if want:
        assert DL == want and D == D0, (DL, want)
        out["dl255"] = led
    return out


# ---- replication factors 5 to 8 and RF = B - 1 (docs/MODEL.md §1, §3.2, §4, §5) ------------------------------------
# Every shape above has RF <= 4 (C7_SHAPES reach 5 and 6 at 50 partitions).  Here: bit 2 and bit 3 of RF (the row pass
# compares bit-sliced counts with four slices of RF), shortfalls of 4 and more (the tensor-core shortfall planes), 8
# and 9 term planes at default weights (RFcur + 1 of them), initial bases that complete rows by five replicas or drop
# the tail, and RF = B - 1, where REPLACE has exactly one broker the row does not use.
RF_SHAPES = {
    "rf7_cm": lambda: make_problem(200, [8] * 8, 7, RFcur=3, seed=201, removed=2),        # column-major, C7 0..1
    "rf7_cur7": lambda: make_problem(200, [8] * 8, 7, seed=202),                         # 8 term planes
    "rf7_cur8": lambda: make_problem(200, [8] * 8, 7, RFcur=8, seed=203),                # 9 term planes: row-major
    "rf8_r8": lambda: make_problem(150, [8] * 8, 8, seed=204),                           # C7 1..1
    # RF 8 on the column-major evaluator: eight racks of eight with C7 0..1 (RF 8 is bit 3 of the row pass's count)
    "rf8_cm": lambda: dataclasses.replace(make_problem(150, [8] * 8, 8, RFcur=3, seed=214, removed=2), ppr_lo=0),
    "rf8_b9": lambda: make_problem(60, [9], 8, seed=205),                                # RF = B - 1, C7 8..8
    "rf8_r3_b9": lambda: make_problem(80, [4, 3, 2], 8, RFcur=5, seed=206),              # RF = B - 1, C7 2..3
    # RF = B - 1 = 2 with C7 1..1: every row needs the one broker of the second rack, so no base is feasible
    "rf2_b3": lambda: make_problem(40, [2, 1], 2, seed=207),
    "rf2_b3_r3": lambda: make_problem(40, [1, 1, 1], 2, seed=207),                       # RF = B - 1, column-major
    "rf8_w8": lambda: make_problem(120, [14] * 16, 8, seed=208, removed=3),              # 16-slot racks, W 8
    "rf5_w8": lambda: make_problem(120, [20] * 6, 5, seed=209, removed=2),               # 32-slot racks, W 8
    # 520 x RF 8 (P RF >= 4,096): the widest weights fit 12 bits, four current replicas keep packed entries
    "rf8_w12": lambda: with_widest_cost_field(make_problem(520, [8] * 8, 8, RFcur=4, seed=210), 210),
    "big_rf8": lambda: make_problem(8300, [8] * 8, 8, RFcur=3, seed=211),                # the HBM path
    "big_rf8_b9": lambda: make_problem(8300, [9], 8, seed=212),                          # the HBM path, RF = B - 1
}
# small enough for HiGHS (oracle/model.py solve_exact), and feasible: RF = B - 1 at both ends, RF 8 over 10 brokers.
# rf2_b3 is not among them: its C7 rows put every partition on the one broker of the second rack.
RF_EXACT_SHAPES = {
    "rf8_b9_p12": lambda: make_problem(12, [9], 8, seed=205),
    "rf2_b3_r3": RF_SHAPES["rf2_b3_r3"],
    "rf8_b10": lambda: make_problem(16, [5, 5], 8, seed=213),
}


def term_planes(pb):
    """docs/MODEL.md §3.2 written out: the term planes of an objective, one per (kind, value) class times the largest
    number of terms one partition has in it (kind F: wF, kind L: the bonus wL - wF); None if some wL < wF"""
    most = {}
    for p in range(pb.P):
        n = {}
        for b in np.flatnonzero(pb.wF[p] | pb.wL[p]):
            f, l = int(pb.wF[p, b]), int(pb.wL[p, b])
            if l < f:
                return None
            for cls in ((0, f), (1, l - f)):
                if cls[1]:
                    n[cls] = n.get(cls, 0) + 1
        for cls, k in n.items():
            most[cls] = max(most.get(cls, 0), k)
    return sum(most.values())


def one_per_rack_base(pb):
    """Rows of RF replicas in RF distinct racks (RF <= R): partition p takes racks p, p + 1, .. (mod R), in each the
    (p // R)-th broker (mod its size), leader first.  With C7 0..1 every row is well formed."""
    members = [np.flatnonzero(pb.rack_of == r) for r in range(pb.R)]
    out = np.empty((pb.P, pb.RF), np.int32)
    for p in range(pb.P):
        for k in range(pb.RF):
            rack = members[(p + k) % pb.R]
            out[p, k] = rack[(p // pb.R) % rack.size]
    return out


def reordered_base(reps):
    """Every row of `reps` with its replicas in another order: row p rotated by 1 + p mod (n - 1), n its replicas, so
    that another replica leads every row of two or more"""
    out = reps.copy()
    for p in range(out.shape[0]):
        n = int((out[p] >= 0).sum())
        if n > 1:
            out[p, :n] = np.roll(out[p, :n], -(1 + p % (n - 1)))
    return out


# ---- 64-bit seeds and late round numbers (docs/MODEL.md §5, §6) ----------------------------------------------------
# A candidate is a function of (base, seed, round, idx): the seed is Philox's 64-bit key, the round number its u32
# counter word 1, and every fourth round (round mod 4 = 3) a cycle round.  Seeds whose high word is set and round
# numbers at and above 2^16, 2^24 and 2^31, and calls that cross 2^32 (rounds first_round + i mod 2^32).
PHI = 0x9E3779B97F4A7C15            # kao_solve: restart r searches with seed + r * PHI mod 2^64
SEEDS = {
    "zero": 0,
    "2^32": 1 << 32,                                # low word 0, high word 1
    "high_word": 0xFFFFFFFF00000000,
    "all_ones": (1 << 64) - 1,
    "restart1_of_0": PHI,
    "goldens_low": 0xDEADBEEF00C0FFEE,              # low word 0xC0FFEE, the goldens' seed
}
# first rounds: free (round mod 4 != 3) and cycle rounds; 2^32 - 2 with a walk of more than two rounds crosses 2^32
ROUNDS = {
    "3": 3,
    "2^16-1": (1 << 16) - 1,
    "2^16": 1 << 16,
    "2^24-1": (1 << 24) - 1,
    "2^24": 1 << 24,
    "2^31+3": (1 << 31) + 3,
    "2^32-2": (1 << 32) - 2,
}
WRAP = ROUNDS["2^32-2"]


def round_at(first, i):
    """round i of a call that starts at `first` (docs/MODEL.md §6)"""
    return (first + i) % (1 << 32)


def patience_stop(keys, n):
    """The kernel's rule: stop after n rounds in a row whose (violation, cost) is not strictly better than the best so
    far -> rounds run"""
    best, stall = None, 0
    for t, k in enumerate(keys):
        vc = int(k) >> 24
        if best is None or vc < best:
            best, stall = vc, 0
        else:
            stall += 1
        if stall >= n:
            return t + 1
    return len(keys)


def ref_solve(r, seed, restarts, rounds, size, patience=0, chunk=100):
    """kao_solve restated over a restatement `r` (oracle/ref.py Ref, TRef, RRef): restart k resets to the initial base
    and searches with seed + k * PHI mod 2^64 from round 0 (stopping where patience says); the best final base by
    (violation, -objective) wins, the lowest restart on a tie.  -> dict(violation, objective, replicas, key, rounds
    (summed over the restarts), restart)"""
    best, total = None, 0
    for k in range(restarts):
        s = (seed + k * PHI) % (1 << 64)
        n = rounds
        if patience:
            bits, ld = r.init_base()
            keys = []
            while len(keys) < rounds and patience_stop(keys, patience) == len(keys):
                keys += list(r.search(bits, ld, s, len(keys), min(chunk, rounds - len(keys)), size)[1])
            n = patience_stop(keys, patience)
        bits, ld = r.init_base()
        _, keys = r.search(bits, ld, s, 0, n, size)
        total += n
        v, o = r.evaluate(bits, ld)
        if best is None or (v, -o) < (best["violation"], -best["objective"]):
            best = dict(violation=v, objective=o, replicas=r.decode(bits, ld), restart=k,
                        key=int(keys[-1]) if n else 0x7FFFFFFFFFFFFFFF)
    best["rounds"] = total
    return best
