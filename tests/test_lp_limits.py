"""The Lagrangian LP bound (docs/MODEL.md §9) at its build limits, without a GPU.

tests/lp_exact.py evaluates L(u) from its definition, with no code or structure in common with the rack DP that the
kernel (csrc/kao_lagrange.cu) and its restatement (tests/lp_ref) share.  It is checked here against the rational
enumeration of test_lp_bound on the small shapes, at u = 0 and at seeded multipliers that reach ±U.  Then, on shapes
at the limits MODEL §9 states, the restatement's bound is ⌊L_exact(u) / 2^F⌋ at the multipliers it returns, no
multiplier leaves the box, and the bound is never below a feasible assignment's objective or the LP relaxation.

The limit shapes (LIMITS, plus grid_shapes(n) for the CTA grid of a device with n SMs) are shared with
tests/test_gpu_lp_limits.py:
- RF 8 with C7 2..2 (racks of 10: at most 2 of 10 brokers a rack, so the leader is often outside the top list), C7
  2..3 on racks of 5, 6 and 7 (tight C6 totals), C7 1..2 with a dense table;
- 32 racks of 8 at RF 8 with 253 to 256 brokers (KAO_MAX_RACKS, every slot);
- 8,160 × 256 × RF 8 (P·RF = 65,280 and 2·256 + 32 = 544 rows), with and without two brokers removed, and
  8,160 × 64 × RF 8 in 16 racks;
- weights up to 65,535 (the widest a problem takes) at P·RF = 256, RF 8 and RF 1, where multipliers reach ±U;
- one topology at P ∈ {1, n − 1, n, n + 1, 2n + 1, 8159, 8160}: one partition per CTA up to n, then chunks of
  ⌈P/n⌉ with a shorter last CTA."""
import dataclasses
import functools
from fractions import Fraction

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
import lp_exact
import lp_ref
from conftest import make_problem
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import with_dense_weights, with_weights
from test_lp_bound import ALL, SMALL, lagrangian, lp_relaxation

SMS = 132               # SMs of an H100 SXM: the kernel runs one CTA per SM; the GPU file reads the device's count
LP_VARIABLES = 50000    # the LP relaxation (HiGHS) is solved up to this many variables


def windows_problem(P, B0, R, RF, remove=0, perturb=0.0, seed=0):
    """Brokers b in rack b % R; partition p currently on the RF consecutive brokers from p·RF (mod B0), that fraction
    of the replicas re-placed at random; the `remove` highest broker ids leave the cluster."""
    rng = np.random.RandomState(seed)
    current = [[(p * RF + i) % B0 for i in range(RF)] for p in range(P)]
    for _ in range(int(round(perturb * P * RF))):
        p, i, b = rng.randint(P), rng.randint(RF), rng.randint(B0)
        if b not in current[p]:
            current[p][i] = b
    return m.build_problem(current, list(range(B0 - remove)), {b: "r%02d" % (b % R) for b in range(B0)}, RF)


def windows_assignment(pb):
    """A feasible assignment of a windows_problem: replica j of the P·RF goes to broker j % B (consecutive brokers
    are in distinct racks, so C7 0..1 holds).  The windows' first brokers run through one residue class mod
    gcd(RF, B) every c = B / gcd(RF, B) partitions; in the q-th such cycle the window's (q mod RF)-th broker leads,
    so every RF cycles each broker leads once per cycle."""
    c = pb.B // np.gcd(pb.RF, pb.B)
    reps = np.zeros((pb.P, pb.RF), np.int32)
    for p in range(pb.P):
        w = [(p * pb.RF + i) % pb.B for i in range(pb.RF)]
        ld = w[(p // c) % pb.RF]
        reps[p] = [ld] + [b for b in w if b != ld]
    return reps


def with_rack_totals(pb, totals):
    """C6 rows of totals ± 1 and C3 rows to match: racks of different sizes with per-partition shares C7 admits"""
    size = np.bincount(pb.rack_of, minlength=pb.R)
    lo, hi = np.asarray(totals) - 1, np.asarray(totals) + 1
    return dataclasses.replace(pb, rack_lo=lo.astype(np.int32), rack_hi=hi.astype(np.int32),
                               rep_lo=(lo // size)[pb.rack_of].astype(np.int32),
                               rep_hi=(-(-hi // size))[pb.rack_of].astype(np.int32))


def with_16bit_weights(pb, seed, favoured):
    """Dense weights 0..999 and 65,535 on the favoured brokers: C3 binds there at a multiplier above U"""
    rng = np.random.RandomState(seed)
    wF, wL = rng.randint(0, 1000, size=pb.wF.shape), rng.randint(0, 1000, size=pb.wL.shape)
    wF[:, favoured] = wL[:, favoured] = 65535
    return with_weights(pb, wF, wL)


# name -> (problem, how its feasible assignment is found: "exact" = HiGHS optimum, "windows" = windows_assignment)
LIMITS = {
    "rf8_c7_22": (lambda: make_problem(60, [10] * 4, 8, seed=101), "exact"),
    "rf8_c7_23": (lambda: with_rack_totals(make_problem(60, [5, 6, 7], 8, seed=102), [140, 162, 178]), "exact"),
    "rf8_c7_12_dense": (lambda: with_dense_weights(make_problem(40, [6] * 5, 8, seed=103), 103), "exact"),
    "w16_rf8": (lambda: with_16bit_weights(make_problem(32, [5] * 5, 8, seed=104), 104, [0, 1, 2]), "exact"),
    "w16_rf1": (lambda: with_16bit_weights(make_problem(256, [4, 4], 1, seed=105), 105, [0, 1]), "exact"),
    **{"r32_b%d" % (256 - rm): (lambda rm=rm: windows_problem(96, 256, 32, 8, remove=rm, perturb=0.05, seed=110 + rm),
                                "windows") for rm in range(4)},
    "size_8160": (lambda: windows_problem(8160, 256, 32, 8, perturb=0.02, seed=1), "windows"),
    "size_8160_rm2": (lambda: windows_problem(8160, 256, 32, 8, remove=2, perturb=0.02, seed=1), "windows"),
    "size_8160_b64": (lambda: windows_problem(8160, 64, 16, 8, perturb=0.02, seed=1), "windows"),
}
BIG = ["size_8160", "size_8160_rm2", "size_8160_b64"]


def grid_shapes(n):
    """one topology (40 brokers, 8 racks, RF 4) at the partition counts where the kernel's grid changes shape"""
    return {"grid_%d" % P: (lambda P=P: windows_problem(P, 40, 8, 4, perturb=0.05, seed=120), "windows")
            for P in sorted({1, n - 1, n, n + 1, 2 * n + 1, 8159, 8160})}


SHAPES = {**LIMITS, **grid_shapes(SMS)}


def iterations(name):
    """the iteration caps a shape is checked at: 1,000 too where P·B is small"""
    return (1, 7, 100) if name in BIG or name in ("grid_8159", "grid_8160") else (1, 7, 100, 1000)


def last_cta(P, n):
    """(partitions per CTA, partitions of the last CTA) of the kernel's grid on n SMs"""
    chunk = -(-P // min(n, P))
    return chunk, P - (-(-P // chunk) - 1) * chunk


@functools.lru_cache(maxsize=None)
def instance(name):
    """(problem, a feasible assignment, its objective)"""
    factory, how = SHAPES[name]
    pb = factory()
    reps = m.solve_exact(pb).replicas if how == "exact" else windows_assignment(pb)
    viol, obj = m.evaluate(pb, reps)
    assert viol == 0, name
    return pb, reps, obj


@functools.lru_cache(maxsize=None)
def restatement(name, k):
    pb, _, T = instance(name)
    return lp_ref.lp_bound(pb, T, k)


def test_exact_evaluator_uses_the_build_constants():
    assert lp_exact.F == lp_ref.fraction_bits() == kopt.LP_FRACTION_BITS and lp_exact.U == lp_ref.box()


def seeded_multipliers(pb, seed):
    """u = 0; uniform in [-U, U] with a third of the entries at +U or -U; only u4 non-zero; only u6 non-zero"""
    rng = np.random.RandomState(seed)
    NR, B, U = 2 * pb.B + pb.R, pb.B, lp_exact.U
    out = [np.zeros(NR, np.int64)]
    for _ in range(3):
        u = rng.randint(-U, U + 1, size=NR, dtype=np.int64)
        pick = rng.rand(NR)
        u[pick < 1 / 6] = U
        u[(pick >= 1 / 6) & (pick < 1 / 3)] = -U
        out.append(u)
    for part in (slice(B, 2 * B), slice(2 * B, NR)):
        u = np.zeros(NR, np.int64)
        u[part] = rng.randint(-U, U + 1, size=u[part].size, dtype=np.int64)
        u[part][0] = U
        out.append(u)
    return out


@pytest.mark.parametrize("name", SMALL)
def test_exact_evaluator_matches_the_enumeration(name):
    pb = ALL[name]()
    for u in seeded_multipliers(pb, 7):
        assert Fraction(lp_exact.lagrangian_fixed(pb, u), 1 << lp_exact.F) == lagrangian(pb, u)


@functools.lru_cache(maxsize=None)
def relaxation(name):
    pb = instance(name)[0]
    return int(np.floor(lp_relaxation(pb) + 1e-6)) if 2 * pb.P * pb.B <= LP_VARIABLES else None


@pytest.mark.parametrize("name,k", [(n, k) for n in SHAPES for k in iterations(n)])
def test_restatement_is_exact_at_the_limits(name, k):
    pb, _, T = instance(name)
    bound, its, u = restatement(name, k)
    assert 1 <= its <= k and u.shape == (2 * pb.B + pb.R,)
    assert (np.abs(u) <= lp_exact.U).all()
    assert lp_exact.lagrangian_fixed(pb, u) >> lp_exact.F == bound
    assert bound >= T
    lp = relaxation(name)
    assert lp is None or bound >= lp, (bound, lp)


def test_the_matrix_reaches_the_limits():
    """What the shapes reach: RF 8, 32 racks, 544 rows, P·RF = 65,280, weight 65,535, a short last CTA on SMS SMs —
    and, in the restatement's results, multipliers of C4 and C6 rows that moved and one at ±U."""
    big = instance("size_8160")[0]
    assert (big.RF, big.R, 2 * big.B + big.R, big.P * big.RF) == (8, 32, 544, 65280)
    assert max(int(instance(n)[0].wL.max()) for n in ("w16_rf8", "w16_rf1")) == 65535
    assert {instance(n)[0].RF for n in ("w16_rf8", "w16_rf1")} == {1, 8}
    assert sorted(instance("r32_b%d" % b)[0].B for b in range(253, 257)) == [253, 254, 255, 256]
    assert any(last_cta(P, SMS)[1] < last_cta(P, SMS)[0] for P in (2 * SMS + 1, 8159, 8160))
    lows = {(instance(n)[0].ppr_lo, instance(n)[0].ppr_hi) for n in ("rf8_c7_22", "rf8_c7_23", "rf8_c7_12_dense")}
    assert lows == {(2, 2), (2, 3), (1, 2)}
    u4 = u6 = box = False
    for name in SHAPES:
        if name in BIG:
            continue
        pb = instance(name)[0]
        for k in iterations(name):
            u = restatement(name, k)[2]
            u4 |= bool(u[pb.B:2 * pb.B].any())
            u6 |= bool(u[2 * pb.B:].any())
            box |= bool((np.abs(u) == lp_exact.U).any())
    assert u4 and u6 and box


def test_kao_lp_bound_refuses_8161_partitions_before_any_cuda_call():
    """P = 8,161 at RF 8 (P·RF = 65,288 < 2^16): the partition limit alone refuses it, with KAO_E_ARG, also where
    there is no device (which would be KAO_E_CUDA)"""
    pb = windows_problem(8161, 256, 32, 8)
    with pytest.raises(kao.KaoError, match=r"libkao error -1: kao_lp_bound: .*P <= 8,160"):
        kopt.lp_bound(kao.Problem.from_fields(pb), windows_assignment(pb))
