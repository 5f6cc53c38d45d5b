"""The shapes that run on the HBM-base search path (DESIGN.md 7.1: every topic session, every instance above 8,160
partitions), on the host: they reach every layout that path's general-bounds evaluator tells apart and every edge it
handles on its own, and the candidate stream keeps the premise its delta evaluation and topic events rest on
(docs/MODEL.md §8): a candidate differs from its base in at most three rows, each by at most one replica move and one
leader change."""
import dataclasses

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import optimizer as kopt
from oracle import model as m
from problems import C7_SHAPES, LARGE_SHAPES, LAYOUT_SHAPES, SHAPES, emptied_base, moved_base, with_widest_cost_field
from conftest import make_problem

HBM_SHAPES = {**SHAPES, **LAYOUT_SHAPES, **C7_SHAPES, **LARGE_SHAPES}


def rack_field(pb):
    """Slots per rack (the smallest power of two >= max(8, largest rack)) as the field the evaluator reads"""
    S = 8
    while S < np.bincount(pb.rack_of, minlength=pb.R).max():
        S <<= 1
    return {8: "8", 16: "16"}.get(S, "word")


def c7_form(pb):
    if (pb.ppr_lo, pb.ppr_hi) in ((0, 1), (1, 1)):
        return "%d..%d" % (pb.ppr_lo, pb.ppr_hi)
    assert pb.ppr_lo > 0, (pb.ppr_lo, pb.ppr_hi)
    return "lo>0"


def objective_form(pb):
    """Packed entries hold at most four non-zero cells of 12 bits per partition; anything else is the dense table"""
    cells = ((pb.wF > 0) | (pb.wL > 0)).sum(1).max()
    return "dense" if max(pb.wF.max(), pb.wL.max()) > 4095 or cells > 4 else "entries"


def impossible(W, rack, c7):
    """Why a (row width, rack field, C7 form) cannot occur, or None.  C7 1..1 needs RF = R racks, a lower bound
    above 0 needs RF > R, and RF <= 8."""
    if c7 != "0..1" and rack == "8" and W >= 4:
        return "rows of more than 64 slots in 8-slot racks are at least nine racks"
    if c7 != "0..1" and rack == "16" and W == 8:
        return "rows of more than 128 slots in 16-slot racks are at least nine racks"
    return None


def edges(name, pb, r):
    out = set()
    rows = (pb.cur >= 0).sum(1)
    if pb.cur.shape[1] < pb.RF:
        out.add("RF raised")
    if pb.cur.shape[1] > pb.RF:
        out.add("RF lowered")
    if rows.min() < rows.max() and rows.min() == 0:
        out.add("ragged rows")
    if pb.RF == 1:
        out.add("RF 1")
    if pb.P == 1:
        out.add("P = 1")
    if pb.P > 8160:
        out.add("P > 8,160")
    if r.evaluate(*r.init_base())[0] > (1 << (39 - r.obj_bits)) - 1:
        out.add("saturation")
    # the emptied-row base: partitions led from a slot they do not hold (nbad > 0)
    bits, ld = r.encode(emptied_base(pb, r.decode(*r.init_base()), 5))
    if (bits == 0).all(1).any() and (ld == 0xFF).any():
        out.add("nbad > 0")
    return out


def test_hbm_shapes_reach_every_layout_and_edge(ref_lib):
    """Every (W, rack field, C7 form, objective form) that can occur is reached by a shape the HBM-path tests run,
    and so is every edge of that path; all of it from the problem fields and the restatement's layout."""
    possible = {(W, rack, c7, obj) for W in (1, 2, 4, 8) for rack in ("8", "16", "word")
                for c7 in ("0..1", "1..1", "lo>0") for obj in ("entries", "dense") if impossible(W, rack, c7) is None}
    reached, seen = set(), set()
    for name, f in HBM_SHAPES.items():
        pb = f()
        r = ref_lib.Ref(pb)
        reached.add((r.W, rack_field(pb), c7_form(pb), objective_form(pb)))
        seen |= edges(name, pb, r)
    assert not {t for t in reached if impossible(*t[:3])}, "a shape reached a combination listed as impossible"
    assert sorted(possible - reached) == []
    assert seen == {"RF raised", "RF lowered", "ragged rows", "RF 1", "P = 1", "saturation", "P > 8,160", "nbad > 0"}


def test_large_shapes_are_what_their_names_say(ref_lib):
    for name, f in LARGE_SHAPES.items():
        pb = f()
        assert pb.P > 8160, name
        assert kopt.key_obj_bits(kao.Problem.from_fields(pb)) > 0, name
    assert kopt.key_obj_bits(kao.Problem.from_fields(LARGE_SHAPES["big_obj24"]())) == 24
    assert objective_form(LARGE_SHAPES["big_dense_w4"]()) == "dense"
    assert ref_lib.Ref(LARGE_SHAPES["big_ppr11_w8"]()).W == 8


def test_weights_above_12_bits_exceed_the_objective_range_above_4096_partition_replicas():
    """Why LARGE_SHAPES has no weights above 12 bits: the engine refuses any instance whose P * RF * largest weight
    reaches 2^24, and 8,161 * 4,096 does."""
    lib = kopt.load_library()
    pb = make_problem(8161, [4, 4, 4], 1, seed=3)
    assert kopt.key_obj_bits(kao.Problem.from_fields(with_widest_cost_field(pb, 1))) == 24
    wide = _every_weight(pb, 4096)
    assert lib.kao_key_obj_bits(kopt._CProblem(kao.Problem.from_fields(wide)).ref()) == -1
    assert "24 bits" in lib.kao_last_error().decode()


def _every_weight(pb, w):
    wF = np.where(pb.wF > 0, w, 0).astype(np.uint16)
    return dataclasses.replace(pb, wF=wF, wL=np.where(pb.wL > 0, w, 0).astype(np.uint16))


# ---- the premise of delta evaluation ------------------------------------------------------------------------
def _bases(pb, r):
    bits, ld = r.init_base()
    reps = r.decode(bits, ld)
    return {"initial": (bits, ld), "emptied": r.encode(emptied_base(pb, reps, 5)),
            "moved": r.encode(moved_base(pb, reps, 6))}


def _held(bits, ld):
    """per row: the leader byte names a slot the row holds"""
    W = bits.shape[1]
    ok = ld < 32 * W
    s = np.where(ok, ld, 0).astype(np.int64)
    word = bits[np.arange(bits.shape[0]), s >> 5]
    return ok & (((word >> (s & 31).astype(np.uint32)) & 1) == 1)


@pytest.mark.parametrize("name", sorted(HBM_SHAPES))
def test_candidates_move_at_most_one_replica_and_one_leader_per_row(ref_lib, name):
    """Every candidate drawn (free and cycle rounds, from the initial base and both damaged ones) differs from its
    base in at most 3 rows, and each such row loses at most one slot and gains at most one.  No candidate changes
    whether a row's leader is a slot the row holds: the count of such rows (nbad) is a constant of a search."""
    pb = HBM_SHAPES[name]()
    r = ref_lib.Ref(pb)
    n = 256 if pb.P > 8160 else 1024
    for base, (bits, ld) in _bases(pb, r).items():
        held = _held(bits, ld)
        for rnd in (0, 3, 6, 7):
            for idx in range(n):
                cb, cl = r.gen(bits, ld, 0xD17A, rnd, idx, 4096)
                rows = np.flatnonzero((cb != bits).any(1) | (cl != ld))
                assert rows.size <= 3, (base, rnd, idx, rows)
                if rows.size == 0:
                    continue
                lost = np.bitwise_count(bits[rows] & ~cb[rows]).sum(1)
                gained = np.bitwise_count(cb[rows] & ~bits[rows]).sum(1)
                assert (lost <= 1).all() and (gained <= 1).all(), (base, rnd, idx, rows, lost, gained)
                changed = held[rows] != _held(cb[rows], cl[rows])
                assert not changed.any(), (base, rnd, idx, rows[changed])
