"""Walks of the shared-memory search kernel's column-major forms under the warp emulators (tests/emu: popcount forms
1-6 and the tensor-core body), with the state every winner patches checked against the same state rebuilt
from the base every 10 rounds (kao_emu_check_state): the transposed, term, rack-field and shortfall planes t_patch_row
rewrites, the leader one-hot plane, the count of invalid leaders that decides whether the leader plane answers the
generator, and the displaced lists.  A mis-patched plane that never changes a winner is invisible to every GPU
trajectory; here it fails at the first check after it happens.  Keys are held to the restatement (oracle/kao_ref.c)."""
import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from oracle import model as m
from problems import LAYOUT_SHAPES, SHAPES, emptied_base, moved_base, with_saturating_violation

CM_SHAPES = {
    "cfg2": SHAPES["cfg2"],
    "cfg2_rm2": SHAPES["cfg2_rm2"],
    "cfg3": lambda: m.synthetic_problem(1000, 64, 8, 3),                  # 32 words: the compile-time form
    "cfg3_small": SHAPES["cfg3_small"],
    "p1100": lambda: m.synthetic_problem(1100, 64, 8, 3, remove=2),       # 64 words: the run-time form
    "planes8_w1": LAYOUT_SHAPES["planes8_w1"],
    "planes8_w2": LAYOUT_SHAPES["planes8_w2"],
    "rf1": SHAPES["rf1"],
    "rf_down": SHAPES["rf_down"],
    "widecm_cfg2": LAYOUT_SHAPES["widecm_cfg2"],
    "widecm_cfg3_small": LAYOUT_SHAPES["widecm_cfg3_small"],
    # the initial base violates the rows by the key's cap + 7: saturated winners first, then the way out
    "sat_cm_cfg2": lambda: with_saturating_violation(LAYOUT_SHAPES["widecm_cfg2"]()),
    "sat_cm_cfg3_small": lambda: with_saturating_violation(LAYOUT_SHAPES["widecm_cfg3_small"]()),
}
CHECK = 10                          # rounds between state checks
PROBE = (300, 4)                    # rounds x candidates: each winner the best of three candidates and the identity
LONG = (60, 512)


@pytest.fixture(scope="module")
def emu():
    import emu as emu_mod

    emu_mod.lib()
    return emu_mod


@pytest.fixture(scope="module")
def mma(emu):
    return lambda pb: emu.MmaSession(pb, 0x300)


def product(pb):
    return kao.Problem.from_fields(pb)


def walk(sess, r, start, want, seed, size, what):
    """`want`: the restatement's round keys from `start`; the session walks them CHECK rounds per call and its patched
    state must equal the rebuilt one after every call"""
    sess.set_base(start)
    for first in range(0, len(want), CHECK):
        got = sess.search(seed, first, CHECK, size)
        bad = np.flatnonzero(got != want[first:first + CHECK])
        assert bad.size == 0, (what, "round", first + int(bad[0]), r.unpack_key(got[bad[0]]),
                               r.unpack_key(want[first + bad[0]]))
        rc, at, msg = sess.check_state()
        assert rc == 0, (what, "after round", first + CHECK - 1, rc, at, msg)


@pytest.mark.parametrize("name", sorted(CM_SHAPES))
def test_patched_state_equals_the_rebuilt_state_along_walks(emu, mma, ref_lib, name):
    pb = CM_SHAPES[name]()
    r = ref_lib.Ref(pb)
    reps = r.decode(*r.init_base())
    starts = {"initial": reps}
    if not name.startswith("sat_"):
        starts.update(moved=moved_base(pb, reps, 6), emptied=emptied_base(pb, reps, 5))
        assert (r.encode(starts["emptied"])[1] == 0xFF).any()     # partitions led from no replica: the count > 0
    forms = {}
    for form in range(1, 7):
        sess = emu.EmuSession(product(pb))
        assert sess.set_evaluator(form), (name, form)
        forms["form %d" % form] = sess
    forms["mma"] = mma(product(pb))
    cap = (1 << (39 - r.obj_bits)) - 1
    for what, start in starts.items():
        walks = [(PROBE, list(forms))]
        if what != "initial" or name.startswith("sat_"):         # long walks from the damaged bases
            walks.append((LONG, ["mma", "form 1"]))
        for (rounds, size), runs in walks:
            seed = 0x5EED + 31 * len(what) + size
            bits, ld = r.encode(start)
            _, want = r.search(bits, ld, seed, 0, rounds, size)
            if name.startswith("sat_") and size == LONG[1]:
                assert r.unpack_key(want[0])[0] == cap
            for form in runs:
                sess = forms[form]
                walk(sess, r, start, want, seed, size, (what, form, rounds, size))
                reps_end, v, o, _ = sess.get_base()
                mv, mo = m.evaluate(pb, reps_end)
                # the emulators evaluate the base as a packed key: its violation field caps a saturated one
                assert (reps_end == r.decode(bits, ld)).all() and (v, o) == (min(mv, cap), mo), (what, form)
    for sess in forms.values():
        sess.close()
