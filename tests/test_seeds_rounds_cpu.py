"""64-bit seeds and late round numbers without a GPU (problems.SEEDS, problems.ROUNDS).  A candidate is a pure function
of (base, seed, round, idx) (docs/MODEL.md §5): the seed is Philox's 64-bit key and the round number its u32 counter
word 1, which also picks the cycle rounds (round mod 4 = 3) and the round the sorted-batch body builds its next list
for.  Every other bit-exact test of the suite uses seeds below 2^32 and round numbers below 2^16, so a search that
dropped the seed's high word or narrowed the round word would pass it.

The engine's device code compiled for the host (tests/emu: the row-major, column-major and delta evaluators, the
tensor-core body with and without sorted batches) is held bit for bit to the restatement (oracle/kao_ref.c) at every
(seed, first round) pair, over 8-round walks that cross 2^32 (a call runs rounds first_round + i mod 2^32, docs/MODEL.md
§6), and a call that crosses 2^32 equals the same rounds split into two calls.  The restatement itself must use both
words: candidates at s and s ^ 2^32, and at rounds t and t ^ 2^16, t ^ 2^24, t ^ 2^31, differ."""
import json
import threading
import urllib.request

import numpy as np
import pytest

import kafka_assignment_optimizer_b200 as kao
from kafka_assignment_optimizer_b200 import service
from problems import ROUNDS, SEEDS, SHAPES, WRAP, moved_base, round_at
from test_gpu_large_layouts import assert_keys
from test_host import README_CURRENT

# one shape per row width: W = 1 and 2 on the column-major evaluator, W = 4 and 8 row-major only
CPU_SHAPES = ["cfg2", "cfg3_small", "w4_s16", "w8_s16"]
SIZE = 128                          # candidates of a key round and of a walk's rounds; the last one is the identity
WALK = 8                            # rounds of a walk from 2^32 - 2: rounds 2^32 - 2, 2^32 - 1, 0, .., 5
KTAG = 0x4B414F21                   # Philox counter word 3 of the control word (docs/MODEL.md §5)


@pytest.fixture(scope="module")
def emu():
    import emu as emu_mod

    emu_mod.lib()
    return emu_mod


def sessions(emu, pb):
    """name -> emulated session: row-major and, where the layout allows it, column-major and the tensor-core body"""
    out = {"row_major": emu.EmuSession(kao.Problem.from_fields(pb))}
    cm = emu.EmuSession(kao.Problem.from_fields(pb))
    if cm.set_evaluator(1):
        out["column_major"] = cm
        out["mma"] = emu.MmaSession(kao.Problem.from_fields(pb), 0x300)
    else:
        cm.close()
    return out


def start_base(pb, r):
    """a damaged base: long displaced lists, so that guided operations and cycle rounds have partitions to pick"""
    return moved_base(pb, r.decode(*r.init_base()), 6)


# ---- the restatement uses every bit of the seed and of the round --------------------------------------------------------
def _differing(r, bits, ld, a, b):
    """candidates 0 .. SIZE - 2 generated at (seed, round) a and b: how many differ"""
    n = 0
    for idx in range(SIZE - 1):
        x, y = r.gen(bits, ld, a[0], a[1], idx, SIZE), r.gen(bits, ld, b[0], b[1], idx, SIZE)
        n += not (np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]))
    return n


@pytest.mark.parametrize("seed", sorted(SEEDS))
def test_the_restatement_reads_the_seeds_high_word_and_every_round_bit(ref_lib, seed):
    pb = SHAPES["cfg2"]()
    r = ref_lib.Ref(pb)
    bits, ld = r.encode(start_base(pb, r))
    s = SEEDS[seed]
    for rnd in (2, 3):                                               # a free and a cycle round
        assert _differing(r, bits, ld, (s, rnd), (s ^ (1 << 32), rnd)) > SIZE // 2, (seed, rnd)
    for rnd in (ROUNDS["2^16"], ROUNDS["2^24-1"], ROUNDS["2^31+3"]):
        for bit in (16, 24, 31):
            assert _differing(r, bits, ld, (s, rnd), (s, rnd ^ (1 << bit))) > SIZE // 2, (seed, rnd, bit)


@pytest.mark.parametrize("seed", sorted(SEEDS))
def test_a_call_across_2_32_is_its_rounds_one_by_one(ref_lib, seed):
    """docs/MODEL.md §6: a call from 2^32 - 2 runs rounds 2^32 - 2, 2^32 - 1, 0, 1, ..; it equals the same rounds in two
    calls and one call per round"""
    pb = SHAPES["cfg2"]()
    r = ref_lib.Ref(pb)
    start = start_base(pb, r)
    s = SEEDS[seed]
    bits, ld = r.encode(start)
    _, whole = r.search(bits, ld, s, WRAP, WALK, SIZE)
    split_bits, split_ld = r.encode(start)
    split = np.concatenate([r.search(split_bits, split_ld, s, WRAP, 2, SIZE)[1],
                            r.search(split_bits, split_ld, s, 0, WALK - 2, SIZE)[1]])
    one_bits, one_ld = r.encode(start)
    one = np.concatenate([r.search(one_bits, one_ld, s, round_at(WRAP, i), 1, SIZE)[1] for i in range(WALK)])
    assert (whole != 0).all() and (whole < 0x7FFFFFFFFFFFFFFF).all()
    assert_keys(whole, split, "split")
    assert_keys(whole, one, "one by one")
    assert np.array_equal(bits, split_bits) and np.array_equal(ld, split_ld)
    assert np.array_equal(bits, one_bits) and np.array_equal(ld, one_ld)


# ---- the device code at every (seed, round) pair -------------------------------------------------------------------------
@pytest.mark.parametrize("name", CPU_SHAPES)
def test_emulated_keys_at_every_seed_and_round(emu, ref_lib, name):
    """keys of every evaluator, the delta keys and the tensor-core body's batches, sorted (a CTA share below the list's
    capacity) and unsorted (above it), against the restatement at every (seed, first round) pair"""
    pb = SHAPES[name]()
    r = ref_lib.Ref(pb)
    start = start_base(pb, r)
    bits, ld = r.encode(start)
    runs = sessions(emu, pb)
    assert ("mma" in runs) == (r.W <= 2), name
    for sess in runs.values():
        sess.set_base(start)
    for seed, s in sorted(SEEDS.items()):
        for rnd_name, rnd in sorted(ROUNDS.items()):
            tag = (seed, rnd_name)
            want = r.candidate_keys(bits, ld, s, rnd, SIZE, 0, SIZE)
            for who, sess in runs.items():
                assert_keys(sess.candidate_keys(s, rnd, SIZE, 0, SIZE), want, tag + (who,))
            assert_keys(runs["row_major"].candidate_keys(s, rnd, SIZE, 0, SIZE, delta=True), want, tag + ("delta",))
            if "mma" in runs:
                for cap in (8192, 16):
                    assert_keys(runs["mma"].sorted_keys(s, rnd, SIZE, 0, SIZE, 2, 4, cap), want, tag + ("sorted", cap))
    for sess in runs.values():
        sess.close()


@pytest.mark.parametrize("name", CPU_SHAPES)
def test_emulated_walks_across_2_32(emu, ref_lib, name):
    """8 rounds from 2^32 - 2 at every seed on every evaluator: in one call, and in two calls split at the wrap; the
    patched state matches the state rebuilt from the walked base, which is the restatement's"""
    pb = SHAPES[name]()
    r = ref_lib.Ref(pb)
    start = start_base(pb, r)
    runs = sessions(emu, pb)
    for seed, s in sorted(SEEDS.items()):
        bits, ld = r.encode(start)
        _, want = r.search(bits, ld, s, WRAP, WALK, SIZE)
        for who, sess in runs.items():
            for split in (False, True):
                tag = (seed, who, "split" if split else "one call")
                sess.set_base(start)
                got = (np.concatenate([sess.search(s, WRAP, 2, SIZE), sess.search(s, 0, WALK - 2, SIZE)]) if split
                       else sess.search(s, WRAP, WALK, SIZE))
                assert_keys(got, want, tag)
                rc, at, msg = sess.check_state()
                assert rc == 0, tag + (rc, at, msg)
                end, v, o, _ = sess.get_base()
                assert (end == r.decode(bits, ld)).all() and (v, o) == r.evaluate(bits, ld), tag
    for sess in runs.values():
        sess.close()


# ---- sorted batches at high seeds ------------------------------------------------------------------------------------
def control_class(ref_lib, seed, rnd, idx, size):
    """The class of a candidate's control word as csrc/kao_device_mma.cuh (cand_class) defines it, with the control
    word from the restatement's Philox; a change to that definition is made there and here.  0 the identity; a cycle
    round: 1 + its two role-match bits; else operations << 6 | first-operation LEADER and guided bits << 4 | link kind
    of operation 2 << 2 | of operation 3"""
    if idx + 1 == size:
        return 0
    ctl = ref_lib.Ref.philox([idx, rnd, 0, KTAG], [seed & 0xFFFFFFFF, seed >> 32])[0]
    if rnd & 3 == 3:
        return 1 + ((ctl >> 11) & 1) * 2 + ((ctl >> 13) & 1)
    nops = 1 if ctl & 3 == 0 else (3 if ctl & 3 == 3 else 2)
    return nops << 6 | ((ctl >> 2) & 3) << 4 | ((((ctl >> 4) & 3) << 2) if nops >= 2 else 0) | (((ctl >> 7) & 3) if nops == 3 else 0)


@pytest.mark.parametrize("rnd", [2, 3])
@pytest.mark.parametrize("seed", sorted(SEEDS))
def test_batches_mostly_share_one_class_at_high_seeds(emu, ref_lib, seed, rnd):
    """At the headline's CTA share a batch of the sorted list holds few classes of control word (unsorted: about 20 in a
    free round, about 4 in a cycle round), counted from the candidates' control words as the restatement draws them: the
    sort must read the same 64-bit key"""
    s, size = SEEDS[seed], 1 << 18
    lst, _, bounds, is_sorted = emu.cta_batches(s, rnd, size, 0, size, 132, 16, 8192, 0)
    assert is_sorted
    cls = np.array([control_class(ref_lib, s, rnd, int(i), size) for i in lst])
    per_batch = [len(set(cls[a:b].tolist())) for a, b in zip(bounds[:-1], bounds[1:])]
    assert np.mean(per_batch) < 3, (seed, rnd, np.mean(per_batch))


# ---- the service ---------------------------------------------------------------------------------------------------------
def test_submit_passes_a_64_bit_seed_through_unchanged():
    """POST /submit over HTTP (JSON integers of 2^63 and more) to a stand-in solver: the seed arrives as sent"""
    from test_service import SEEN, oracle_solver

    srv = service.make_server(port=0, solver=oracle_solver)
    threading.Thread(target=srv.serve_forever, daemon=True).start()
    try:
        base = {"assignment": json.loads(README_CURRENT), "brokers": ",".join(map(str, range(19))),
                "racks": ",".join("%d:%s" % (b, "b" if b % 2 else "a") for b in range(20)), "rf": 2, "restarts": 3}
        for s in ((1 << 63) + 5, (1 << 64) - 1, SEEDS["goldens_low"]):
            req = urllib.request.Request("http://127.0.0.1:%d/submit" % srv.server_address[1],
                                         data=json.dumps(dict(base, seed=s)).encode(),
                                         headers={"Content-Type": "application/json"})
            out = json.loads(urllib.request.urlopen(req, timeout=60).read())
            assert SEEN["seed"] == s and SEEN["restarts"] == 3 and out["feasible"], s
    finally:
        srv.shutdown()
        srv.server_close()
