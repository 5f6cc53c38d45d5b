"""Measuring the engine's full-evaluation variants on the GPU at hand.

The engine has two full evaluators with bit-identical results (column-major: the default wherever the
layout allows it, docs/MODEL.md §3.3; row-major: every layout) and builds the column-major one in a few
*schedules* of the same arithmetic (include/kao.h, kao_set_schedule).  The library's default schedule is
the one that was fastest on an H100 (config 3); nothing has to be tuned to get it.  `probe()` re-measures
every built variant on the caller's problem — `python bench.py --probe-schedules` prints its lines — and
checks that all of them return the row-major evaluator's round keys and final assignment.
"""
from __future__ import annotations

import json

# (sync, pop, threads) — the variants csrc/kao_kernels.cuh builds (KAO_FOR_SCHEDULES); the first is the default.
# pop 0x100: the sums on the tensor cores (binary MMA, csrc/kao_device_mma.cuh); 0x200: the same with the merged generator;
# 0x300: the same with each CTA's candidates sorted by class (control word) before a round, so a batch runs mostly one body,
# and the MMA epilogue scoring two candidates per instruction in 16 x 2 halfword pairs; 0x1300: the same with the epilogue
# in 32 bits per candidate
SCHEDULES = [(1, 0x300, 512), (1, 0x1300, 512), (1, 0x200, 512), (1, 0x100, 512), (4, 0x22, 1024), (4, 0x22, 896)]
DEFAULT_SCHEDULE = SCHEDULES[0]
SCHEDULE_FIELDS = ("sync", "pop", "threads")


def schedule_name(sched) -> str:
    return "column_major sync=%d pop=%05x threads=%d" % tuple(sched)


def probe(pb, device: int = 0, rounds: int = 32, round_size: int = 1 << 18, seed: int = 0x5EED, out=print):
    """One warm, one recorded and two timed launches of `rounds` rounds with each variant on the same
    stream of candidates.  -> list of dicts (also printed as `PROBE {json}` lines)."""
    from .optimizer import Session

    ref, rows = {}, []

    def run(name, col, sched):
        sess = Session(pb, device=device)
        try:
            if not sess.set_evaluator(col):
                return {"name": name, "error": "layout not covered"}
            if sched is not None and not sess.set_schedule(*sched):
                return {"name": name, "error": "schedule not built"}
            sess.search(seed, 50_000, 2, round_size)
            sess.reset()
            keys, _ = sess.search(seed, 60_000, rounds, round_size)
            base = sess.get_base()[0]
            ms = min(sess.search(seed, 70_000 + i * rounds, rounds, round_size)[1] for i in range(2))
            if not ref:
                ref["keys"], ref["base"] = keys.copy(), base.copy()
            same = bool((keys == ref["keys"]).all() and (base == ref["base"]).all())
            return {"name": name, "schedule": list(sched) if sched else None, "ms_per_launch": ms,
                    "identical_to_row_major": same}
        finally:
            sess.close()

    for name, col, sched in [("row_major", False, None)] + [(schedule_name(s), True, s) for s in SCHEDULES]:
        row = run(name, col, sched)
        rows.append(row)
        out("PROBE " + json.dumps(row))
    return rows
