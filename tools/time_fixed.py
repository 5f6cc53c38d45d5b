#!/usr/bin/env python
"""Fixed partitions (docs/MODEL.md §12, DESIGN.md 7.4) on one GPU: "move these topics and leave everything else where it
is" through kao_solve_fixed, against kao_solve over the whole cluster with the same options.

Instance: 65,280 partitions x 64 brokers x 8 racks, RF 3, in 1,306 topics of up to 50 (tools/time_topics.py), broker 63
removed.  A partition is searched when its topic is moved or when it has a replica on broker 63 (about 3,060 of them),
every other one is fixed, as `kao-cli --topics-to-move` decides.  For each k the first k topics are moved: 10 and 50
topics (3,539 and 5,443 searched rows) run on the shared-memory path with full evaluation; 100 topics (7,826 rows) are
more than its plan holds at 64 brokers (7,680 rows, make_plan) and, like 400 topics (22,124 rows), run on the HBM path.
Each line reports the median end-to-end time (total_ms) of --calls calls after one warm-up call, the
device time, moves, violation, `optimal`, and the path taken.  The card's name, power limit and max SM clock are read
in the same run.  python tools/time_fixed.py [--calls 3] [--out time_fixed.json]"""
import argparse
import dataclasses
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kafka_assignment_optimizer_b200 as kao  # noqa: E402
from kafka_assignment_optimizer_b200 import optimizer as kopt  # noqa: E402
from kafka_assignment_optimizer_b200.problem import fixed_rows  # noqa: E402

P, B0, R, RF, PER_TOPIC = 65280, 64, 8, 3, 50
OPTS = dict(seed=0x5EED, rounds=3000, round_size=1 << 13, patience=500)
MOVED = (10, 50, 100, 400)
SMEM_ROWS = 7680             # at 64 brokers the shared-memory plan holds this many rows (make_plan, packed entries)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def cluster():
    pb = kao.synthetic_problem(P, B0, R, RF, remove=1)
    pb.topics = [("t%d" % (p // PER_TOPIC), p) for p in range(P)]
    return pb


def timed(pb, calls):
    times, res = [], None
    for call in range(calls + 1):
        res = kopt.solve(pb, **OPTS)
        if call:
            times.append(res.total_ms)
    return statistics.median(times), res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"card": card(), "options": OPTS, "runs": {}}
    pb = cluster()
    current = [[int(pb.broker_ids[b]) if b >= 0 else B0 - 1 for b in row] for row in pb.cur]   # -1: broker 63, removed
    for k in (0,) + MOVED:
        if k == 0:
            name, q, path = "whole cluster (kao_solve)", pb, "HBM (base in HBM, delta evaluation)"
            free = P
        else:
            fx = fixed_rows(current, pb.broker_ids, pb.topics, ["t%d" % t for t in range(k)])
            q = dataclasses.replace(pb, fixed=fx)
            free = int((~fx).sum())
            name = "%d topics moved (kao_solve_fixed)" % k
            path = ("shared memory (full evaluation)" if free <= SMEM_ROWS
                    else "HBM (base in HBM, delta evaluation)")
        ms, res = timed(q, a.calls)
        out["runs"][name] = {"searched_rows": free, "path": path, "total_ms": ms, "device_ms": res.device_ms,
                                 "moves": res.moves, "violation": res.violation, "objective": res.objective,
                                 "optimal": res.optimal, "rounds_run": res.rounds}
        print("%s: %d rows searched, %s: %.1f ms end to end (%.1f ms device), moves %d, violation %d, objective %d, "
              "optimal %s, %d rounds" % (name, free, path, ms, res.device_ms, res.moves, res.violation, res.objective,
                                         res.optimal, res.rounds), flush=True)
    print("card: %s" % out["card"])
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
