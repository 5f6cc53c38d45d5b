#!/usr/bin/env python
"""Per-partition replication rows (docs/MODEL.md §11, DESIGN.md 7.3) on one GPU: 20,000 partitions x 48 brokers x 8
racks in 400 topics of 50, half of the topics at RF 3 and half at RF 2, broker 47 removed, every topic keeping its RF
(build_problem(keep_rf=True)); against the same shape at RF 3 everywhere (a plain session), each with and without
topic rows:
  rate    device-timed candidates per second of the HBM-base search kernel (kao_search_delta's CUDA-event time)
  solve   end-to-end kao_solve* (total_ms), moves against the lower bound (the removed broker's replicas)
Medians of --calls runs after one warm-up call each; the card's name, power limit and max SM clock are printed with the
numbers.  python tools/time_rf.py [--calls 3] [--out time_rf.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import kafka_assignment_optimizer_b200 as kao  # noqa: E402
from kafka_assignment_optimizer_b200 import optimizer as kopt  # noqa: E402

P, B0, R, PER_TOPIC = 20000, 48, 8, 50
SOLVE = dict(seed=0x5EED, rounds=3000, round_size=1 << 13, patience=500)


def document(mixed):
    """(replica lists, topics): round robin over B0 brokers; with `mixed` the odd topics at RF 2"""
    rows, topics = [], []
    for p in range(P):
        t = p // PER_TOPIC
        rf = 2 if mixed and t % 2 else 3
        rows.append([(p + i) % B0 for i in range(rf)])
        topics.append(("t%03d" % t, p % PER_TOPIC))
    return rows, topics


def problem(mixed):
    rows, topics = document(mixed)
    racks = {b: "r%d" % (b % R) for b in range(B0)}
    pb = kao.build_problem(rows, range(B0 - 1), racks, None if mixed else 3, topics, keep_rf=mixed)
    return pb, sum(1 for r in rows if B0 - 1 in r)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=32)
    ap.add_argument("--round-size", type=int, default=1 << 16)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"card": card()}
    for shape, mixed in (("uniform_rf3", False), ("mixed_rf3_rf2", True)):
        pb, lower = problem(mixed)
        out[shape] = {"lower_bound_moves": lower}
        for kind, tr in (("plain", None), ("topics", kao.topic_rows(pb))):
            sess = kao.Session(pb, topics=tr)
            runs = []
            for call in range(a.calls + 1):
                sess.reset()
                _, ms = sess.search_delta(0x5EED, 0, a.rounds, a.round_size)
                if call:
                    runs.append(a.rounds * a.round_size / (ms * 1e-3))
            sess.close()
            times, res = [], None
            for call in range(a.calls + 1):
                res = kopt.solve(pb, **SOLVE, topics=tr)
                if call:
                    times.append(res.total_ms)
            r = out[shape][kind] = {"candidates_per_s": statistics.median(runs), "solve_total_ms": statistics.median(times),
                                    "solve_device_ms": res.device_ms, "feasible": res.feasible, "violation": res.violation,
                                    "moves": res.moves, "objective": res.objective, "rounds_run": res.rounds}
            print("%s %s: %.3g candidates/s (%d rounds x %d); solve %.1f ms end to end (%.1f ms device), feasible %s, "
                  "moves %d (lower bound %d), %d rounds"
                  % (shape, kind, r["candidates_per_s"], a.rounds, a.round_size, r["solve_total_ms"], res.device_ms,
                     res.feasible, res.moves, lower, res.rounds), flush=True)
    print("card: %s" % out["card"])
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
