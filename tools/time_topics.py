#!/usr/bin/env python
"""Per-topic balance rows (docs/MODEL.md §10, DESIGN.md 7.2) on one GPU, each number with and without topic rows:
  rate    device-timed candidates per second of search_large_kernel (kao_search_delta's CUDA-event time) at
          20,000 x 48 brokers x 8 racks in 400 topics of 50 and at 65,280 x 64 x 8 in 1,306 topics of up to 50
  round   the fixed cost of a round: rounds of two candidates each (two grid barriers, the winner's re-materialisation,
          the patch of the HBM state and, with topic rows, of the topic counts)
  solve   end-to-end kao_solve / kao_solve_topics (total_ms) of the broker-removal recipe of tests/test_gpu_topics.py
Medians of --calls runs after one warm-up call each; the card's name, power limit and max SM clock are printed with the
numbers.  python tools/time_topics.py [--calls 3] [--out time_topics.json]"""
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


def with_topics(P, B0, R, RF, per_topic):
    pb = kao.synthetic_problem(P, B0, R, RF, remove=1)
    pb.topics = [("t%d" % (p // per_topic), p) for p in range(P)]
    return pb, kao.topic_rows(pb)


SHAPES = {"p20000_w2_t400": (20000, 48, 8, 3, 50), "p65280_w2_t1306": (65280, 64, 8, 3, 50)}
BROKER_REMOVAL = ((20000, 48, 8, 3, 50), dict(seed=0x5EED, rounds=3000, round_size=1 << 13, patience=500))


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
    for name, shape in SHAPES.items():
        pb, tr = with_topics(*shape)
        out[name] = {}
        for kind, topics in (("plain", None), ("topics", tr)):
            sess = kao.Session(pb, topics=topics)
            runs, fixed = [], []
            for call in range(a.calls + 1):
                sess.reset()
                _, ms = sess.search_delta(0x5EED, 0, a.rounds, a.round_size)
                if call:
                    runs.append(a.rounds * a.round_size / (ms * 1e-3))
            for call in range(a.calls + 1):
                sess.reset()
                _, ms = sess.search_delta(0x5EED, 0, 512, 2)
                if call:
                    fixed.append(ms * 1e3 / 512)
            sess.close()
            r = out[name][kind] = {"candidates_per_s": statistics.median(runs), "round_fixed_us": statistics.median(fixed)}
            print("%s %s: %.3g candidates/s (%d rounds x %d), fixed cost %.1f us per round"
                  % (name, kind, r["candidates_per_s"], a.rounds, a.round_size, r["round_fixed_us"]), flush=True)
    shape, opts = BROKER_REMOVAL
    pb, tr = with_topics(*shape)
    lower = int((pb.cur < 0).sum())
    out["broker_removal"] = {"lower_bound_moves": lower}
    for kind, extra in (("plain", {}), ("topics", {"topic_balance": True})):
        times, res = [], None
        for call in range(a.calls + 1):
            res = kopt.solve(pb, **opts, **extra)
            if call:
                times.append(res.total_ms)
        out["broker_removal"][kind] = {"total_ms": statistics.median(times), "device_ms": res.device_ms,
                                       "moves": res.moves, "objective": res.objective, "feasible": res.feasible,
                                       "violation": res.violation, "rounds_run": res.rounds}
        print("broker removal 20,000 x 48 in 400 topics (one broker removed), %s: %.1f ms end to end (%.1f ms device), "
              "feasible %s, moves %d (lower bound %d), objective %d, %d rounds"
              % (kind, statistics.median(times), res.device_ms, res.feasible, res.moves, lower, res.objective,
                 res.rounds), flush=True)
    print("card: %s" % out["card"])
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
