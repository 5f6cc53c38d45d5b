#!/usr/bin/env python
"""The large path (DESIGN.md 7.1, 8,161 .. 65,280 partitions with the base in HBM) on one GPU:
  rate    device-timed candidates per second of search_large_kernel (kao_search_delta's CUDA-event time) at
          65,280 x 64 slots x 8 racks (W 2) and at 20,000 x 3 racks of 20 (W 4)
  round   the fixed cost of a round: rounds of two candidates each, so that the time is the two grid barriers, the
          winner's re-materialisation and the patch of the HBM state
  solve   end-to-end kao_solve (total_ms) of the broker-removal recipe of tests/test_gpu_large.py
Medians of --calls runs after one warm-up call each; the card's name, power limit and max SM clock are printed with the
numbers.  python tools/time_large.py [--calls 3] [--out time_large.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kafka_assignment_optimizer_b200 as kao  # noqa: E402
from kafka_assignment_optimizer_b200 import optimizer as kopt  # noqa: E402
from oracle import model as m  # noqa: E402

SHAPES = {
    "p65280_w2": lambda: m.synthetic_problem(65280, 64, 8, 3, remove=1),
    "p20000_w4": lambda: __import__("conftest").make_problem(20000, [20, 20, 20], 3, seed=41, removed=2),
}
BROKER_REMOVAL = ((20000, 48, 8, 3, 1), dict(seed=0x5EED, rounds=3000, round_size=1 << 13, patience=500))


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
    for name, make in SHAPES.items():
        sess = kao.Session(kao.Problem.from_fields(make()))
        runs, fixed = [], []
        for call in range(a.calls + 1):
            sess.reset()
            keys, ms = sess.search_delta(0x5EED, 0, a.rounds, a.round_size)
            if call:
                runs.append(a.rounds * a.round_size / (ms * 1e-3))
        for call in range(a.calls + 1):
            sess.reset()
            _, ms = sess.search_delta(0x5EED, 0, 512, 2)
            if call:
                fixed.append(ms * 1e3 / 512)
        sess.close()
        out[name] = {"candidates_per_s": statistics.median(runs), "round_fixed_us": statistics.median(fixed),
                     "rounds": a.rounds, "round_size": a.round_size}
        print("%s: %.3g candidates/s (%d rounds x %d), fixed cost %.1f us per round"
              % (name, out[name]["candidates_per_s"], a.rounds, a.round_size, out[name]["round_fixed_us"]), flush=True)
    args, opts = BROKER_REMOVAL
    pb = m.synthetic_problem(*args)
    kp = kao.Problem.from_fields(pb)
    lower = int((pb.cur < 0).sum())
    times, res = [], None
    for call in range(a.calls + 1):
        res = kopt.solve(kp, **opts)
        if call:
            times.append(res.total_ms)
    out["broker_removal"] = {"total_ms": statistics.median(times), "device_ms": res.device_ms, "moves": res.moves,
                             "lower_bound_moves": lower, "objective": res.objective, "objective_bound": res.objective_bound,
                             "feasible": res.feasible, "rounds_run": res.rounds}
    print("broker removal 20,000 x 48 (one removed): %.1f ms end to end (%.1f ms device), feasible %s, moves %d "
          "(lower bound %d), objective %d, bound %d, %d rounds"
          % (out["broker_removal"]["total_ms"], res.device_ms, res.feasible, res.moves, lower, res.objective,
             res.objective_bound, res.rounds))
    print("card: %s" % out["card"])
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
