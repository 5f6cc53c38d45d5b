#!/usr/bin/env python
"""Time to certificate: how long proving a search result optimal takes on configs 3, 4 and 5' (4096 x 256 x 16,
2 % of the replicas re-placed), per bound.
  lp    kao_lp_bound from the search's assignment: kernel time (torch.profiler, CUDA activities), wall time, bound,
        iterations run
  flow  the host flow bound of kao_objective_bound from the same assignment: wall time and bound
  solve kao_solve without a certificate, with KAO_FLAG_BOUND and with KAO_FLAG_LP_BOUND: total_ms, bound, optimal
Medians of --calls runs; the card's name and power limit are printed with the numbers.
python tools/time_bound.py [--calls 3] [--out time_bound.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import kafka_assignment_optimizer_b200 as kao  # noqa: E402
from kafka_assignment_optimizer_b200 import optimizer as kopt  # noqa: E402
from oracle import model as m  # noqa: E402

# the solve recipes that reach the optima of configs 3 and 4 (INTEGRATION.md 5, tests/test_gpu_configs.py); config 5'
# starts from its stored exact optimum instead (a search does not reach it quickly)
CONFIGS = {
    "cfg3": ((1000, 64, 8, 3, 0), dict(rounds=2000, round_size=1 << 14, patience=100)),
    "cfg4": ((1000, 64, 8, 3, 2), dict(seed=7, rounds=400, round_size=1 << 12, patience=150, restarts=12)),
    "cfg5_p02": ((4096, 256, 16, 3, 0, 0.02, 5), dict(rounds=200, round_size=1 << 15, patience=50)),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def lp_kernel_ms(kp, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        kopt.lp_bound(kp, reps)
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages() if "lagrange_kernel" in e.key) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    torch.cuda.init()
    out = {"card": card(), "configs": {}}
    print("card (name, power limit, max SM clock):", out["card"], flush=True)
    for name, (args, recipe) in CONFIGS.items():
        pb = m.synthetic_problem(*args)
        kp = kao.Problem.from_fields(pb)
        if name == "cfg5_p02":
            reps = np.load(os.path.join(ROOT, "tests", "golden", "cfg5_p02_optimum.npy")).astype(np.int32)
        else:
            reps = kopt.solve(kp, **recipe).replicas
        obj = m.evaluate(pb, reps)[1]
        r = {"objective": obj}
        lp_wall, lp_dev, flow_wall = [], [], []
        for _ in range(a.calls):
            t0 = time.perf_counter()
            bound, its = kopt.lp_bound(kp, reps)
            lp_wall.append((time.perf_counter() - t0) * 1e3)
            lp_dev.append(lp_kernel_ms(kp, reps))
            t0 = time.perf_counter()
            flow = kao.objective_bound(kp, reps)
            flow_wall.append((time.perf_counter() - t0) * 1e3)
        r.update(lp_bound=bound, lp_iterations=its, lp_kernel_ms=statistics.median(lp_dev),
                 lp_wall_ms=statistics.median(lp_wall), flow_bound=flow, flow_wall_ms=statistics.median(flow_wall))
        for flag, kw in (("none", {}), ("flow", dict(tight_bound=True)), ("lp", dict(lp_bound=True))):
            ms, res = [], None
            for _ in range(a.calls):
                res = kopt.solve(kp, **recipe, **kw)
                ms.append(res.total_ms)
            r["solve_" + flag] = dict(total_ms=statistics.median(ms), objective=res.objective,
                                      bound=res.objective_bound, optimal=res.optimal)
        out["configs"][name] = r
        print(name, json.dumps(r), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
