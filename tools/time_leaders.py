"""Time leader-only rebalancing (kao_solve_leaders, docs/MODEL.md §13) on a whole cluster: 65,280 partitions of RF 3 in
1,306 topics on 64 brokers in 8 racks, replicas drawn at random and every leader on one of 8 brokers (leadership piled
up after restarts).  Four cases: without and with the per-topic rows (C4t, --topic-balance), and the same with 400
topics fixed (--topics-to-move naming the other 906).  Host-side, one thread: no GPU is used.

    python tools/time_leaders.py [--repeat 3]

Prints one line per case: the median wall time of the call over the repeats, the violation before and after, its
fixed part, the leaders changed and the objective."""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import kafka_assignment_optimizer_b200 as kao  # noqa: E402


def cluster(P=65280, B=64, R=8, RF=3, T=1306, hot=8, seed=0):
    rng = np.random.RandomState(seed)
    current = []
    for _ in range(P):
        lead = int(rng.randint(hot))
        current.append([lead] + [int(b) for b in rng.choice(np.delete(np.arange(B), lead), RF - 1, replace=False)])
    topic = np.sort(np.arange(P) % T)                       # 1,306 topics of 49 or 50 partitions
    first = np.searchsorted(topic, np.arange(T))
    topics = [("topic%04d" % t, p - int(first[t])) for p, t in enumerate(topic)]
    return kao.build_problem(current, range(B), {b: "rack%d" % (b % R) for b in range(B)}, RF, topics)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    pb = cluster()
    tr = kao.topic_rows(pb)
    fixed = np.asarray(tr.topic_of) < 400
    lcnt = np.bincount(pb.cur[:, 0], minlength=pb.B)
    print("cluster: %d partitions, %d topics, %d brokers, %d racks; leaders per broker %d..%d (C4 %d..%d)"
          % (pb.P, tr.T, pb.B, pb.R, lcnt.min(), lcnt.max(), pb.ldr_lo[0], pb.ldr_hi[0]))
    for name, fx, tb in (("no topic rows", None, False), ("topic rows", None, True),
                         ("no topic rows, 400 topics fixed", fixed, False), ("topic rows, 400 topics fixed", fixed, True)):
        q = pb if fx is None else kao.Problem(**{**pb.__dict__, "fixed": fx})
        times, res = [], None
        for _ in range(a.repeat):
            t0 = time.perf_counter()
            res = kao.solve_leaders(q, topic_balance=tb)
            times.append(time.perf_counter() - t0)
        before = kao.solve_leaders(kao.Problem(**{**pb.__dict__, "fixed": np.ones(pb.P, bool)}), topic_balance=tb)
        changed = int((res.replicas[:, 0] != pb.cur[:, 0]).sum())
        print("%-34s %8.1f ms  violation %6d -> %6d (fixed part %d)  leaders changed %6d  objective %d"
              % (name, 1e3 * float(np.median(times)), before.violation, res.violation, res.fixed_violation, changed,
                 res.objective))


if __name__ == "__main__":
    main()
