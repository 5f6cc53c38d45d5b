#!/usr/bin/env python
"""Where a launch of the headline search goes, in SM cycles, per phase of the persistent tensor-core kernel:
python tools/time_phases.py [--schedule 1,300,512 ...] [--rounds 32] [--round-size 262144] [--steps 20] [--lib PATH]

It builds libkao with -DKAO_PHASE_CLOCKS into a temporary directory (or loads --lib, a library built that way), so
that the kernel records clock64 stamps per warp and round (csrc/kao_kernels.cuh, KAO_PHASE), runs one warm and one
recorded search on config 3 (1000 x 64 x 8, RF 3) per schedule and prints, separately for free rounds and cycle rounds
(round & 3 == 3, docs/MODEL.md 5), the mean and the median over (CTA, warp, round): generate + park and eval_batch_mma
per batch, and per round the work, the wait at the CTA reduce, the grid barrier, the winner's re-materialisation and
patch, and rebuild_lists; with sorted batches also how long warps 1.. take to sort the next round's candidates, which
they do while warp 0 waits at the grid barrier.  Then the whole launch: the prologue (kernel entry -> round 0's start),
the rounds, the tail (last round -> kernel exit), their sum in milliseconds at the SM clock the stamps ran at, against
the launch's CUDA event time; and a bench.py step (L2 flushed, events around the whole call) against the device_ms the
same call reports, so the work outside the kernel is one number.  The stamps cost cycles themselves: compare the
schedules with each other, and take speed from bench.py.  Prints the card's name, power limit and clocks."""
import argparse
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SLOTS, WARPS, ROUNDS_CAP = 14, 32, 64          # csrc/kao_kernels.cuh: kPhSlots, kPhaseWarps, kPhaseRounds
(GEN, EVAL, BATCHES, START, BATCHES_END, REDUCE, BARRIER, APPLY, REBUILD, LIST,
 ENTRY, EXIT, ENTRY_NS, EXIT_NS) = range(SLOTS)


def build_probe_lib(out_dir):
    csrc = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "csrc")
    lib = os.path.join(out_dir, "libkao.so")
    subprocess.run(["make", "-s", "-j", str(os.cpu_count() or 4), "-C", csrc, lib, "OUT=" + lib,
                    "OBJDIR=" + os.path.join(out_dir, "obj"), "EXTRA=-DKAO_PHASE_CLOCKS"],
                   check=True, stdout=subprocess.DEVNULL)
    return lib


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "nvidia-smi: not available"


def round_rows(r, rounds, kind):
    """[(phase, values)] over the (CTA, warp, round) records of one round kind; CTA-wide phases from warp 0 alone (the
    four sub-partitions' clocks need not agree to a few hundred cycles)."""
    import numpy as np

    sel = np.zeros(rounds, bool)
    sel[[t for t in range(rounds) if (t & 3 == 3) == (kind == "cycle")]] = True
    rr = r[:, :, :rounds, :][:, :, sel, :]
    live = rr[:, :, :, START] != 0
    rec = rr[live]
    nb = np.maximum(rec[:, BATCHES], 1)
    w0 = rr[:, 0, :, :]
    w0 = w0[w0[:, :, START] != 0]
    rows = [
        ("batches per warp and round", rec[:, BATCHES]),
        ("generate + park, per batch", rec[:, GEN] / nb),
        ("eval_batch_mma, per batch", rec[:, EVAL] / nb),
        ("round: start -> warp's last batch done", rec[:, BATCHES_END] - rec[:, START]),
        ("round: warp's wait at the CTA reduce", rec[:, REDUCE] - rec[:, BATCHES_END]),
        ("round: grid barrier (reduce -> all CTAs in)", w0[:, BARRIER] - w0[:, REDUCE]),
        ("round: winner re-materialised and patched", w0[:, APPLY] - w0[:, BARRIER]),
        ("round: rebuild_lists", w0[:, REBUILD] - w0[:, APPLY]),
        ("round: total (start -> rebuild done)", w0[:, REBUILD] - w0[:, START]),
    ]
    lst = rec[:, LIST] != 0                                           # warps 1.. of a sorted-batch schedule
    if lst.any():
        rows.insert(6, ("round: next round sorted, warps 1.. (reduce -> done)", rec[lst, LIST] - rec[lst, REDUCE]))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--schedule", action="append", help="sync,pop(hex),threads; default: the default schedule")
    ap.add_argument("--rounds", type=int, default=32)
    ap.add_argument("--round-size", type=int, default=1 << 18)
    ap.add_argument("--steps", type=int, default=20, help="bench.py-style steps timed per schedule")
    ap.add_argument("--lib", help="a libkao.so built with -DKAO_PHASE_CLOCKS")
    a = ap.parse_args()
    if a.rounds > ROUNDS_CAP:
        sys.exit("at most %d rounds are recorded" % ROUNDS_CAP)
    tmp = None
    if not a.lib:
        tmp = tempfile.TemporaryDirectory(prefix="kao_phase_")
        a.lib = build_probe_lib(tmp.name)
    os.environ["KAO_LIB"] = a.lib
    import ctypes as C

    import numpy as np
    import torch

    import kafka_assignment_optimizer_b200 as kao
    from kafka_assignment_optimizer_b200 import optimizer, tuning

    lib = optimizer.load_library()
    scheds = [tuple(int(x, 16) if i == 1 else int(x) for i, x in enumerate(s.split(","))) for s in a.schedule] if a.schedule \
        else [tuning.DEFAULT_SCHEDULE]
    print("card (name, power limit, max SM clock, SM clock): %s" % card())
    pb = kao.synthetic_problem(1000, 64, 8, 3, 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")     # > 50 MB L2, as bench.py
    for sched in scheds:
        sess = kao.Session(pb, device=0)
        if not sess.set_schedule(*sched):
            print("%s: not built" % tuning.schedule_name(sched))
            continue
        sms = torch.cuda.get_device_properties(0).multi_processor_count      # one CTA per SM
        buf = torch.zeros(sms, WARPS, ROUNDS_CAP, SLOTS, dtype=torch.int64, device="cuda:0")
        assert lib.kao_phase_clocks_bind_t2(C.c_void_p(buf.data_ptr())) == 0     # 64 slots: rows of two words
        sess.search(0x5EED, 0, a.rounds, a.round_size)
        sess.reset()
        buf.zero_()
        flush.fill_(1)
        _, ms = sess.search(0x5EED, 0, a.rounds, a.round_size)
        torch.cuda.synchronize()
        r = buf.cpu().numpy()
        # bench.py's step on the same session: L2 flushed outside the events, events around the whole call
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.steps)]
        dev_ms = []
        for k in range(a.steps):
            flush.fill_(k & 0xFF)
            ev[k][0].record()
            dev_ms.append(sess.search(0x5EED, (k + 1) * a.rounds, a.rounds, a.round_size)[1])
            ev[k][1].record()
        torch.cuda.synchronize()
        step_ms = [x.elapsed_time(y) for x, y in ev]
        sess.close()
        live = r[:, :, :a.rounds, START] != 0                           # (CTA, warp, round) that ran
        ctas = int(live.any(axis=(1, 2)).sum())
        warps = int(live.any(axis=(0, 2)).sum())
        print("%s: %.3f ms for %d rounds x %d candidates, %d CTAs x %d warps" % (
            tuning.schedule_name(sched), ms, a.rounds, a.round_size, ctas, warps))
        free, cyc = round_rows(r, a.rounds, "free"), round_rows(r, a.rounds, "cycle")
        print("  %-54s %10s %10s %10s %10s %7s" % ("SM cycles", "free mean", "median", "cycle mean", "median", "c/f"))
        for (name, fv), (_, cv) in zip(free, cyc):
            fm, cm = float(np.mean(fv)), float(np.mean(cv))
            print("  %-54s %10.0f %10.0f %10.0f %10.0f %7.2f" % (name, fm, float(np.median(fv)), cm, float(np.median(cv)),
                                                               cm / fm if fm else float("nan")))
        # the whole launch, per CTA from warp 0's stamps: prologue + rounds + tail = entry -> exit
        w0 = r[:ctas, 0, :, :]
        last = np.array([int(np.nonzero(w0[c, :a.rounds, START])[0].max()) for c in range(ctas)])
        prologue = w0[:, 0, START] - w0[:, 0, ENTRY]
        rounds_sum = np.array([(w0[c, :last[c] + 1, REBUILD] - w0[c, :last[c] + 1, START]).sum() for c in range(ctas)])
        tail = w0[:, 0, EXIT] - w0[np.arange(ctas), last, REBUILD]
        span = w0[:, 0, EXIT] - w0[:, 0, ENTRY]
        span_ns = w0[:, 0, EXIT_NS] - w0[:, 0, ENTRY_NS]
        mhz = float(np.median(span / np.maximum(span_ns, 1) * 1e3))
        to_ms = lambda cyc_: float(np.mean(cyc_)) / (mhz * 1e3)
        print("  launch (mean over CTAs, warp 0), SM clock from the stamps: %.0f MHz" % mhz)
        for name, v in (("prologue: entry -> round 0's start", prologue), ("rounds: sum of the per-round totals", rounds_sum),
                        ("tail: last rebuild_lists -> exit", tail), ("entry -> exit", span)):
            print("    %-52s %12.0f cycles %8.3f ms" % (name, float(np.mean(v)), to_ms(v)))
        print("    %-52s %12s        %8.3f ms" % ("launch's event time (kao_search device_ms)", "", ms))
        print("  bench.py step (events around the call, L2 flushed) %.3f ms median, device_ms %.3f ms median, "
              "outside device_ms %.3f ms (%d steps)" % (float(np.median(step_ms)), float(np.median(dev_ms)),
                                                       float(np.median(np.array(step_ms) - np.array(dev_ms))), a.steps))
    print("SM cycles; card: %s" % card())


if __name__ == "__main__":
    main()
