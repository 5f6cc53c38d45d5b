#!/usr/bin/env python
"""Where a round of the headline search goes, in SM cycles, per phase of the persistent tensor-core kernel:
python tools/time_phases.py [--schedule 1,100,512 ...] [--rounds 32] [--round-size 262144] [--lib PATH]

It builds libkao with -DKAO_PHASE_CLOCKS into a temporary directory (or loads --lib, a library built that way), so
that the kernel records clock64 stamps per warp and round (csrc/kao_kernels.cuh, KAO_PHASE), runs one warm and one
recorded search on config 3 (1000 x 64 x 8, RF 3) per schedule and prints medians over (CTA, warp, round):
generate + park and eval_batch_mma per batch, and per round the work, the wait at the CTA reduce, the grid
barrier, the winner's re-materialisation and patch, and rebuild_lists; with sorted batches also how long warps 1.. take
to sort the next round's candidates, which they do while warp 0 waits at the grid barrier.  The stamps cost cycles themselves: compare
the schedules with each other, and take speed from bench.py.  Prints the card's name, power limit and clocks."""
import argparse
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SLOTS, WARPS, ROUNDS_CAP = 10, 32, 64          # csrc/kao_kernels.cuh: kPhSlots, kPhaseWarps, kPhaseRounds
GEN, EVAL, BATCHES, START, BATCHES_END, REDUCE, BARRIER, APPLY, REBUILD, LIST = range(SLOTS)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--schedule", action="append", help="sync,pop(hex),threads; default: every tensor-core schedule")
    ap.add_argument("--rounds", type=int, default=32)
    ap.add_argument("--round-size", type=int, default=1 << 18)
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
        else [s for s in tuning.SCHEDULES if s[1] >> 8]
    print("card (name, power limit, max SM clock, SM clock): %s" % card())
    pb = kao.synthetic_problem(1000, 64, 8, 3, 0)
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
        _, ms = sess.search(0x5EED, 0, a.rounds, a.round_size)
        torch.cuda.synchronize()
        sess.close()
        r = buf.cpu().numpy()[:, :, :a.rounds, :]
        live = r[:, :, :, START] != 0                                   # (CTA, warp, round) that ran
        ctas = int(live.any(axis=(1, 2)).sum())
        warps = int(live.any(axis=(0, 2)).sum())
        rec = r[live]
        nb = np.maximum(rec[:, BATCHES], 1)
        med = lambda x: float(np.median(x))
        # the CTA's stamps from warp 0 alone: the four sub-partitions' clocks need not agree to a few hundred cycles
        w0 = r[:, 0, :, :]
        ok0 = w0[:, :, START] != 0
        print("%s: %.3f ms for %d rounds x %d candidates, %d CTAs x %d warps" % (
            tuning.schedule_name(sched), ms, a.rounds, a.round_size, ctas, warps))
        rows = [
            ("batches per warp and round", med(rec[:, BATCHES])),
            ("generate + park, per batch", med(rec[:, GEN] / nb)),
            ("eval_batch_mma, per batch", med(rec[:, EVAL] / nb)),
            ("round: start -> warp's last batch done", med(rec[:, BATCHES_END] - rec[:, START])),
            ("round: warp's wait at the CTA reduce", med(rec[:, REDUCE] - rec[:, BATCHES_END])),
            ("round: grid barrier (reduce -> all CTAs in)", med((w0[:, :, BARRIER] - w0[:, :, REDUCE])[ok0])),
            ("round: winner re-materialised and patched", med((w0[:, :, APPLY] - w0[:, :, BARRIER])[ok0])),
            ("round: rebuild_lists", med((w0[:, :, REBUILD] - w0[:, :, APPLY])[ok0])),
            ("round: total (start -> rebuild done)", med((w0[:, :, REBUILD] - w0[:, :, START])[ok0])),
        ]
        lst = rec[:, LIST] != 0                                           # warps 1.. of a sorted-batch schedule
        if lst.any():
            rows.insert(6, ("round: next round sorted, warps 1.. (reduce -> done)", med((rec[lst, LIST] - rec[lst, REDUCE]))))
        for name, v in rows:
            print("  %-46s %10.0f" % (name, v))
    print("SM cycles, medians over (CTA, warp, round); card: %s" % card())


if __name__ == "__main__":
    main()
