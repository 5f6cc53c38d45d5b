"""kafka_assignment_optimizer_b200/tuning.py lists the schedules of the column-major evaluator that
csrc/kao_kernels.cuh builds; the two lists must stay in step (no GPU needed to check that)."""
import os
import re

from kafka_assignment_optimizer_b200 import tuning


def test_schedule_list_matches_the_kernel_header():
    src = open(os.path.join(os.path.dirname(os.path.abspath(tuning.__file__)), "csrc", "kao_kernels.cuh")).read()
    body = re.search(r"#define KAO_FOR_SCHEDULES\(X\) \\\n(.*)\n", src).group(1)
    built = [(int(a), int(b, 16), int(c)) for a, b, c in re.findall(r"X\((\d+), (0x[0-9a-fA-F]+), (\d+)\)", body)]
    assert built == tuning.SCHEDULES and len(set(built)) == len(built) == 2
    default = (int(re.search(r"#define KAO_SCHEDULE_DEFAULT_SYNC (\d+)", src).group(1)),
               int(re.search(r"#define KAO_SCHEDULE_DEFAULT_POP (0x[0-9a-fA-F]+)", src).group(1), 16),
               int(re.search(r"#define KAO_SCHEDULE_DEFAULT_THREADS (\d+)", src).group(1)))
    assert default == tuning.DEFAULT_SCHEDULE == built[0]
    for sync, pop, threads in built:
        assert sync in (1, 4) and threads in (512, 1024)
        assert pop == 0x300 or (all(0 <= (pop >> (4 * i)) & 15 <= 3 for i in range(2)) and pop >> 8 == 0)


def test_schedule_names_are_unique():
    names = [tuning.schedule_name(s) for s in tuning.SCHEDULES]
    assert len(set(names)) == len(names) and all(n.startswith("column_major sync=") for n in names)
