"""The phase probe (tools/time_phases.py) is a separate build of the search kernels with -DKAO_PHASE_CLOCKS: that
build must keep compiling and export the hook that binds its stamp buffer, and the shipped objects carry none of it
(no GPU needed for either)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kafka_assignment_optimizer_b200", "csrc")


def _symbols(path):
    return subprocess.run(["nm", path], capture_output=True, text=True, check=True).stdout


def test_shipped_objects_carry_no_phase_probe():
    objs = [os.path.join(ROOT, "kafka_assignment_optimizer_b200", "_obj", "kao_inst_trans_%d.o" % w) for w in (1, 2)]
    objs.append(os.path.join(ROOT, "kafka_assignment_optimizer_b200", "libkao.so"))
    objs = [o for o in objs if os.path.exists(o)]
    if not objs or not shutil.which("nm"):
        pytest.skip("in-tree build or nm not available")
    for o in objs:
        assert "kao_phase" not in _symbols(o), o


def test_phase_probe_build_compiles(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc) or not shutil.which("nm"):
        pytest.skip("nvcc or nm not available")
    out = str(tmp_path / "probe_trans_1.o")
    subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-DKAO_PHASE_CLOCKS",
                    "-DKAO_INST_MODE=2", "-DKAO_INST_W=1", "-c", "-o", out, os.path.join(CSRC, "kao_inst.cu")],
                   check=True, capture_output=True)
    assert "T kao_phase_clocks_bind_t1" in _symbols(out)
