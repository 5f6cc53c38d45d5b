"""TEST INFRASTRUCTURE — ctypes loader of tests/emu_sorted/kao_emu_sorted.cpp: the sorted-batch body of the tensor-core
schedules (pop 0x300) restated for the host on top of the tensor-core emulation of tests/emu_mma.  Never part of the
product; nothing outside tests/ imports it."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libkao_emu_sorted.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", _HERE])
        _lib = C.CDLL(_SO)
        _lib.kao_emu_mma_create.restype = C.c_void_p
        _lib.kao_emu_last_error.restype = C.c_char_p
    return _lib


class SortedSession:
    """Keys of a round as the sorted-batch body computes them.  Raises ValueError on a layout the column-major
    evaluator does not cover."""

    def __init__(self, pb):
        from kafka_assignment_optimizer_b200.optimizer import _CProblem

        self.pb = pb
        self._cp = _CProblem(pb)
        self._h = C.c_void_p(lib().kao_emu_mma_create(self._cp.ref()))
        if not self._h:
            raise ValueError(lib().kao_emu_last_error().decode())

    def close(self):
        if self._h:
            lib().kao_emu_mma_destroy(self._h)
            self._h = C.c_void_p()

    def sorted_keys(self, seed, rnd, round_size, idx_lo, idx_hi, grid, warps, cap):
        """Keys of candidates idx_lo .. idx_hi - 1: `grid` CTAs of `warps` warps, a CTA share of more than `cap`
        candidates walked unsorted."""
        out = np.zeros(idx_hi - idx_lo, np.uint64)
        lib().kao_emu_sorted_keys(self._h, C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size), C.c_uint32(idx_lo),
                                  C.c_uint32(idx_hi), C.c_uint32(grid), C.c_uint32(warps), C.c_uint32(cap),
                                  C.c_void_p(out.ctypes.data))
        return out


def cta_batches(seed, rnd, round_size, idx_lo, idx_hi, grid, warps, cap, cta):
    """-> (candidates of CTA `cta` in the order its warps generate them, their classes, batch ends, sorted?)"""
    n = idx_hi - idx_lo
    lst, cls, bounds, nb = np.zeros(n + 1, np.uint32), np.zeros(n + 1, np.uint32), np.zeros(n + 2, np.uint32), C.c_uint32()
    srt = lib().kao_emu_sorted_cta_batches(C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size), C.c_uint32(idx_lo),
                                           C.c_uint32(idx_hi), C.c_uint32(grid), C.c_uint32(warps), C.c_uint32(cap),
                                           C.c_uint32(cta), C.c_void_p(lst.ctypes.data), C.c_void_p(cls.ctypes.data),
                                           C.c_void_p(bounds.ctypes.data), C.byref(nb))
    b = bounds[:nb.value]
    return lst[:b[-1]], cls[:b[-1]], b, bool(srt)
