"""TEST INFRASTRUCTURE — ctypes loader of tests/emu_packed/kao_emu_packed.cpp: the packed MMA epilogue (pop 0x300,
csrc/kao_device_mma.cuh) compiled for the host on top of the tensor-core emulation of tests/emu_mma, with the header's
host restatement of the 16 x 2 SIMD intrinsics.  Never part of the product; nothing outside tests/ imports it."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libkao_emu_packed.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", _HERE])
        _lib = C.CDLL(_SO)
        _lib.kao_emu_mma_create.restype = C.c_void_p
        _lib.kao_emu_last_error.restype = C.c_char_p
    return _lib


class PackedSession:
    """Keys and searches with every key from the packed epilogue.  Raises ValueError on a layout the column-major
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

    def set_base(self, replicas):
        reps = np.ascontiguousarray(replicas, dtype=np.int32)
        lib().kao_emu_mma_set_base(self._h, C.c_void_p(reps.ctypes.data))

    def get_base(self):
        reps = np.empty((self.pb.P, self.pb.RF), np.int32)
        v, o, mv = C.c_int64(), C.c_int64(), C.c_int32()
        lib().kao_emu_mma_get_base(self._h, C.c_void_p(reps.ctypes.data), C.byref(v), C.byref(o), C.byref(mv))
        return reps, v.value, o.value, mv.value

    def candidate_keys(self, seed, rnd, round_size, idx_begin, count):
        out = np.empty(count, np.uint64)
        lib().kao_emu_packed_candidate_keys(self._h, C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size),
                                            C.c_uint32(idx_begin), C.c_uint32(count), C.c_void_p(out.ctypes.data))
        return out

    def search(self, seed, first_round, rounds, round_size):
        keys = np.zeros(rounds, np.uint64)
        lib().kao_emu_packed_search(self._h, C.c_uint64(seed), C.c_uint32(first_round), C.c_uint32(rounds),
                                    C.c_uint32(round_size), C.c_void_p(keys.ctypes.data))
        return keys


def simd(op, a, b, sel=0):
    """The host form of intrinsic `op` ("vmaxu2", "vminu2", "byte_perm") over uint32 arrays a, b."""
    a = np.ascontiguousarray(a, np.uint32)
    b = np.ascontiguousarray(b, np.uint32)
    out = np.empty_like(a)
    lib().kao_emu_simd(C.c_int(["vmaxu2", "vminu2", "byte_perm"].index(op)), C.c_void_p(a.ctypes.data),
                       C.c_void_p(b.ctypes.data), C.c_uint32(sel), C.c_void_p(out.ctypes.data), C.c_int(a.size))
    return out
