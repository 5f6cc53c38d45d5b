"""TEST INFRASTRUCTURE — ctypes loader of tests/lp_ref/lagrange_ref.c, the plain-C restatement of the Lagrangian
LP bound (docs/MODEL.md §9) that the CUDA kernel is compared with bit for bit.  Never part of the product."""
import ctypes as C
import os

import numpy as np

import native

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "lagrange_ref.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(native.shared_library(os.path.join(_HERE, "_build"), "liblagrange_ref.so",
                                            ["gcc", "-O2", "-std=c11", "-Wall", "-Wextra", "-fPIC", "-shared", _SRC], [_SRC]))
        _lib.lagrange_ref_box.restype = C.c_int64
    return _lib


def fraction_bits():
    return lib().lagrange_ref_fraction_bits()


def box():
    return lib().lagrange_ref_box()


def lp_bound(pb, T, max_iterations):
    """-> (bound, iterations run, multipliers int64[2B + R]) of the integer iteration started from u = 0 with the
    target T (the objective of a feasible assignment)."""
    a = lambda x, dt: np.ascontiguousarray(x, dtype=dt)
    keep = [a(pb.rack_of, np.uint8), a(pb.wF, np.uint16), a(pb.wL, np.uint16), a(pb.rep_lo, np.int32),
            a(pb.rep_hi, np.int32), a(pb.ldr_lo, np.int32), a(pb.ldr_hi, np.int32), a(pb.rack_lo, np.int32),
            a(pb.rack_hi, np.int32)]
    bound, its = C.c_int64(), C.c_uint32()
    mult = np.zeros(2 * pb.B + pb.R, np.int64)
    rc = lib().lagrange_ref(C.c_int(pb.P), C.c_int(pb.B), C.c_int(pb.R), C.c_int(pb.RF),
                            *(C.c_void_p(x.ctypes.data) for x in keep), C.c_int(int(pb.ppr_lo)), C.c_int(int(pb.ppr_hi)),
                            C.c_int64(int(T)), C.c_uint32(max_iterations), C.byref(bound), C.byref(its),
                            C.c_void_p(mult.ctypes.data))
    if rc != 0:
        raise ValueError("a partition has no row that satisfies C1, C2, C5 and C7")
    return bound.value, its.value, mult
