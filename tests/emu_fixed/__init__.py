"""TEST INFRASTRUCTURE — ctypes loader of tests/emu_fixed/kao_emu_fixed.cpp: the engine's own fixed-partition reduction
(reduce_fixed, csrc/kao_host.hpp) compiled for the host.  :func:`reduce` returns what kao_solve_fixed searches, as a
tests/fixed_ref.Reduced, so that the emulated sessions of tests/emu can score it."""
import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libkao_emu_fixed.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", _HERE])
        _lib = C.CDLL(_SO)
        _lib.kao_fx_reduce.restype = C.c_void_p
        _lib.kao_fx_last_error.restype = C.c_char_p
    return _lib


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


def reduce(pb, fixed, tr=None, rr=None):
    """-> fixed_ref.Reduced built by reduce_fixed; ValueError with the engine's message when it refuses the input."""
    from fixed_ref import Reduced
    from kafka_assignment_optimizer_b200.optimizer import _CProblem, _CReplication, _CTopics
    from kafka_assignment_optimizer_b200.problem import ReplicationRows, TopicRows

    cp, ct, cr = _CProblem(pb), _CTopics(tr), _CReplication(rr)
    fx = np.ascontiguousarray(fixed, np.uint8)
    h = lib().kao_fx_reduce(cp.ref(), ct.ref(), cr.ref(), _ptr(fx))
    if not h:
        raise ValueError(lib().kao_fx_last_error().decode())
    h = C.c_void_p(h)
    try:
        sizes, consts = np.zeros(2, np.int32), np.zeros(2, np.int64)
        lib().kao_fx_sizes(h, _ptr(sizes), _ptr(consts))
        P, T = int(sizes[0]), int(sizes[1])
        searched = np.zeros(P, np.int32)
        wF, wL = np.zeros((P, pb.B), np.uint16), np.zeros((P, pb.B), np.uint16)
        cur = np.zeros((P, pb.cur.shape[1]), np.int32)
        lib().kao_fx_rows(h, _ptr(searched), _ptr(wF), _ptr(wL), _ptr(cur))
        b = [np.zeros(n, np.int32) for n in (pb.B, pb.B, pb.B, pb.B, pb.R, pb.R)]
        lib().kao_fx_bounds(h, *map(_ptr, b))
        red = dataclasses.replace(pb, P=P, wF=wF, wL=wL, cur=cur, rep_lo=b[0], rep_hi=b[1], ldr_lo=b[2], ldr_hi=b[3],
                                  rack_lo=b[4], rack_hi=b[5], topics=[pb.topics[p] for p in searched] if pb.topics else None)
        for name in ("fixed", "replication"):
            if hasattr(red, name):
                setattr(red, name, None)
        rr2 = tr2 = None
        if rr is not None:
            r = [np.zeros(P, np.int32) for _ in range(3)]
            lib().kao_fx_replication(h, *map(_ptr, r))
            rr2 = ReplicationRows(*r)
        if tr is not None:
            t = [np.zeros(P, np.int32)] + [np.zeros(T, np.int32) for _ in range(4)]
            lib().kao_fx_topics(h, *map(_ptr, t))
            tr2 = TopicRows(*t, names=[None] * T)
        return Reduced(red, tr2, rr2, int(consts[0]), int(consts[1]), searched)
    finally:
        lib().kao_fx_free(h)


def expand(pb, fixed, reduced_replicas, tr=None, rr=None):
    """expand_fixed: [P', RF] of the reduced problem -> [P, RF] of pb."""
    from kafka_assignment_optimizer_b200.optimizer import _CProblem, _CReplication, _CTopics

    cp, ct, cr = _CProblem(pb), _CTopics(tr), _CReplication(rr)
    fx = np.ascontiguousarray(fixed, np.uint8)
    h = C.c_void_p(lib().kao_fx_reduce(cp.ref(), ct.ref(), cr.ref(), _ptr(fx)))
    out = np.zeros((pb.P, pb.RF), np.int32)
    r = np.ascontiguousarray(reduced_replicas, np.int32)
    lib().kao_fx_expand(h, cp.ref(), _ptr(r), _ptr(out))
    lib().kao_fx_free(h)
    return out
