"""TEST INFRASTRUCTURE — ctypes loader of tests/emu/kao_emu.cpp: the engine's own device functions
(csrc/kao_device.cuh, csrc/kao_device_t.cuh, the tensor-core body of csrc/kao_device_mma.cuh) compiled for the host,
one warp = 32 lock-stepped fibers, and the fixed-partition reduction of csrc/kao_host.hpp.  It lets the CPU suite
exercise the arithmetic of the CUDA path; it is never part of the product (libkao.so has no CPU path) and nothing
outside tests/ imports it."""
import ctypes as C
import dataclasses
import glob
import os

import numpy as np

import native

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_CUDA_INC = os.environ.get("CUDA_INC", "/usr/local/cuda/include")
# the emulator's sources, every header of the engine it may include, and the C ABI
_CSRC = os.path.join(_ROOT, "kafka_assignment_optimizer_b200", "csrc")
_DEPS = (glob.glob(os.path.join(_HERE, "*.[ch]pp")) + glob.glob(os.path.join(_CSRC, "*.cuh")) +
         glob.glob(os.path.join(_CSRC, "*.hpp")) + [os.path.join(_ROOT, "include", "kao.h")])
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(native.shared_library(
            os.path.join(_HERE, "_build"), "libkao_emu.so",
            ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas", "-I" + _CUDA_INC,
             os.path.join(_HERE, "kao_emu.cpp")], _DEPS))
        for fn in ("kao_emu_create", "kao_emu_create_replication", "kao_emu_create_topics", "kao_emu_tc_create",
                   "kao_fx_reduce"):
            getattr(_lib, fn).restype = C.c_void_p
        _lib.kao_emu_last_error.restype = C.c_char_p
        _lib.kao_emu_rows_charged_one_by_one.restype = C.c_longlong
    return _lib


class EmuSession:
    """Same surface as kafka_assignment_optimizer_b200.Session for the calls the parity tests use.  replication: a
    ReplicationRows, opened as kao_create_replication does; topics: a TopicRows, opened as kao_create_topics does.  Both
    are scored as the HBM-base kernels do (delta keys, whole rounds and get_base only)."""

    def __init__(self, pb, replication=None, topics=None):
        from kafka_assignment_optimizer_b200.optimizer import _CProblem, _CReplication, _CTopics

        assert replication is None or topics is None
        self.pb = pb
        self._cp = _CProblem(pb)
        self.large = replication is not None or topics is not None     # the HBM-base kernels' session
        if replication is not None:
            self._cr = _CReplication(replication)
            self._h = C.c_void_p(lib().kao_emu_create_replication(self._cp.ref(), self._cr.ref()))
        elif topics is not None:
            self._ct = _CTopics(topics)
            self._h = C.c_void_p(lib().kao_emu_create_topics(self._cp.ref(), self._ct.ref()))
        else:
            self._h = C.c_void_p(lib().kao_emu_create(self._cp.ref()))
        if not self._h:
            raise ValueError(lib().kao_emu_last_error().decode())

    def close(self):
        if self._h:
            lib().kao_emu_destroy(self._h)
            self._h = C.c_void_p()

    def config(self):
        """Evaluator configuration of the row-major evaluator: EvalCfg<W, NPH, rack, obj> and the dense flag."""
        out = (C.c_int32 * 5)()
        lib().kao_emu_config(self._h, out)
        return dict(W=out[0], NPH=out[1], rack=out[2], obj=out[3], dense=bool(out[4]))

    def set_evaluator(self, mode):
        """0: row-major evaluator; 1: column-major evaluator (csrc/kao_device_t.cuh) as the engine picks it;
        2: its run-time-sized form even where the 32-word specialisation applies; 3: a POPC per word
        (kPop = 0x00); 4: kPop = 0x11; 5: kPop = 0x23 (Harley-Seal on the column totals); 6: kPop = 0x33
        (Harley-Seal on both streams).  False is returned for unsupported layouts."""
        return lib().kao_emu_set_evaluator(self._h, C.c_int32(mode)) == 0

    def set_base(self, replicas):
        reps = np.ascontiguousarray(replicas, dtype=np.int32)
        lib().kao_emu_set_base(self._h, C.c_void_p(reps.ctypes.data))

    def get_base(self):
        reps = np.empty((self.pb.P, self.pb.RF), np.int32)
        v, o, mv = C.c_int64(), C.c_int64(), C.c_int32()
        lib().kao_emu_get_base(self._h, C.c_void_p(reps.ctypes.data), C.byref(v), C.byref(o), C.byref(mv))
        return reps, v.value, o.value, mv.value

    def candidate_keys(self, seed, rnd, round_size, idx_begin, count, delta=False):
        if self.large and not delta:
            raise ValueError("a replication or topic session scores candidates by delta evaluation only")
        out = np.empty(count, np.uint64)
        fn = lib().kao_emu_candidate_keys_delta if delta else lib().kao_emu_candidate_keys
        rc = fn(self._h, C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size), C.c_uint32(idx_begin),
                C.c_uint32(count), C.c_void_p(out.ctypes.data))
        if delta and rc != 0:
            raise ValueError(lib().kao_emu_last_error().decode())
        return out

    def search(self, seed, first_round, rounds, round_size):
        keys = np.zeros(rounds, np.uint64)
        lib().kao_emu_search(self._h, C.c_uint64(seed), C.c_uint32(first_round), C.c_uint32(rounds),
                             C.c_uint32(round_size), C.c_void_p(keys.ctypes.data))
        return keys

    def check_state(self):
        """The state the walk patched (transposed / term planes, one-hot plane, count of invalid leaders, displaced
        lists) against the same state rebuilt from the base (kao_emu_check_state) -> (0, -1, "") or (code, index,
        message)."""
        at = C.c_int64(-1)
        rc = lib().kao_emu_check_state(self._h, C.byref(at))
        return rc, at.value, lib().kao_emu_last_error().decode() if rc else ""

    def evaluate(self, replicas):
        if self.large:
            raise ValueError("kao_eval scores C1 / C7 against one RF and without topic rows")
        reps = np.ascontiguousarray(replicas, dtype=np.int32)
        n = reps.shape[0]
        v, o = np.empty(n, np.int64), np.empty(n, np.int64)
        lib().kao_emu_eval(self._h, C.c_void_p(reps.ctypes.data), C.c_int32(n), C.c_void_p(v.ctypes.data),
                           C.c_void_p(o.ctypes.data))
        return v, o


def dispatch_configs():
    """Every (W, NPH, rack, obj) the engine's dispatch instantiates, as the emulation mirrors it."""
    out = (C.c_int32 * 256)()
    n = lib().kao_emu_dispatch_configs(out, C.c_int32(64))
    return [tuple(out[4 * i:4 * i + 4]) for i in range(n)]


def rows_charged_one_by_one():
    """Rows the column-major evaluator sent through its exact one-by-one path since the last call."""
    return int(lib().kao_emu_rows_charged_one_by_one())


class MmaSession:
    """The calls the parity tests use, with every key from the batched tensor-core body (csrc/kao_device_mma.cuh) of
    pop digit `pop`: 0x300, the default schedule's, with its packed epilogue.  Raises ValueError on any other pop
    digit and on a layout the column-major evaluator does not cover."""

    def __init__(self, pb, pop):
        from kafka_assignment_optimizer_b200.optimizer import _CProblem

        self.pb = pb
        self._cp = _CProblem(pb)
        self._h = C.c_void_p(lib().kao_emu_tc_create(self._cp.ref(), C.c_int32(pop)))
        if not self._h:
            raise ValueError(lib().kao_emu_last_error().decode())

    def close(self):
        if self._h:
            lib().kao_emu_tc_destroy(self._h)
            self._h = C.c_void_p()

    def set_base(self, replicas):
        reps = np.ascontiguousarray(replicas, dtype=np.int32)
        lib().kao_emu_tc_set_base(self._h, C.c_void_p(reps.ctypes.data))

    def get_base(self):
        """Replica lists of the base and its evaluation by the row-major evaluator."""
        reps = np.empty((self.pb.P, self.pb.RF), np.int32)
        v, o, mv = C.c_int64(), C.c_int64(), C.c_int32()
        lib().kao_emu_tc_get_base(self._h, C.c_void_p(reps.ctypes.data), C.byref(v), C.byref(o), C.byref(mv))
        return reps, v.value, o.value, mv.value

    def candidate_keys(self, seed, rnd, round_size, idx_begin, count):
        """Keys of candidates idx_begin .. idx_begin + count - 1, evaluated in batches of 32 in index order."""
        out = np.empty(count, np.uint64)
        lib().kao_emu_tc_candidate_keys(self._h, C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size),
                                        C.c_uint32(idx_begin), C.c_uint32(count), C.c_void_p(out.ctypes.data))
        return out

    def sorted_keys(self, seed, rnd, round_size, idx_lo, idx_hi, grid, warps, cap):
        """Keys of candidates idx_lo .. idx_hi - 1 as the sorted-batch body computes them: `grid` CTAs of `warps`
        warps, a CTA share of more than `cap` candidates walked unsorted."""
        out = np.zeros(idx_hi - idx_lo, np.uint64)
        lib().kao_emu_tc_sorted_keys(self._h, C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size),
                                     C.c_uint32(idx_lo), C.c_uint32(idx_hi), C.c_uint32(grid), C.c_uint32(warps),
                                     C.c_uint32(cap), C.c_void_p(out.ctypes.data))
        return out

    def check_state(self):
        """Patched planes, one-hot plane, count of invalid leaders and displaced lists against the same state rebuilt
        from the base (kao_emu_tc_check_state) -> (0, -1, "") or (code, index, message)."""
        at = C.c_int64(-1)
        rc = lib().kao_emu_tc_check_state(self._h, C.byref(at))
        return rc, at.value, lib().kao_emu_last_error().decode() if rc else ""

    def search(self, seed, first_round, rounds, round_size):
        keys = np.zeros(rounds, np.uint64)
        lib().kao_emu_tc_search(self._h, C.c_uint64(seed), C.c_uint32(first_round), C.c_uint32(rounds),
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


def cta_batches(seed, rnd, round_size, idx_lo, idx_hi, grid, warps, cap, cta):
    """-> (candidates of CTA `cta` in the order its warps generate them, their classes, batch ends, sorted?)"""
    n = idx_hi - idx_lo
    lst, cls, bounds, nb = np.zeros(n + 1, np.uint32), np.zeros(n + 1, np.uint32), np.zeros(n + 2, np.uint32), C.c_uint32()
    srt = lib().kao_emu_cta_batches(C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size), C.c_uint32(idx_lo),
                                    C.c_uint32(idx_hi), C.c_uint32(grid), C.c_uint32(warps), C.c_uint32(cap),
                                    C.c_uint32(cta), C.c_void_p(lst.ctypes.data), C.c_void_p(cls.ctypes.data),
                                    C.c_void_p(bounds.ctypes.data), C.byref(nb))
    b = bounds[:nb.value]
    return lst[:b[-1]], cls[:b[-1]], b, bool(srt)


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
        raise ValueError(lib().kao_emu_last_error().decode())
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
