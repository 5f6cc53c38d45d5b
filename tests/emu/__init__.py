"""TEST INFRASTRUCTURE — ctypes loader of tests/emu/kao_emu.cpp: the engine's own device functions
(csrc/kao_device.cuh) compiled for the host, one warp = 32 lock-stepped fibers.  It lets the CPU
suite exercise the arithmetic of the CUDA path; it is never part of the product (libkao.so has no
CPU path) and nothing outside tests/ imports it."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libkao_emu.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", _HERE])
        _lib = C.CDLL(_SO)
        _lib.kao_emu_create.restype = C.c_void_p
        _lib.kao_emu_create_replication.restype = C.c_void_p
        _lib.kao_emu_create_topics.restype = C.c_void_p
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
