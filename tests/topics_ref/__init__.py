"""TEST INFRASTRUCTURE — the per-topic balance rows (docs/MODEL.md §10) in the test oracles: a ctypes loader of
tests/topics_ref/kao_topics_ref.c (the plain-C restatement of the search with topic rows, built on oracle/kao_ref.c)
and the rows added to oracle.model's evaluation and HiGHS program.  Never part of the product."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import model, ref

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kao_topics_ref.c")
_DEPS = (_SRC, os.path.join(os.path.dirname(os.path.dirname(_HERE)), "oracle", "kao_ref.c"))
_lib = None


def _build():
    out_dir = os.path.join(_HERE, "_build")
    try:
        os.makedirs(out_dir, exist_ok=True)
        if not os.access(out_dir, os.W_OK):
            raise OSError
    except OSError:
        out_dir = tempfile.mkdtemp(prefix="kao_topics_ref_")
    so = os.path.join(out_dir, "libkao_topics_ref.so")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(d) for d in _DEPS):
        subprocess.check_call(["gcc", "-O3", "-fopenmp", "-fPIC", "-std=c11", "-shared", "-o", so, _SRC])
    return so


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_build())
        _lib.kao_tref_search.restype = C.c_uint64
        _lib.kao_tref_topic_violation.restype = C.c_int64
        _lib.kao_ref_pack.restype = C.c_uint64
        _lib.kao_ref_pack.argtypes = [C.c_int64, C.c_int64, C.c_uint32, C.c_int]
    return _lib


class _RefTopics(C.Structure):
    _fields_ = [("T", C.c_int32), ("topic_of", C.c_void_p), ("rep_lo", C.c_void_p), ("rep_hi", C.c_void_p),
                ("ldr_lo", C.c_void_p), ("ldr_hi", C.c_void_p)]


class TRef(ref.Ref):
    """oracle.ref.Ref whose evaluation, candidate keys and search include the topic rows `tr` (a TopicRows)."""

    def __init__(self, pb, tr):
        super().__init__(pb)
        self.tr = tr
        self._tkeep = [np.ascontiguousarray(x, dtype=np.int32) for x in (tr.topic_of, tr.rep_lo, tr.rep_hi, tr.ldr_lo, tr.ldr_hi)]
        self.tc = _RefTopics(len(self._tkeep[1]), *(x.ctypes.data for x in self._tkeep))

    def _t(self):
        return C.byref(self.tc)

    def evaluate(self, bits, ld):
        v, o = C.c_int64(), C.c_int64()
        lib().kao_tref_eval(self._p(), self._t(), C.c_void_p(bits.ctypes.data), C.c_void_p(ld.ctypes.data),
                            C.byref(v), C.byref(o))
        return v.value, o.value

    def topic_violation(self, bits, ld):
        return int(lib().kao_tref_topic_violation(self._p(), self._t(), C.c_void_p(bits.ctypes.data),
                                                  C.c_void_p(ld.ctypes.data)))

    def candidate_keys(self, bits, ld, seed, rnd, round_size, idx_begin, count, nthreads=0):
        out = np.empty(count, np.uint64)
        lib().kao_tref_candidate_keys(self._p(), self._t(), C.c_void_p(bits.ctypes.data), C.c_void_p(ld.ctypes.data),
                                      C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size), C.c_uint32(idx_begin),
                                      C.c_uint32(count), C.c_void_p(out.ctypes.data), C.c_int(nthreads))
        return out

    def search(self, bits, ld, seed, first_round, rounds, round_size, nthreads=0):
        keys = np.zeros(rounds, np.uint64)
        last = lib().kao_tref_search(self._p(), self._t(), C.c_void_p(bits.ctypes.data), C.c_void_p(ld.ctypes.data),
                                     C.c_uint64(seed), C.c_uint32(first_round), C.c_uint32(rounds),
                                     C.c_uint32(round_size), C.c_void_p(keys.ctypes.data), C.c_int(nthreads))
        return last, keys


# ---------------------------------------------------------------------------------- the model with topic rows
def _topic_counts(pb, tr, replicas):
    """[T, B] replicas and leaders (first entry) of each topic per broker (replica lists as model.evaluate reads them)"""
    T = len(tr.rep_lo)
    cnt = np.zeros((T, pb.B), np.int64)
    lcnt = np.zeros((T, pb.B), np.int64)
    for p in range(pb.P):
        row = [int(b) for b in replicas[p] if 0 <= b < pb.B]
        t = int(tr.topic_of[p])
        for b in set(row):
            cnt[t, b] += 1
        if row:
            lcnt[t, row[0]] += 1
    return cnt, lcnt


def topic_violation(pb, tr, replicas):
    """Sum over topics t and brokers b of the amount by which the replicas / the leaders of t's partitions on b miss
    [rep_lo[t], rep_hi[t]] / [ldr_lo[t], ldr_hi[t]]."""
    cnt, lcnt = _topic_counts(pb, tr, replicas)
    band = lambda c, lo, hi: int(np.maximum(c - hi[:, None], 0).sum() + np.maximum(lo[:, None] - c, 0).sum())
    return band(cnt, np.asarray(tr.rep_lo), np.asarray(tr.rep_hi)) + band(lcnt, np.asarray(tr.ldr_lo), np.asarray(tr.ldr_hi))


def violated_rows(pb, tr, replicas):
    """How many of the 2 * T * B topic rows (C3t and C4t of every topic and broker) `replicas` violates."""
    cnt, lcnt = _topic_counts(pb, tr, replicas)
    out = lambda c, lo, hi: int(((c > np.asarray(hi)[:, None]) | (c < np.asarray(lo)[:, None])).sum())
    return out(cnt, tr.rep_lo, tr.rep_hi) + out(lcnt, tr.ldr_lo, tr.ldr_hi)


def evaluate(pb, tr, replicas):
    v, o = model.evaluate(pb, replicas)
    return v + topic_violation(pb, tr, replicas), o


def topic_program_rows(pb, tr):
    """C3t / C4t as extra rows of model.solve_exact over [x (P*B) | l (P*B)], index p*B+b."""
    import scipy.sparse as sp

    T, P, B = len(tr.rep_lo), pb.P, pb.B
    n = P * B
    p = np.repeat(np.arange(P), B)
    b = np.tile(np.arange(B), P)
    row = np.asarray(tr.topic_of, np.int64)[p] * B + b          # (topic, broker) of variable p*B+b
    S = sp.csr_matrix((np.ones(n), (row, np.arange(n))), shape=(T * B, n))
    Z = sp.csr_matrix((T * B, n))
    A = sp.vstack([sp.hstack([S, S]), sp.hstack([Z, S])], format="csr")
    lo = np.concatenate([np.repeat(tr.rep_lo, B), np.repeat(tr.ldr_lo, B)]).astype(np.float64)
    hi = np.concatenate([np.repeat(tr.rep_hi, B), np.repeat(tr.ldr_hi, B)]).astype(np.float64)
    return A, lo, hi


def solve_exact(pb, tr, time_limit=None):
    return model.solve_exact(pb, time_limit=time_limit, extra_rows=topic_program_rows(pb, tr))
