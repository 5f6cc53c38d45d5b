"""TEST INFRASTRUCTURE — the per-partition replication rows (docs/MODEL.md §11) in the test oracles: a ctypes loader of
tests/rf_ref/kao_rf_ref.c (the plain-C restatement of the search with per-partition C1 / C7 rows, built on
oracle/kao_ref.c and tests/topics_ref) and the rows put into oracle.model's evaluation and HiGHS program.  Never part
of the product."""
import ctypes as C
import os

import numpy as np

import native
import topics_ref
from oracle import model, ref

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "kao_rf_ref.c")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_DEPS = (_SRC, os.path.join(_ROOT, "oracle", "kao_ref.c"), os.path.join(_ROOT, "tests", "topics_ref", "kao_topics_ref.c"))
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(native.shared_library(os.path.join(_HERE, "_build"), "libkao_rf_ref.so",
                                            ["gcc", "-O3", "-fopenmp", "-fPIC", "-std=c11", "-shared", _SRC], _DEPS))
        _lib.kao_rref_search.restype = C.c_uint64
    return _lib


class _RefReplication(C.Structure):
    _fields_ = [("rf", C.c_void_p), ("ppr_lo", C.c_void_p), ("ppr_hi", C.c_void_p)]


class RRef(ref.Ref):
    """oracle.ref.Ref whose initial base, evaluation, candidate keys and search use the per-partition rows `rr` (a
    ReplicationRows), and the topic rows `tr` (a TopicRows) when given."""

    def __init__(self, pb, rr, tr=None):
        super().__init__(pb)
        self._rkeep = [np.ascontiguousarray(x, dtype=np.int32) for x in (rr.rf, rr.ppr_lo, rr.ppr_hi)]
        self.rc = _RefReplication(*(x.ctypes.data for x in self._rkeep))
        self.tc = None
        if tr is not None:
            self._tkeep = [np.ascontiguousarray(x, dtype=np.int32) for x in (tr.topic_of, tr.rep_lo, tr.rep_hi, tr.ldr_lo, tr.ldr_hi)]
            self.tc = topics_ref._RefTopics(len(self._tkeep[1]), *(x.ctypes.data for x in self._tkeep))

    def _t(self):
        return None if self.tc is None else C.byref(self.tc)

    def init_base(self):
        bits, ld = self.new_candidate()
        lib().kao_rref_init_base(self._p(), C.byref(self.rc), C.c_void_p(bits.ctypes.data), C.c_void_p(ld.ctypes.data))
        return bits, ld

    def evaluate(self, bits, ld):
        v, o = C.c_int64(), C.c_int64()
        lib().kao_rref_eval(self._p(), self._t(), C.byref(self.rc), C.c_void_p(bits.ctypes.data),
                            C.c_void_p(ld.ctypes.data), C.byref(v), C.byref(o))
        return v.value, o.value

    def candidate_keys(self, bits, ld, seed, rnd, round_size, idx_begin, count, nthreads=0):
        out = np.empty(count, np.uint64)
        lib().kao_rref_candidate_keys(self._p(), self._t(), C.byref(self.rc), C.c_void_p(bits.ctypes.data),
                                      C.c_void_p(ld.ctypes.data), C.c_uint64(seed), C.c_uint32(rnd),
                                      C.c_uint32(round_size), C.c_uint32(idx_begin), C.c_uint32(count),
                                      C.c_void_p(out.ctypes.data), C.c_int(nthreads))
        return out

    def search(self, bits, ld, seed, first_round, rounds, round_size, nthreads=0):
        keys = np.zeros(rounds, np.uint64)
        last = lib().kao_rref_search(self._p(), self._t(), C.byref(self.rc), C.c_void_p(bits.ctypes.data),
                                     C.c_void_p(ld.ctypes.data), C.c_uint64(seed), C.c_uint32(first_round),
                                     C.c_uint32(rounds), C.c_uint32(round_size), C.c_void_p(keys.ctypes.data),
                                     C.c_int(nthreads))
        return last, keys


# ---------------------------------------------------------------------------------- the model with per-partition rows
def _row_terms(pb, replicas, p, n, lo, hi):
    uniq = {int(b) for b in replicas[p] if b >= 0}
    pr = np.bincount([int(pb.rack_of[b]) for b in uniq], minlength=pb.R)
    return abs(len(uniq) - n) + int(np.maximum(pr - hi, 0).sum() + np.maximum(lo - pr, 0).sum())


def evaluate(pb, rr, replicas, tr=None):
    """oracle.model.evaluate with row p's C1 / C7 against rr.rf[p] / rr.ppr_lo[p]..rr.ppr_hi[p] (and the topic rows)."""
    v, o = topics_ref.evaluate(pb, tr, replicas) if tr is not None else model.evaluate(pb, replicas)
    for p in range(pb.P):
        v += _row_terms(pb, replicas, p, int(rr.rf[p]), int(rr.ppr_lo[p]), int(rr.ppr_hi[p])) - \
            _row_terms(pb, replicas, p, pb.RF, pb.ppr_lo, pb.ppr_hi)
    return v, o


def solve_exact(pb, rr, tr=None, time_limit=None):
    """oracle.model.solve_exact with the C1 rows = rf[p] and the C7 rows of partition p = ppr_lo[p]..ppr_hi[p]."""
    import scipy.sparse as sp
    from scipy.optimize import Bounds, LinearConstraint, milp

    A, lo, hi = model._constraints(pb)
    P, R = pb.P, pb.R
    lo[:P] = hi[:P] = np.asarray(rr.rf, np.float64)                          # C1: the first P rows
    lo[-P * R:] = np.repeat(np.asarray(rr.ppr_lo, np.float64), R)            # C7: the last P * R rows, p-major
    hi[-P * R:] = np.repeat(np.asarray(rr.ppr_hi, np.float64), R)
    if tr is not None:
        At, lt, ht = topics_ref.topic_program_rows(pb, tr)
        A, lo, hi = sp.vstack([A, At], format="csr"), np.concatenate([lo, lt]), np.concatenate([hi, ht])
    c = -np.concatenate([pb.wF.reshape(-1), pb.wL.reshape(-1)]).astype(np.float64)
    opts = {"mip_rel_gap": 0.0}
    if time_limit:
        opts["time_limit"] = time_limit
    res = milp(c, constraints=LinearConstraint(A, lo, hi), integrality=np.ones(c.size), bounds=Bounds(0, 1), options=opts)
    if res.status == 0 and res.x is not None:
        reps = model.decode(pb, res.x)
        return model.Solution("optimal", int(round(-res.fun)), reps, model.replica_moves(pb, reps), 0.0, 0.0)
    return model.Solution({2: "infeasible", 1: "limit"}.get(res.status, "other"), None, None, None, 0.0, 0.0)
