"""ctypes binding of ``libkao.so`` (include/kao.h) and the Python mirror of the reference's
operator surface: assignment JSON + broker list + rack map in, reassignment JSON out
(/root/reference/README.md:52-63 -> :67-78).  No CPU path: a missing library or GPU raises."""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
from typing import Optional

import numpy as np

from .problem import (Problem, ReplicationRows, TopicRows, build_problem, parse_assignment_json, parse_broker_list, parse_rack_map,
                      parse_topics_to_move, reassignment_json, topic_rows)

_LIB_PATH = os.environ.get("KAO_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "libkao.so")
KAO_OK, KAO_INFEASIBLE = 0, 1
KEY_NONE = 0x7FFFFFFFFFFFFFFF


class KaoError(RuntimeError):
    pass


class _KaoProblem(C.Structure):
    _fields_ = [("P", C.c_int32), ("B", C.c_int32), ("R", C.c_int32), ("RF", C.c_int32),
                ("RFcur", C.c_int32), ("rack_of", C.c_void_p), ("wF", C.c_void_p), ("wL", C.c_void_p),
                ("rep_lo", C.c_void_p), ("rep_hi", C.c_void_p), ("ldr_lo", C.c_void_p),
                ("ldr_hi", C.c_void_p), ("rack_lo", C.c_void_p), ("rack_hi", C.c_void_p),
                ("ppr_lo", C.c_int32), ("ppr_hi", C.c_int32), ("cur", C.c_void_p)]


class _KaoOptions(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("rounds", C.c_uint32), ("round_size", C.c_uint32),
                ("device", C.c_int32), ("flags", C.c_uint32), ("n_gpus", C.c_int32), ("device_mask", C.c_uint32)]


class _KaoResult(C.Structure):
    _fields_ = [("replicas", C.c_void_p), ("objective", C.c_int64), ("violation", C.c_int64),
                ("moves", C.c_int32), ("feasible", C.c_int32), ("key", C.c_uint64),
                ("n_candidates", C.c_uint64), ("rounds_run", C.c_uint32), ("restarts", C.c_uint32),
                ("device_ms", C.c_double), ("total_ms", C.c_double), ("objective_bound", C.c_int64),
                ("optimal", C.c_int32), ("key_obj_bits", C.c_int32), ("n_gpus", C.c_int32), ("reserved", C.c_int32)]


_lib = None


def load_library():
    """Loads libkao.so from the package directory; if it has not been built yet (fresh checkout) it
    is compiled once with the in-tree Makefile (nvcc, sm_90a).  Raises KaoError when neither works:
    there is no CPU fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH) and not os.environ.get("KAO_LIB"):
            import subprocess

            csrc = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
            r = subprocess.run(["make", "-s", "-j", str(os.cpu_count() or 4), "-C", csrc], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            if r.returncode != 0:
                raise KaoError("libkao.so is not built and building it failed (no CPU fallback):\n" + r.stdout[-2000:])
        if not os.path.exists(_LIB_PATH):
            raise KaoError("libkao.so is not built (%s); there is no CPU fallback" % _LIB_PATH)
        lib = C.CDLL(_LIB_PATH)
        lib.kao_last_error.restype = C.c_char_p
        lib.kao_version.restype = C.c_int
        lib.kao_solve_leaders.restype = C.c_int
        _lib = lib
    return _lib


def _check(rc, allow_infeasible=False):
    if rc == KAO_OK or (allow_infeasible and rc == KAO_INFEASIBLE):
        return rc
    raise KaoError("libkao error %d: %s" % (rc, load_library().kao_last_error().decode()))


def unpack_key(key: int, obj_bits: int):
    """packed key -> (violation, objective, index)  (include/kao.h KAO_KEY_*); obj_bits = key_obj_bits(problem)
    = Session.key_obj_bits = SolveResult.key_obj_bits: the width of the cost field of that problem's keys."""
    key, omax = int(key), (1 << obj_bits) - 1
    return key >> (24 + obj_bits), omax - ((key >> 24) & omax), key & 0xFFFFFF


def key_obj_bits(pb: Problem) -> int:
    """Width of the cost field of this problem's packed keys (kao_key_obj_bits; needs no GPU)."""
    rc = load_library().kao_key_obj_bits(_CProblem(pb).ref())
    if rc < 0:
        _check(rc)
    return rc


def objective_bound(pb: Problem, replicas=None) -> int:
    """Upper bound on the objective of every feasible assignment (kao_objective_bound; needs no GPU): the cheap
    per-partition bound, or — given a feasible assignment [P, RF], leader first — the flow bound Y* + L*."""
    out = C.c_int64()
    r = None if replicas is None else np.ascontiguousarray(replicas, dtype=np.int32)
    rp = None if r is None else C.c_void_p(r.ctypes.data)
    if pb.fixed is not None:    # fixed rows (docs/MODEL.md §12): the bound of the reduced problem plus their objective
        cr, fx = _CReplication(pb.replication), _fixed(pb)
        _check(load_library().kao_objective_bound_fixed(_CProblem(pb).ref(), cr.ref(), C.c_void_p(fx.ctypes.data), rp,
                                                        C.byref(out)))
    elif pb.replication is None:
        _check(load_library().kao_objective_bound(_CProblem(pb).ref(), rp, C.byref(out)))
    else:       # per-partition rows: kao_objective_bound_replication (rf[p] replicas per row)
        cr = _CReplication(pb.replication)
        _check(load_library().kao_objective_bound_replication(_CProblem(pb).ref(), cr.ref(), rp, C.byref(out)))
    return out.value


LP_ITERATIONS = 4096          # KAO_LP_ITERATIONS: the cap kao_solve uses with lp_bound=True
LP_FRACTION_BITS = 20         # KAO_LP_FRACTION_BITS of the multipliers


def lp_bound(pb: Problem, replicas, device: int = 0, max_iterations: int = LP_ITERATIONS, multipliers: bool = False):
    """The Lagrangian LP bound of kao_lp_bound (docs/MODEL.md 9; GPU): an upper bound on the objective of every
    feasible assignment, aimed at the objective of `replicas` (a feasible assignment [P, RF], leader first).  -> (bound,
    iterations run), or (bound, iterations run, multipliers int64[2B + R] with LP_FRACTION_BITS fractional bits)."""
    _refuse_fixed(pb, "lp_bound")
    if pb.replication is not None:
        raise ValueError("lp_bound: the Lagrangian LP bound is built for one RF and one C7 row for every partition "
                         "(docs/MODEL.md 9), not for per-partition replication factors")
    r = np.ascontiguousarray(replicas, dtype=np.int32)
    if r.shape != (pb.P, pb.RF):
        raise ValueError("replicas must be [P, RF]")
    out, its = C.c_int64(), C.c_uint32()
    u = np.zeros(2 * pb.B + pb.R, np.int64)
    _check(load_library().kao_lp_bound(_CProblem(pb).ref(), C.c_void_p(r.ctypes.data), C.c_int32(device),
                                       C.c_uint32(max_iterations), C.byref(out), C.byref(its),
                                       C.c_void_p(u.ctypes.data)))
    return (out.value, its.value, u) if multipliers else (out.value, its.value)


def _fixed(pb: Problem) -> np.ndarray:
    fx = np.ascontiguousarray(pb.fixed, dtype=np.uint8)
    if fx.shape != (pb.P,):
        raise ValueError("fixed must be [P]")
    return fx


def _refuse_fixed(pb: Problem, what: str):
    if pb.fixed is not None:
        raise ValueError("%s: a problem with fixed rows is searched through solve (kao_solve_fixed); the session API and "
                         "kao_eval take the problem they search, e.g. the reduced one (docs/MODEL.md §12)" % what)


class _CProblem:
    """Keeps contiguous numpy buffers alive next to the C struct that points into them."""

    def __init__(self, pb: Problem):
        a = lambda x, dt: np.ascontiguousarray(x, dtype=dt)
        self.keep = [a(pb.rack_of, np.uint8), a(pb.wF, np.uint16), a(pb.wL, np.uint16),
                     a(pb.rep_lo, np.int32), a(pb.rep_hi, np.int32), a(pb.ldr_lo, np.int32),
                     a(pb.ldr_hi, np.int32), a(pb.rack_lo, np.int32), a(pb.rack_hi, np.int32),
                     a(pb.cur, np.int32)]
        k = self.keep
        self.c = _KaoProblem(pb.P, pb.B, pb.R, pb.RF, pb.cur.shape[1],
                             *(x.ctypes.data for x in k[:9]), int(pb.ppr_lo), int(pb.ppr_hi),
                             k[9].ctypes.data)

    def ref(self):
        return C.byref(self.c)


class _KaoTopics(C.Structure):
    _fields_ = [("T", C.c_int32), ("topic_of", C.c_void_p), ("rep_lo", C.c_void_p), ("rep_hi", C.c_void_p),
                ("ldr_lo", C.c_void_p), ("ldr_hi", C.c_void_p)]


class _CTopics:
    """kao_topics over contiguous copies of a TopicRows (None: no topic rows, a NULL pointer)."""

    def __init__(self, tr: Optional[TopicRows]):
        self.c = None
        if tr is not None:
            self.keep = [np.ascontiguousarray(x, dtype=np.int32) for x in
                         (tr.topic_of, tr.rep_lo, tr.rep_hi, tr.ldr_lo, tr.ldr_hi)]
            self.c = _KaoTopics(len(self.keep[1]), *(x.ctypes.data for x in self.keep))

    def ref(self):
        return None if self.c is None else C.byref(self.c)


class _KaoReplication(C.Structure):
    _fields_ = [("rf", C.c_void_p), ("ppr_lo", C.c_void_p), ("ppr_hi", C.c_void_p)]


class _CReplication:
    """kao_replication over contiguous copies of a ReplicationRows (None: no replication rows, a NULL pointer)."""

    def __init__(self, rr: Optional[ReplicationRows]):
        self.c = None
        if rr is not None:
            self.keep = [np.ascontiguousarray(x, dtype=np.int32) for x in (rr.rf, rr.ppr_lo, rr.ppr_hi)]
            self.c = _KaoReplication(*(x.ctypes.data for x in self.keep))

    def ref(self):
        return None if self.c is None else C.byref(self.c)


@dataclasses.dataclass
class SolveResult:
    replicas: np.ndarray      # int32 [P, RF] dense broker indices, leader first
    objective: int
    violation: int
    moves: int
    feasible: bool
    key: int
    n_candidates: int
    rounds: int
    device_ms: float
    total_ms: float
    objective_bound: int = 0  # upper bound on any feasible assignment's objective (kao_result.objective_bound)
    optimal: bool = False     # proven optimal: feasible and objective == objective_bound
    key_obj_bits: int = 24    # cost-field width of `key` (unpack_key)
    n_gpus: int = 1
    fixed_violation: int = 0  # solve_leaders: the part of `violation` the replica sets fix (C1, C3, C5, C6, C7, C3t)


class Session:
    """Device-resident problem (kao_create .. kao_destroy).  topics: per-topic balance rows (a TopicRows, e.g.
    topic_rows(pb)) through kao_create_topics; such a session searches with delta evaluation only.  A problem with
    per-partition rows (pb.replication, build_problem(keep_rf=...)) opens through kao_create_replication, with or
    without topics, and also searches with delta evaluation only."""

    def __init__(self, pb: Problem, device: int = 0, topics: Optional[TopicRows] = None):
        _refuse_fixed(pb, "Session")
        self.pb = pb
        self._cp = _CProblem(pb)
        self._h = C.c_void_p()
        self._lib = load_library()
        if pb.replication is not None:
            self._ct, self._cr = _CTopics(topics), _CReplication(pb.replication)
            _check(self._lib.kao_create_replication(self._cp.ref(), self._ct.ref(), self._cr.ref(), C.c_int32(device),
                                                    C.byref(self._h)))
        elif topics is None:
            _check(self._lib.kao_create(self._cp.ref(), C.c_int32(device), C.byref(self._h)))
        else:
            self._ct = _CTopics(topics)
            _check(self._lib.kao_create_topics(self._cp.ref(), self._ct.ref(), C.c_int32(device), C.byref(self._h)))
        self.key_obj_bits = self._lib.kao_key_obj_bits(self._cp.ref())

    def unpack_key(self, key):
        return unpack_key(key, self.key_obj_bits)

    def close(self):
        if self._h:
            self._lib.kao_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_evaluator(self, column_major: bool) -> bool:
        """Selects the full-evaluation kernel of this session (kao_set_evaluator): column-major (the default
        where the layout allows it) or row-major.  Same keys either way.  Returns False when the layout is
        not covered by the column-major evaluator (the session then stays as it was)."""
        rc = self._lib.kao_set_evaluator(self._h, C.c_int32(1 if column_major else 0))
        if rc == KAO_OK:
            return True
        if column_major and rc == -1:           # KAO_E_ARG: unsupported layout
            return False
        _check(rc)
        return False

    def set_schedule(self, sync: int, pop: int, threads: int) -> bool:
        """Schedule of the column-major evaluator (kao_set_schedule): results never depend on it.
        False when that variant is not built."""
        rc = self._lib.kao_set_schedule(self._h, C.c_int32(sync), C.c_int32(pop), C.c_int32(threads))
        if rc == -1:
            return False
        _check(rc)
        return True

    def set_patience(self, rounds_without_improvement: int):
        _check(self._lib.kao_set_patience(self._h, C.c_uint32(rounds_without_improvement)))

    def last_rounds(self) -> int:
        n = C.c_uint32()
        _check(self._lib.kao_last_rounds(self._h, C.byref(n)))
        return n.value

    def reset(self):
        _check(self._lib.kao_reset(self._h))

    def set_base(self, replicas):
        r = np.ascontiguousarray(replicas, dtype=np.int32)
        assert r.shape == (self.pb.P, self.pb.RF)
        _check(self._lib.kao_set_base(self._h, C.c_void_p(r.ctypes.data)))

    def get_base(self):
        """-> (replicas [P,RF], violation, objective, moves)"""
        r = np.empty((self.pb.P, self.pb.RF), np.int32)
        v, o, mv = C.c_int64(), C.c_int64(), C.c_int32()
        _check(self._lib.kao_get_base(self._h, C.c_void_p(r.ctypes.data), C.byref(v), C.byref(o), C.byref(mv)))
        return r, v.value, o.value, mv.value

    def search(self, seed: int, first_round: int, rounds: int, round_size: int):
        """-> (per-round winning keys uint64[rounds], device milliseconds)"""
        keys = np.zeros(max(rounds, 1), np.uint64)
        ms = C.c_double()
        _check(self._lib.kao_search(self._h, C.c_uint64(seed), C.c_uint32(first_round), C.c_uint32(rounds),
                                    C.c_uint32(round_size), C.c_void_p(keys.ctypes.data), C.byref(ms)))
        return keys[:rounds], ms.value

    def search_delta(self, seed: int, first_round: int, rounds: int, round_size: int):
        """Same search and keys as `search`, candidates scored by delta evaluation (SURVEY 8(f)3)."""
        keys = np.zeros(max(rounds, 1), np.uint64)
        ms = C.c_double()
        _check(self._lib.kao_search_delta(self._h, C.c_uint64(seed), C.c_uint32(first_round), C.c_uint32(rounds),
                                          C.c_uint32(round_size), C.c_void_p(keys.ctypes.data), C.byref(ms)))
        return keys[:rounds], ms.value

    def candidate_keys_delta(self, seed: int, rnd: int, round_size: int, idx_begin: int, count: int):
        keys = np.zeros(max(count, 1), np.uint64)
        _check(self._lib.kao_candidate_keys_delta(self._h, C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size),
                                                  C.c_uint32(idx_begin), C.c_uint32(count),
                                                  C.c_void_p(keys.ctypes.data)))
        return keys[:count]

    def candidate_keys(self, seed: int, rnd: int, round_size: int, idx_begin: int, count: int):
        keys = np.zeros(max(count, 1), np.uint64)
        _check(self._lib.kao_candidate_keys(self._h, C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size),
                                            C.c_uint32(idx_begin), C.c_uint32(count),
                                            C.c_void_p(keys.ctypes.data)))
        return keys[:count]

    def round_launch(self, seed, rnd, round_size, idx_lo, idx_hi, d_key_ptr: int, stream: int = 0):
        _check(self._lib.kao_round_launch(self._h, C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size),
                                          C.c_uint32(idx_lo), C.c_uint32(idx_hi), C.c_void_p(d_key_ptr),
                                          C.c_void_p(stream)))

    def round_apply(self, seed, rnd, round_size, d_key_ptr: int, stream: int = 0):
        _check(self._lib.kao_round_apply(self._h, C.c_uint64(seed), C.c_uint32(rnd), C.c_uint32(round_size),
                                         C.c_void_p(d_key_ptr), C.c_void_p(stream)))

    # ---- sharded search with the per-round reduction inside the kernel (NVLink peer mailboxes)
    def p2p_export(self) -> bytes:
        buf = (C.c_uint8 * 64)()
        _check(self._lib.kao_p2p_export(self._h, buf))
        return bytes(buf)

    def p2p_connect(self, rank: int, world: int, handles):
        """handles: the world's `p2p_export()` blobs in rank order."""
        blob = b"".join(handles)
        assert len(blob) == 64 * world
        arr = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        _check(self._lib.kao_p2p_connect(self._h, C.c_int32(rank), C.c_int32(world), arr))

    def p2p_setup_torch(self, device):
        """Exchange the mailbox handles through torch.distributed (any backend) and connect."""
        import torch
        import torch.distributed as dist

        rank, world = dist.get_rank(), dist.get_world_size()
        mine = torch.tensor(list(self.p2p_export()), dtype=torch.uint8, device=device)
        got = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(got, mine)
        self.p2p_connect(rank, world, [bytes(t.cpu().tolist()) for t in got])

    def search_sharded(self, seed: int, first_round: int, rounds: int, round_size: int, delta: bool = False):
        """Every rank calls this with identical arguments -> (per-round keys, device ms)."""
        keys = np.zeros(max(rounds, 1), np.uint64)
        ms = C.c_double()
        fn = self._lib.kao_search_sharded_delta if delta else self._lib.kao_search_sharded
        _check(fn(self._h, C.c_uint64(seed), C.c_uint32(first_round), C.c_uint32(rounds),
                                            C.c_uint32(round_size), C.c_void_p(keys.ctypes.data), C.byref(ms)))
        return keys[:rounds], ms.value

    def profile_rounds(self, seed, first_round, rounds, round_size):
        """-> (sum of search-kernel ms, sum of apply-kernel ms), CUDA events around every launch"""
        a, b = C.c_double(), C.c_double()
        _check(self._lib.kao_profile_rounds(self._h, C.c_uint64(seed), C.c_uint32(first_round), C.c_uint32(rounds),
                                            C.c_uint32(round_size), C.byref(a), C.byref(b)))
        return a.value, b.value

    def stats(self):
        n, w, s, dn = C.c_uint64(), C.c_int32(), C.c_int32(), C.c_int32()
        _check(self._lib.kao_stats(self._h, C.byref(n), C.byref(w), C.byref(s), C.byref(dn)))
        ev, sy, pop, th = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        _check(self._lib.kao_get_evaluator(self._h, C.byref(ev), C.byref(sy), C.byref(pop), C.byref(th)))
        return {"kernel_launches": n.value, "words_per_row": w.value, "slots": s.value,
                "dense_weights": bool(dn.value), "column_major": ev.value == 1,
                "schedule": (sy.value, pop.value, th.value)}


def solve(pb: Problem, seed: int = 0x5EED, rounds: int = 256, round_size: int = 1 << 15,
          device: int = 0, require_feasible: bool = False, restarts: int = 1, delta: bool = False,
          patience: int = 0, row_major: bool = False, n_gpus: int = 1, device_mask: int = 0,
          tight_bound: bool = False, spread_restarts: bool = False, lp_bound: bool = False,
          topic_balance: bool = False, topics: Optional[TopicRows] = None) -> SolveResult:
    """One blocking kao_solve from host buffers (tables up, winner down).  n_gpus > 1: every round is sharded
    over that many GPUs of this process (devices device .. device+n_gpus-1, or those of device_mask), or with
    spread_restarts the restarts run side by side, one single-GPU search per GPU at a time; either way the
    result is the same as on one GPU with the same arguments.  tight_bound / lp_bound: objective_bound from the flow
    bound (KAO_FLAG_BOUND) / also from the Lagrangian LP bound (KAO_FLAG_LP_BOUND); either can prove optimality.
    topic_balance: every topic spread over the brokers too (kao_solve_topics with `topics`, by default
    topic_rows(pb)); the bounds then leave the topic rows out and may be looser.  A problem with per-partition rows
    (pb.replication) is solved through kao_solve_replication, one with fixed rows (pb.fixed, build_problem(topics_to_move=
    ...)) through kao_solve_fixed: only the other rows are searched, the fixed ones come back as pb.cur lists them, and
    topic_balance then needs every topic fixed or searched whole (docs/MODEL.md §12)."""
    lib = load_library()
    cp = _CProblem(pb)
    if topic_balance and topics is None:
        topics = topic_rows(pb)
    reps = np.full((pb.P, pb.RF), -1, np.int32)
    flags = (max(1, min(255, restarts)) | (0x100 if delta else 0) | (0x200 if row_major else 0) | (0x400 if tight_bound else 0) | (0x800 if spread_restarts else 0) | (0x1000 if lp_bound else 0) |
             (max(0, min(65535, patience)) << 16))
    opt = _KaoOptions(seed & (2 ** 64 - 1), rounds, round_size, device, flags, n_gpus, device_mask)
    res = _KaoResult()
    res.replicas = reps.ctypes.data
    if pb.fixed is not None:
        if topics is not None:          # a topic is moved or kept whole (docs/MODEL.md §12): name the ones that are not
            t_of, fx = np.asarray(topics.topic_of), np.asarray(pb.fixed, bool)
            part = [t for t in range(topics.T) if fx[t_of == t].any() and not fx[t_of == t].all()]
            if part:
                raise ValueError("topic rows with fixed partitions: a topic is moved or kept whole, and these topics are "
                                 "partly fixed (a partition on a leaving broker is searched): %s; add them to the topics "
                                 "to move" % ", ".join(str(topics.names[t]) if topics.names else str(t) for t in part))
        ct, cr, fx = _CTopics(topics), _CReplication(pb.replication), _fixed(pb)
        rc = _check(lib.kao_solve_fixed(cp.ref(), ct.ref(), cr.ref(), C.c_void_p(fx.ctypes.data), C.byref(opt), C.byref(res)),
                    allow_infeasible=not require_feasible)
    elif pb.replication is not None:
        ct, cr = _CTopics(topics), _CReplication(pb.replication)
        rc = _check(lib.kao_solve_replication(cp.ref(), ct.ref(), cr.ref(), C.byref(opt), C.byref(res)),
                    allow_infeasible=not require_feasible)
    elif topics is None:
        rc = _check(lib.kao_solve(cp.ref(), C.byref(opt), C.byref(res)), allow_infeasible=not require_feasible)
    else:
        ct = _CTopics(topics)
        rc = _check(lib.kao_solve_topics(cp.ref(), ct.ref(), C.byref(opt), C.byref(res)),
                    allow_infeasible=not require_feasible)
    return SolveResult(reps, res.objective, res.violation, res.moves, rc == KAO_OK, res.key,
                       res.n_candidates, res.rounds_run, res.device_ms, res.total_ms, res.objective_bound,
                       bool(res.optimal), res.key_obj_bits, res.n_gpus)


def solve_leaders(pb: Problem, topic_balance: bool = False, topics: Optional[TopicRows] = None) -> SolveResult:
    """Leaders only (kao_solve_leaders, docs/MODEL.md §13; host-side, needs no GPU): every partition keeps its replicas
    and the leader is chosen among them, exactly — the least violation of C4 (and, with topic_balance, of the C4t rows
    of `topics`, by default topic_rows(pb)), then the largest objective.  Rows come back leader first, the other replicas
    in their order in pb.cur; pb.fixed keeps those partitions' leaders.  moves is 0, objective_bound the optimum over
    leader-only assignments (not a bound on the full program), and fixed_violation the part of the violation the
    replica sets fix.  Per-partition replication rows (pb.replication) ask for data movement and are refused."""
    if pb.replication is not None:
        raise ValueError("solve_leaders: per-partition replication factors change replica sets; leaders only keeps them "
                         "as they are")
    if topic_balance and topics is None:
        topics = topic_rows(pb)
    reps = np.full((pb.P, pb.RF), -1, np.int32)
    res = _KaoResult()
    res.replicas = reps.ctypes.data
    fv = C.c_int64()
    cp, ct = _CProblem(pb), _CTopics(topics)
    fx = None if pb.fixed is None else _fixed(pb)
    rc = _check(load_library().kao_solve_leaders(cp.ref(), ct.ref(), None if fx is None else C.c_void_p(fx.ctypes.data),
                                                 C.byref(res), C.byref(fv)), allow_infeasible=True)
    return SolveResult(reps, res.objective, res.violation, res.moves, rc == KAO_OK, res.key, res.n_candidates,
                       res.rounds_run, res.device_ms, res.total_ms, res.objective_bound, bool(res.optimal),
                       res.key_obj_bits, res.n_gpus, fv.value)


def evaluate(pb: Problem, replicas, device: int = 0):
    """GPU evaluation of explicit assignments: replicas [n, P, RF] (or [P, RF]) -> (violation[n],
    objective[n]).  Not for a problem with per-partition rows (pb.replication): kao_eval scores C1 / C7 against RF;
    Session(pb).get_base() evaluates such a problem's base."""
    _refuse_fixed(pb, "evaluate")
    if pb.replication is not None:
        raise ValueError("evaluate: kao_eval scores C1 / C7 against one RF; a problem with per-partition replication "
                         "factors is evaluated through a Session (set_base, get_base)")
    lib = load_library()
    cp = _CProblem(pb)
    r = np.ascontiguousarray(replicas, dtype=np.int32)
    if r.ndim == 2:
        r = r[None]
    n = r.shape[0]
    v = np.zeros(n, np.int64)
    o = np.zeros(n, np.int64)
    _check(lib.kao_eval(cp.ref(), C.c_int32(device), C.c_void_p(r.ctypes.data), C.c_int32(n),
                        C.c_void_p(v.ctypes.data), C.c_void_p(o.ctypes.data)))
    return v, o


class AssignmentOptimizer:
    """Operator-level mirror of the reference: feed it what `kafka-reassign-partitions --generate`
    printed plus the target broker list and topology, get the reassignment JSON back."""

    def __init__(self, seed: int = 0x5EED, rounds: int = 256, round_size: int = 1 << 15, device: int = 0, **solve_options):
        """solve_options: anything else `solve` takes (restarts, patience, delta, n_gpus, spread_restarts, tight_bound,
        lp_bound)."""
        self.seed, self.rounds, self.round_size, self.device = seed, rounds, round_size, device
        self.solve_options = solve_options

    def optimize(self, assignment_json, broker_list, rack_map, rf: Optional[int] = None, keep_rf: bool = False,
                 topic_rf: Optional[dict] = None, topics_to_move=None):
        """keep_rf: every topic keeps the length of its longest replica list; topic_rf {name: RF}: those topics take
        that RF, the others keep theirs (keep_rf) or take `rf` (build_problem).  topics_to_move: a list of topic names
        or Kafka's topics-to-move.json document ({"topics": [{"topic": name}], "version": 1}); only those topics and the
        partitions that must leave a broker are searched, and only they are in the returned reassignment."""
        rows, topics = parse_assignment_json(assignment_json)
        brokers = parse_broker_list(broker_list) if isinstance(broker_list, str) else list(broker_list)
        racks = parse_rack_map(rack_map) if isinstance(rack_map, str) else dict(rack_map)
        if rf is None and not (keep_rf or topic_rf):
            rf = max(len(r) for r in rows)
        if topics_to_move is not None:
            topics_to_move = parse_topics_to_move(topics_to_move)
        pb = build_problem(rows, brokers, racks, rf, topics, keep_rf=keep_rf, topic_rf=topic_rf, topics_to_move=topics_to_move)
        res = solve(pb, self.seed, self.rounds, self.round_size, self.device, **self.solve_options)
        return reassignment_json(pb, res.replicas), res
