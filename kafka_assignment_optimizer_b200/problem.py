"""Host-side model builder: Kafka JSON -> dense integer tables of ``kao_problem``.

Mirrors the reference's L2/L3 layers (SURVEY.md §1): input shapes from
/root/reference/README.md:52-63 (current assignment JSON), :48 (target broker list), :27-29
(broker -> rack/AZ); the tables are the coefficients and right-hand sides of the LP at
README.md:144-185.  What the README leaves open (weights, bound formulas; SURVEY.md §A.3) is a
documented default here and can be overridden by the caller.
"""
from __future__ import annotations

import dataclasses
import json
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

LEADER_WEIGHT_BY_POS = (4, 2, 1)    # README.md:146 shows coefficients {1, 2, 4}; :131-133 leader > follower
FOLLOWER_WEIGHT_BY_POS = (2, 2, 1)


@dataclasses.dataclass
class Problem:
    P: int
    B: int
    R: int
    RF: int
    rack_of: np.ndarray     # uint8  [B]
    wF: np.ndarray          # uint16 [P, B]   README.md:145-146
    wL: np.ndarray          # uint16 [P, B]
    rep_lo: np.ndarray      # int32  [B]      C3 README.md:158-161
    rep_hi: np.ndarray
    ldr_lo: np.ndarray      # int32  [B]      C4 README.md:163-166
    ldr_hi: np.ndarray
    rack_lo: np.ndarray     # int32  [R]      C6 README.md:173-176
    rack_hi: np.ndarray
    ppr_lo: int             #                 C7 README.md:178-180
    ppr_hi: int
    cur: np.ndarray         # int32  [P, RFcur] dense indices, -1 = absent
    broker_ids: np.ndarray  # int32  [B]      dense index -> Kafka broker id
    topics: Optional[list] = None   # per-row (topic, partition)
    replication: Optional["ReplicationRows"] = None   # per-partition C1 / C7 rows (docs/MODEL.md §11), None: RF for all

    @classmethod
    def from_fields(cls, other) -> "Problem":
        """Copy any object exposing the same attributes (e.g. the test oracle's Problem)."""
        return cls(**{f.name: getattr(other, f.name) if f.default is dataclasses.MISSING else getattr(other, f.name, f.default)
                      for f in dataclasses.fields(cls)})


@dataclasses.dataclass
class ReplicationRows:
    """Per-partition replication rows (kao_replication, docs/MODEL.md §11): partition p holds exactly rf[p] replicas,
    and between ppr_lo[p] and ppr_hi[p] of them in every rack.  They replace the problem's C1 (= RF) and C7."""
    rf: np.ndarray          # int32 [P]
    ppr_lo: np.ndarray      # int32 [P]
    ppr_hi: np.ndarray      # int32 [P]


def default_weights(cur: np.ndarray, P: int, B: int) -> Tuple[np.ndarray, np.ndarray]:
    """Existing placements get weight so the optimum keeps them; the preferred (first) replica
    gets more (README.md:116-120, :131-133)."""
    wF = np.zeros((P, B), np.uint16)
    wL = np.zeros((P, B), np.uint16)
    for i in range(cur.shape[1]):
        col = cur[:, i]
        rows = np.flatnonzero(col >= 0)
        wF[rows, col[rows]] = FOLLOWER_WEIGHT_BY_POS[i] if i < 3 else 1
        wL[rows, col[rows]] = LEADER_WEIGHT_BY_POS[i] if i < 3 else 1
    return wF, wL


def default_bounds(P: int, B: int, R: int, RF: int, rack_of: np.ndarray):
    """floor/ceil balance for C3/C4 (README.md:158-166 show <=2,>=1 and <=1,>=0 for 20 replicas on
    19 brokers), rack totals proportional to rack size for C6 (:173-176), floor/ceil of RF/R for
    C7 (:178-180)."""
    tot = P * RF
    size = np.bincount(rack_of, minlength=R).astype(np.int64)
    return (np.full(B, tot // B, np.int32), np.full(B, -(-tot // B), np.int32),
            np.full(B, P // B, np.int32), np.full(B, -(-P // B), np.int32),
            ((tot * size) // B).astype(np.int32), (-((-tot * size) // B)).astype(np.int32),
            RF // R, -(-RF // R))


def partition_rf(current: Sequence[Sequence[int]], topics: Optional[list], rf: Optional[int], keep_rf: bool = False,
                 topic_rf: Optional[Dict[str, int]] = None) -> np.ndarray:
    """The replication factor of every row: with keep_rf (or without `rf`) the length of the longest replica list of its
    topic, else `rf`; then topic_rf[name] for the topics it names (a name the rows do not contain is a ValueError).
    Rows without topics form the one topic "t1"."""
    names = [t[0] if topics else "t1" for t in (topics or [None] * len(current))]
    longest: Dict[str, int] = {}
    for name, reps in zip(names, current):
        longest[name] = max(longest.get(name, 1), len(reps))
    unknown = sorted(set(topic_rf or {}) - set(longest))
    if unknown:
        raise ValueError("topic_rf names topics the assignment does not contain: %s" % ", ".join(unknown))
    out = np.array([longest[n] if keep_rf or rf is None else int(rf) for n in names], np.int32)
    for name, n in (topic_rf or {}).items():
        out[[i for i, t in enumerate(names) if t == name]] = int(n)
    return out


def build_problem(current: Sequence[Sequence[int]], broker_ids: Iterable[int],
                  rack_by_broker: Dict[int, str], rf: Optional[int], topics: Optional[list] = None,
                  keep_rf: bool = False, topic_rf: Optional[Dict[str, int]] = None) -> Problem:
    """keep_rf / topic_rf (partition_rf): every topic keeps its own replication factor, or takes the one named for it.
    When the partitions then differ, RF becomes the largest of them (the width of every replica list), C3 / C6 follow
    from the sum of the per-partition factors and the problem carries per-partition rows (ReplicationRows, C7 = floor /
    ceil of rf[p] / R); when they all agree the problem is the plain one with that RF."""
    if keep_rf or topic_rf:
        rfs = partition_rf(current, topics, rf, keep_rf, topic_rf)
        pb = build_problem(current, broker_ids, rack_by_broker, int(rfs.max()), topics)
        if (rfs == rfs[0]).all():
            return pb
        tot, size = int(rfs.sum()), np.bincount(pb.rack_of, minlength=pb.R).astype(np.int64)
        pb.rep_lo, pb.rep_hi = np.full(pb.B, tot // pb.B, np.int32), np.full(pb.B, -(-tot // pb.B), np.int32)
        pb.rack_lo, pb.rack_hi = ((tot * size) // pb.B).astype(np.int32), (-((-tot * size) // pb.B)).astype(np.int32)
        pb.replication = ReplicationRows(rfs, (rfs // pb.R).astype(np.int32), (-(-rfs // pb.R)).astype(np.int32))
        return pb
    ids = sorted({int(b) for b in broker_ids})          # a repeated id is one broker (as kao-cli's build_model)
    dense = {b: i for i, b in enumerate(ids)}
    racks = sorted({str(rack_by_broker[b]) for b in ids})
    ridx = {r: i for i, r in enumerate(racks)}
    rack_of = np.array([ridx[str(rack_by_broker[b])] for b in ids], np.uint8)
    P, B, R = len(current), len(ids), len(racks)
    rfc = max(1, max(len(c) for c in current))
    cur = np.full((P, rfc), -1, np.int32)
    for p, reps in enumerate(current):
        for i, b in enumerate(reps):
            cur[p, i] = dense.get(int(b), -1)
    wF, wL = default_weights(cur, P, B)
    return Problem(P, B, R, int(rf), rack_of, wF, wL, *default_bounds(P, B, R, int(rf), rack_of), cur,
                   np.array(ids, np.int32), topics)


def synthetic_problem(P: int, B0: int, R: int, RF: int, remove: int = 0, perturb: float = 0.0,
                      seed: int = 0) -> Problem:
    """Benchmark topologies (SURVEY.md §8d): rack_of[b] = b mod R, round-robin current
    assignment, `remove` highest broker ids dropped, optional seeded re-placement of a fraction."""
    rng = np.random.RandomState(seed)
    current = [[(p + i) % B0 for i in range(RF)] for p in range(P)]
    if perturb > 0:
        for _ in range(int(round(perturb * P * RF))):
            p, i, nb = int(rng.randint(P)), int(rng.randint(RF)), int(rng.randint(B0))
            if nb not in current[p]:
                current[p][i] = nb
    return build_problem(current, range(B0 - remove), {b: "r%02d" % (b % R) for b in range(B0)}, RF)


@dataclasses.dataclass
class TopicRows:
    """Per-topic balance rows (kao_topics, docs/MODEL.md §10): for every topic t and broker, the replicas of t's
    partitions there within [rep_lo[t], rep_hi[t]] (C3t) and the partitions of t led from there within
    [ldr_lo[t], ldr_hi[t]] (C4t)."""
    topic_of: np.ndarray    # int32 [P]  topic index of each row
    rep_lo: np.ndarray      # int32 [T]
    rep_hi: np.ndarray
    ldr_lo: np.ndarray      # int32 [T]
    ldr_hi: np.ndarray
    names: list             # [T] topic names

    @property
    def T(self) -> int:
        return len(self.names)


def topic_rows(pb: Problem) -> TopicRows:
    """The default per-topic rows of `pb`: the topics of pb.topics (one topic "t1" for all rows when absent) in order of
    first appearance, bounds floor / ceil of n_t * RF / B for replicas and of n_t / B for leaders (n_t = the topic's
    partitions), the §1 formulas of C3 / C4 per topic.  For the README's one topic they are its rows C3 / C4
    (README.md:158-166)."""
    names, index = [], {}
    topic_of = np.zeros(pb.P, np.int32)
    for p in range(pb.P):
        name = pb.topics[p][0] if pb.topics else "t1"
        if name not in index:
            index[name] = len(names)
            names.append(name)
        topic_of[p] = index[name]
    n = np.bincount(topic_of, minlength=len(names)).astype(np.int64)
    # replicas of each topic: n_t * RF, or the sum of its partitions' factors with per-partition rows
    reps = n * pb.RF if pb.replication is None else \
        np.bincount(topic_of, weights=pb.replication.rf, minlength=len(names)).astype(np.int64)
    return TopicRows(topic_of, (reps // pb.B).astype(np.int32), (-(-reps // pb.B)).astype(np.int32),
                     (n // pb.B).astype(np.int32), (-(-n // pb.B)).astype(np.int32), names)


# ---------------------------------------------------------------------------------- Kafka JSON
def parse_assignment_json(text: str):
    """`kafka-reassign-partitions --generate` "Current partition replica assignment" JSON
    (README.md:52-63).  Returns (rows of replica lists, [(topic, partition)])."""
    doc = json.loads(text) if isinstance(text, str) else text
    parts = sorted(doc["partitions"], key=lambda e: (e["topic"], int(e["partition"])))
    return [list(map(int, e["replicas"])) for e in parts], [(e["topic"], int(e["partition"])) for e in parts]


def parse_broker_list(text: str) -> List[int]:
    """`--broker-list 0,1,...,18` (README.md:48)."""
    return [int(t) for t in str(text).replace(" ", "").split(",") if t != ""]


def parse_rack_map(text: str) -> Dict[int, str]:
    """`id:rack` pairs, comma separated (the wire format is not in the reference snapshot;
    README.md:27-29 only describes the topology), e.g. "0:a,1:b,2:a"."""
    out = {}
    for tok in str(text).replace(" ", "").split(","):
        if tok:
            k, v = tok.split(":", 1)
            out[int(k)] = v
    return out


def reassignment_json(pb: Problem, replicas: np.ndarray) -> dict:
    """`--reassignment-json-file` document (README.md:67-78, :88): same shape as the input,
    leader (preferred replica) first."""
    parts = []
    for p in range(pb.P):
        topic, part = pb.topics[p] if pb.topics else ("t1", p)
        parts.append({"topic": topic, "partition": part,
                      "replicas": [int(pb.broker_ids[b]) for b in replicas[p] if b >= 0]})
    return {"version": 1, "partitions": parts}
