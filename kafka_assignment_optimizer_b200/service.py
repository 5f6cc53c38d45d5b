"""Minimal HTTP façade (SURVEY.md §8(f)4): POST /submit, JSON in, reassignment JSON out.

The reference only names its hosted endpoint (`/root/reference/README.md:187-194`,
"API endpoint: …/submit"); the request schema is not in the snapshot, so this one is ours:

    POST /submit  {"assignment": {"version":1,"partitions":[...]},      README.md:52-63
                   "brokers": "0,1,2,...",                               README.md:48
                   "racks": "0:a,1:b,...",                               README.md:27-29
                   "rf": 2, "rounds": 256, "round_size": 32768, "restarts": 1, "patience": 0, "delta": false,
                   "gpus": 1, "spread_restarts": false, "certificate": false,
                   "lp_certificate": false, "topic_balance": false, "keep_rf": false, "topic_rf": {}}
    200           {"reassignment": {"version":1,"partitions":[...]},    README.md:67-78
                   "objective": ..., "violation": ..., "moves": ..., "feasible": ...,
                   "objective_bound": ..., "proven_optimal": ...}

`gpus` > 1 shards every round over that many GPUs (or, with `spread_restarts`, runs the restarts side by side);
`certificate` asks for the flow bound, so that `proven_optimal` can say the answer is what lp_solve would return
(README.md:135-136); `lp_certificate` also asks for the Lagrangian LP bound (GPU, docs/MODEL.md §9), which proves
optima the flow bound cannot, e.g. after brokers are removed.  `topic_balance` also spreads every topic over the
brokers (the per-topic rows of docs/MODEL.md §10, default bounds of `topic_rows`).  `keep_rf` keeps every topic's own
replication factor (the length of its longest replica list) and `topic_rf` ({"topic": N}) sets it for the named
topics, the others keeping theirs or taking `rf` when it is given (per-partition rows, docs/MODEL.md §11).

`python -m kafka_assignment_optimizer_b200.service --port 8080` (needs a GPU: there is no CPU path).
"""
from __future__ import annotations

import argparse
import json
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer
from typing import Callable, Optional

from .problem import build_problem, parse_assignment_json, parse_broker_list, parse_rack_map, reassignment_json


MAX_ROUNDS = 1 << 20            # KAO_MAX_ROUNDS
MAX_ROUND_SIZE = 1 << 24        # KAO_MAX_ROUND_SIZE
MAX_CANDIDATES = 1 << 36        # per request: minutes of one GPU, not days


def _bounded(body: dict, name: str, default: int, lo: int, hi: int) -> int:
    v = int(body.get(name, default))
    if not lo <= v <= hi:
        raise ValueError("%s must be %d..%d" % (name, lo, hi))
    return v


def handle_submit(body: dict, solver: Optional[Callable] = None) -> dict:
    """Pure request -> response function (the HTTP layer only moves bytes)."""
    rows, topics = parse_assignment_json(body["assignment"])
    brokers = body["brokers"]
    brokers = parse_broker_list(brokers) if isinstance(brokers, str) else [int(b) for b in brokers]
    racks = body["racks"]
    racks = parse_rack_map(racks) if isinstance(racks, str) else {int(k): str(v) for k, v in racks.items()}
    keep_rf, topic_rf = bool(body.get("keep_rf", False)), body.get("topic_rf") or None
    if keep_rf or topic_rf:
        # per-partition replication factors (docs/MODEL.md §11): the problem carries them to the solver
        rf = int(body["rf"]) if body.get("rf") else None
        topic_rf = {str(k): int(v) for k, v in topic_rf.items()} if topic_rf else None
        pb = build_problem(rows, brokers, racks, rf, topics, keep_rf=keep_rf, topic_rf=topic_rf)
    else:
        rf = int(body.get("rf") or max(len(r) for r in rows))
        pb = build_problem(rows, brokers, racks, rf, topics)
    if solver is None:
        from .optimizer import solve as solver
    # a request cannot ask for an unbounded search: the limits of include/kao.h, checked here as well
    rounds = _bounded(body, "rounds", 256, 0, MAX_ROUNDS)
    round_size = _bounded(body, "round_size", 1 << 15, 2, MAX_ROUND_SIZE)
    restarts = _bounded(body, "restarts", 1, 1, 255)
    patience = _bounded(body, "patience", 0, 0, 65535)
    if rounds * round_size * restarts > MAX_CANDIDATES:
        raise ValueError("rounds * round_size * restarts exceeds %d candidates per request" % MAX_CANDIDATES)
    gpus = _bounded(body, "gpus", 1, 1, 8)                      # KAO_MAX_GPUS
    # only asked for when wanted: a solver without topic rows keeps its signature
    extra = {"topic_balance": True} if body.get("topic_balance") else {}
    res = solver(pb, seed=int(body.get("seed", 0x5EED)) & (2**64 - 1), rounds=rounds, round_size=round_size,
                 restarts=restarts, delta=bool(body.get("delta", False)), patience=patience, n_gpus=gpus,
                 spread_restarts=bool(body.get("spread_restarts", False)), tight_bound=bool(body.get("certificate", False)),
                 lp_bound=bool(body.get("lp_certificate", False)), **extra)
    return {"reassignment": reassignment_json(pb, res.replicas), "objective": int(res.objective),
            "violation": int(res.violation), "moves": int(res.moves), "feasible": bool(res.feasible),
            "objective_bound": int(res.objective_bound), "proven_optimal": bool(res.optimal)}


class _Handler(BaseHTTPRequestHandler):
    solver = None

    def do_POST(self):  # noqa: N802
        if self.path.rstrip("/") != "/submit":
            self.send_error(404)
            return
        try:
            body = json.loads(self.rfile.read(int(self.headers.get("Content-Length", "0"))))
            out, code = handle_submit(body, self.solver), 200
        except (KeyError, ValueError, TypeError) as e:
            out, code = {"error": "bad request: %s" % e}, 400
        except RuntimeError as e:            # KaoError: no GPU, CUDA failure
            out, code = {"error": str(e)}, 503
        data = json.dumps(out).encode()
        self.send_response(code)
        self.send_header("Content-Type", "application/json")
        self.send_header("Content-Length", str(len(data)))
        self.end_headers()
        self.wfile.write(data)

    def log_message(self, fmt, *args):  # quiet
        pass


def make_server(host: str = "127.0.0.1", port: int = 8080, solver: Optional[Callable] = None):
    handler = type("Handler", (_Handler,), {"solver": staticmethod(solver) if solver else None})
    return ThreadingHTTPServer((host, port), handler)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--host", default="127.0.0.1")
    ap.add_argument("--port", type=int, default=8080)
    a = ap.parse_args()
    make_server(a.host, a.port).serve_forever()
