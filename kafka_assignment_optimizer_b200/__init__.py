"""H100-native replacement for the solver step of killerwhile/kafka-assignment-optimizer.

The reference turns (current assignment, target broker list, rack map, RF) into a 0/1 linear
program and hands it to lp_solve (/root/reference/README.md:135-136, model at :139-185).  This
package keeps that JSON-in / JSON-out surface (README.md:52-63 in, :67-78 out) and replaces the
solve with a GPU candidate search behind the C ABI of ``include/kao.h`` (``libkao.so``).

There is no CPU fallback: importing works without a GPU, solving raises ``KaoError``.
"""
from .problem import Problem, ReplicationRows, TopicRows, build_problem, default_bounds, default_weights, synthetic_problem, topic_rows  # noqa: F401
from .optimizer import AssignmentOptimizer, KaoError, Session, SolveResult, key_obj_bits, lp_bound, objective_bound, unpack_key  # noqa: F401

__all__ = ["Problem", "ReplicationRows", "TopicRows", "build_problem", "default_bounds", "default_weights", "synthetic_problem", "topic_rows",
           "AssignmentOptimizer", "KaoError", "Session", "SolveResult", "key_obj_bits", "lp_bound", "objective_bound", "unpack_key"]
