/*
 * kao.h — C ABI of the H100-native Kafka assignment-search engine (libkao.so).
 *
 * This is the drop-in boundary for the solver step of killerwhile/kafka-assignment-optimizer:
 * where the reference builds an lp_solve model from (current assignment, broker list, rack map,
 * RF) and reads the 0/1 solution back (/root/reference/README.md:135-136 "lp_solve is used
 * behind the scene", model at README.md:139-185), a caller fills a kao_problem with the same
 * model data as dense integer tables and calls kao_solve().  The reference snapshot contains no
 * source, hence no FFI declarations to cite; every entry point cites the README lines whose
 * behaviour it replaces.  The binding a maintainer adds (JNI / java.lang.foreign / ctypes) is
 * shown in INTEGRATION.md.
 *
 * Conventions: plain C types only; the caller owns every buffer; nothing is retained after a
 * call returns except inside an explicit kao_handle; functions return 0 on success, > 0 for a
 * model-level outcome (KAO_INFEASIBLE), < 0 for argument / CUDA errors, and never throw or exit.
 * kao_last_error() returns a thread-local message for the last non-zero return.
 *
 * Brokers are dense indices 0..B-1 = position in the *target* broker list (README.md:48);
 * mapping Kafka broker ids <-> dense indices is host-side work (JSON codec).
 */
#ifndef KAO_H_
#define KAO_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KAO_VERSION 0x00020000 /* major.minor.patch = 0.2.0 (kao_options / kao_result grew, per-problem key layout) */

/* return codes */
#define KAO_OK 0
#define KAO_INFEASIBLE 1      /* search ended without a candidate satisfying C1..C7 */
#define KAO_E_ARG (-1)        /* bad argument / unsupported problem shape */
#define KAO_E_CUDA (-2)       /* CUDA runtime error (no device, launch failure, OOM) */
#define KAO_E_STATE (-3)      /* handle used in the wrong state */

/* limits of this build */
#define KAO_MAX_SLOTS 256     /* racks * pow2ceil(max(8, largest rack)) must not exceed this */
#define KAO_MAX_RACKS 32
#define KAO_MAX_RF 8
#define KAO_MAX_ROUND_SIZE (1u << 24)
#define KAO_MAX_ROUNDS (1u << 20)  /* rounds of one search call (one cooperative launch per 8192 when sharded) */
#define KAO_MAX_GPUS 8
#define KAO_MAX_PARTITIONS 65280      /* P: the largest multiple of 256 below 2^16 (u16 partition ids) */
#define KAO_MAX_SMEM_PARTITIONS 8160  /* above this many partitions a session keeps its base in HBM (DESIGN.md 7.1) and
                                         searches with delta evaluation only: kao_search, kao_candidate_keys (full
                                         per-candidate evaluation, O(P * W) per candidate), kao_set_evaluator,
                                         kao_set_schedule, KAO_FLAG_ROW_MAJOR, kao_profile_rounds and every sharded
                                         entry point (kao_round_*, kao_p2p_*, kao_search_sharded*, kao_solve with
                                         n_gpus > 1 without KAO_FLAG_SPREAD_RESTARTS) return KAO_E_ARG there */

/*
 * The model, README.md:139-185.  x[b,p] / l[b,p] are the reference's binaries t1b{b}p{p} /
 * t1b{b}p{p}_l (README.md:146, :182-184); an assignment is exchanged as replica lists.
 */
typedef struct kao_problem {
    int32_t P;                /* partitions, 1..KAO_MAX_PARTITIONS (rows; multi-topic input is flattened host-side) */
    int32_t B;                /* brokers in the target list, README.md:48 */
    int32_t R;                /* racks / AZs, README.md:27-29 */
    int32_t RF;               /* target replication factor, C1 README.md:148-151 */
    int32_t RFcur;            /* row length of `cur` */
    const uint8_t *rack_of;   /* [B] rack index of each broker */
    const uint16_t *wF;       /* [P*B] objective weight of a follower replica, README.md:145-146 */
    const uint16_t *wL;       /* [P*B] objective weight of the leader replica, README.md:131-133 */
    const int32_t *rep_lo;    /* [B] C3 min replicas per broker, README.md:158-161 */
    const int32_t *rep_hi;    /* [B] C3 max */
    const int32_t *ldr_lo;    /* [B] C4 min leaders per broker, README.md:163-166 */
    const int32_t *ldr_hi;    /* [B] C4 max */
    const int32_t *rack_lo;   /* [R] C6 min total replicas per rack, README.md:173-176 */
    const int32_t *rack_hi;   /* [R] C6 max */
    int32_t ppr_lo;           /* C7 min replicas of one partition in one rack, README.md:178-180; 0..63: the
                                 evaluators sum four 8-slot racks' deficits in one byte (4 * 63 = 252) */
    int32_t ppr_hi;           /* C7 max, ppr_lo..127 */
    const int32_t *cur;       /* [P*RFcur] current assignment, leader first (README.md:52-63),
                                 dense indices; -1 = padding or a broker not in the target list */
} kao_problem;

typedef struct kao_options {
    uint64_t seed;            /* Philox key of the candidate stream */
    uint32_t rounds;          /* search rounds (<= KAO_MAX_ROUNDS); candidates evaluated = rounds * round_size */
    uint32_t round_size;      /* candidates per round over ALL GPUs of the call, 2 .. KAO_MAX_ROUND_SIZE */
    int32_t device;           /* CUDA device ordinal (the first one when n_gpus > 1 and device_mask == 0) */
    uint32_t flags;           /* bits 0-7: independent restarts (0 or 1 = one search); the best final
                                 assignment of rounds*round_size candidates each is returned.
                                 KAO_FLAG_DELTA: score candidates by delta evaluation (same keys and
                                 trajectory, several times more candidates per second).
                                 KAO_FLAG_PATIENCE(n): early stop; rounds_run / n_candidates report what ran */
    int32_t n_gpus;           /* 0 or 1: one GPU.  N (<= KAO_MAX_GPUS): every round's index range is sharded over N
                                 GPUs of this process (devices device .. device+N-1, or those of device_mask), one
                                 host thread each; the per-round minimum travels through peer-mapped mailboxes inside
                                 the kernels (NVLink).  The result does not depend on N: same round_size, same
                                 trajectory, same assignment. */
    uint32_t device_mask;     /* != 0: bit i selects CUDA device i; n_gpus must then be 0 or its popcount */
} kao_options;

#define KAO_FLAG_DELTA 0x100u
#define KAO_FLAG_ROW_MAJOR 0x200u     /* full evaluation by the row-major evaluator even where the (default, faster)
                                         column-major one applies (see kao_set_evaluator); same keys, same result */
#define KAO_FLAG_BOUND 0x400u         /* kao_result.objective_bound from the flow relaxations of kao_objective_bound (host work
                                         after the search, milliseconds at config 3) instead of the per-partition bound */
#define KAO_FLAG_SPREAD_RESTARTS 0x800u /* n_gpus > 1: run the restarts side by side, restart r on GPU r mod N as an ordinary
                                         single-GPU search (nothing is exchanged between the GPUs), instead of sharding every
                                         round of every restart; same result as one GPU.  The way to use several GPUs for
                                         the recipe that finds optima: many short independent searches (INTEGRATION.md 5) */
#define KAO_FLAG_LP_BOUND 0x1000u     /* feasible result: kao_result.objective_bound becomes the minimum of the bound above and the
                                         Lagrangian LP bound of kao_lp_bound (GPU, at most KAO_LP_ITERATIONS iterations, aimed at
                                         the returned objective) -- the certificate that proves optima the flow bound cannot */
#define KAO_FLAG_PATIENCE(n) ((uint32_t)(n) << 16)  /* stop a search after n (<= 65535) rounds without a better key */

typedef struct kao_result {
    int32_t *replicas;        /* [P*RF] caller-allocated; leader first, then followers by
                                 ascending dense index (README.md:65-78, :88); -1 padded */
    int64_t objective;        /* README.md:145-146 value of the returned assignment */
    int64_t violation;        /* 0 <=> C1..C7 all hold */
    int32_t moves;            /* replicas placed on a broker that did not hold the partition */
    int32_t feasible;
    uint64_t key;             /* packed (violation, cost, index) of the last winning candidate */
    uint64_t n_candidates;    /* candidates generated and fully evaluated */
    uint32_t rounds_run;      /* rounds actually run, summed over restarts */
    uint32_t restarts;        /* restarts performed */
    double device_ms;         /* CUDA-event time of the search kernels (max over the GPUs) */
    double total_ms;          /* wall time of the call incl. host<->device copies */
    int64_t objective_bound;  /* an upper bound on the objective of ANY feasible assignment: per partition the best
                                 leader + best RF-1 followers (C3..C7 ignored), or with KAO_FLAG_BOUND the much
                                 tighter flow bound of kao_objective_bound, and with KAO_FLAG_LP_BOUND at most the
                                 Lagrangian LP bound of kao_lp_bound; lp_solve's optimum (README.md:135-136)
                                 lies between `objective` and this */
    int32_t optimal;          /* 1: feasible and objective == objective_bound, i.e. PROVEN optimal; 0: not proven
                                 (the search is a heuristic: it never claims more than the bound shows) */
    int32_t key_obj_bits;     /* width of the cost field of `key` (KAO_KEY_* macros) */
    int32_t n_gpus;           /* GPUs that took part */
    int32_t reserved;
} kao_result;

int kao_version(void);
const char *kao_last_error(void);

/* One blocking solve from host buffers: tables -> device, `rounds` search rounds, winner -> host.
 * Replaces "emit LP + run lp_solve + parse variables" (README.md:135-136, :139-185).  Above KAO_MAX_SMEM_PARTITIONS
 * partitions KAO_FLAG_DELTA is implied (the result is the assignment, whichever evaluator scored it); the options that
 * path does not offer, and KAO_FLAG_LP_BOUND beyond the LP bound's limits, fail with KAO_E_ARG before any search. */
int kao_solve(const kao_problem *pb, const kao_options *opt, kao_result *res);

/* An upper bound on the objective of every feasible assignment of `pb` — what tells a caller how far a search
 * result can be from the optimum lp_solve would return (README.md:135-136).  Host-side, needs no GPU.
 * replicas == NULL: per partition the best leader + best RF-1 followers, constraints C3..C7 ignored.
 * replicas = a FEASIBLE assignment ([P*RF], leader first): Y* + L*, the optima of two network-flow relaxations
 * (placement under C1/C3/C6/C7, leadership under C2/C4; only their coupling is dropped), found by cancelling
 * negative cycles from that assignment; never above the first bound.  objective == bound proves optimality. */
int kao_objective_bound(const kao_problem *pb, const int32_t *replicas, int64_t *bound);

/* The Lagrangian LP bound (docs/MODEL.md §9): C3, C4 and C6 dualised with multipliers u of KAO_LP_FRACTION_BITS
 * fractional bits; for ANY u, L(u) = sum over those rows of (u > 0 ? u*hi : u*lo) + sum over partitions of the best row
 * under the reduced weights bounds the objective of every feasible assignment from above, and its minimum is the value of
 * the LP relaxation of the whole 0/1 program.  A subgradient iteration in exact integer arithmetic (one cooperative GPU
 * launch) aims at the objective T of `replicas`, a FEASIBLE assignment ([P*RF], leader first), and stops when the bound
 * reaches T (objective == bound proves optimality), when the subgradient or the step vanishes, or after max_iterations
 * (1 .. KAO_MAX_LP_ITERATIONS).  bound = floor(min over the iterations of L / 2^KAO_LP_FRACTION_BITS); iterations_run =
 * evaluations of L; multipliers (optional, [2B + R]: C3 per broker, C4 per broker, C6 per rack) = the u of that
 * minimum.  The result is the same on every GPU and in every run.  KAO_E_ARG for an infeasible or malformed
 * assignment, and beyond the build limits of MODEL §9 (P <= KAO_MAX_SMEM_PARTITIONS, P * RF < 2^16); KAO_E_CUDA
 * without a device (there is no CPU path). */
#define KAO_LP_FRACTION_BITS 20
#define KAO_LP_ITERATIONS 4096              /* the cap kao_solve uses with KAO_FLAG_LP_BOUND */
#define KAO_MAX_LP_ITERATIONS (1u << 20)
int kao_lp_bound(const kao_problem *pb, const int32_t *replicas, int32_t device, uint32_t max_iterations,
                 int64_t *bound, uint32_t *iterations_run, int64_t *multipliers);

/*
 * Per-topic balance rows (docs/MODEL.md §10).  The balance rows of README.md:158-166 sum over ONE topic's
 * partitions; kao_problem flattens every topic into rows, so C3 / C4 bound cluster-wide totals only.  A kao_topics
 * ADDS, for every topic t and broker b:
 *   C3t  rep_lo[t] <= replicas of topic t's partitions on b        <= rep_hi[t]
 *   C4t  ldr_lo[t] <= partitions of topic t led (validly) from b   <= ldr_hi[t]
 * to the violation; every other row, the objective and the candidate stream stay as they are.  Valid input:
 * 1 <= T <= P, 0 <= topic_of[p] < T, 0 <= lo <= hi, rep_lo[t] <= n_t * RF and ldr_lo[t] <= n_t (n_t = partitions of
 * topic t); anything else is KAO_E_ARG before any CUDA call.  The defaults of the Python binding (topic_rows) are
 * floor / ceil of n_t * RF / B and n_t / B.
 */
typedef struct kao_topics {
    int32_t T;                  /* topics */
    const int32_t *topic_of;    /* [P] topic of each partition */
    const int32_t *rep_lo, *rep_hi;   /* [T] C3t */
    const int32_t *ldr_lo, *ldr_hi;   /* [T] C4t */
} kao_topics;

/* kao_solve with the topic rows of `tp` (tp == NULL: exactly kao_solve); see kao_create_topics */
int kao_solve_topics(const kao_problem *pb, const kao_topics *tp, const kao_options *opt, kao_result *res);

/* Evaluate n explicit assignments (each [P*RF] replica lists, leader first, -1 padded) on the
 * GPU with the same evaluator the search uses: C1..C7 violation amount and objective.  (Above
 * KAO_MAX_SMEM_PARTITIONS partitions: one CTA per assignment, per-row terms and per-slot totals.) */
int kao_eval(const kao_problem *pb, int32_t device, const int32_t *replicas, int32_t n,
             int64_t *violation, int64_t *objective);

/* ---- device-resident session: tables stay in HBM between calls (multi-round, multi-GPU) ---- */
typedef struct kao_handle kao_handle;

int kao_create(const kao_problem *pb, int32_t device, kao_handle **out);
/* kao_create with the topic rows of `tp` (tp == NULL: exactly kao_create).  A topic session keeps its base in HBM at
 * every P (DESIGN.md 7.2) and searches by delta evaluation (KAO_FLAG_DELTA implied); what a session above
 * KAO_MAX_SMEM_PARTITIONS refuses, it refuses at any P (KAO_E_ARG).  kao_search_delta, kao_candidate_keys_delta,
 * kao_set_base, kao_get_base (the violation includes the topic rows), patience, restarts and KAO_FLAG_SPREAD_RESTARTS
 * work as on any session.  KAO_FLAG_BOUND / KAO_FLAG_LP_BOUND bound the problem WITHOUT the topic rows: still an upper
 * bound (the topic rows only remove assignments), possibly a looser one; optimal = 1 still means proven.  Device
 * memory: 4 bytes per (topic, slot) for the counts (67 MB at 65,280 topics x 256 slots). */
int kao_create_topics(const kao_problem *pb, const kao_topics *tp, int32_t device, kao_handle **out);

/*
 * Per-partition replication rows (docs/MODEL.md §11).  kao_problem gives every partition the same C1 (= RF) and C7
 * (ppr_lo .. ppr_hi per rack); a cluster that mixes RF-3 and RF-2 topics then either raises or lowers a replica count
 * of every partition of one kind.  A kao_replication REPLACES those two rows, partition by partition:
 *   C1  sum over brokers of (replica + leader) of p          = rf[p]
 *   C7  ppr_lo[p] <= sum over the brokers of a rack r of it  <= ppr_hi[p]
 * pb->RF stays the width of every replica list ([P*RF], -1 padded) and must be >= every rf[p]; pb->ppr_lo / ppr_hi are
 * still validated but not used.  The initial base (MODEL §4) keeps or completes each row to rf[p].  Every other row,
 * the objective, the candidate stream and the key layout stay as they are.  Valid input: 1 <= rf[p] <= min(RF, B - 1),
 * 0 <= ppr_lo[p] <= 63, ppr_lo[p] <= ppr_hi[p] <= 127 (as for pb->ppr_lo / ppr_hi: the evaluators sum the C7 deficits
 * of four 8-slot racks in one byte, exact up to 4 * 63), and with topic rows, rep_lo[t] <= the sum of rf over topic t;
 * anything else is KAO_E_ARG before any CUDA call.  The defaults of the Python binding are ppr = floor / ceil of
 * rf[p] / R.
 */
typedef struct kao_replication {
    const int32_t *rf;                  /* [P] exactly rf[p] replicas */
    const int32_t *ppr_lo, *ppr_hi;     /* [P] C7 of partition p, per rack */
} kao_replication;

/* kao_create_topics with the replication rows of `rp` (rp == NULL: exactly kao_create_topics, tp may be NULL).  A
 * session with `rp` keeps its base in HBM at every P and searches by delta evaluation, as a topic session does, and
 * refuses what that session refuses (KAO_E_ARG).  kao_get_base returns rows of up to RF entries, -1 padded. */
int kao_create_replication(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp, int32_t device,
                           kao_handle **out);
/* kao_solve_topics with the replication rows of `rp` (rp == NULL: exactly kao_solve_topics).  KAO_FLAG_BOUND and the
 * default bound are the bounds of kao_objective_bound_replication; KAO_FLAG_LP_BOUND with `rp` is KAO_E_ARG. */
int kao_solve_replication(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp,
                          const kao_options *opt, kao_result *res);
/* kao_objective_bound with the replication rows of `rp` (rp == NULL: exactly kao_objective_bound): the cheap bound
 * takes the best leader plus the best rf[p] - 1 followers; the flow bound has supply rf[p] at partition p and C7 arcs
 * ppr_lo[p] .. ppr_hi[p].  replicas: a FEASIBLE assignment under those rows, [P*RF], leader first, -1 padded. */
int kao_objective_bound_replication(const kao_problem *pb, const kao_replication *rp, const int32_t *replicas,
                                    int64_t *bound);

/*
 * Fixed partitions (docs/MODEL.md §12): "move these topics and leave everything else where it is".  fixed[p] = 1 keeps
 * partition p exactly as cur[p] lists it (its non-negative entries in their order, the first one leading); its C1,
 * C2/C5, C7 and per-partition replication rows leave the program, while its replicas still count in C3, C6 and C3t and
 * its leader in C4 and C4t.  The call reduces the problem once on the host, to the searched rows with those loads moved
 * into the bounds (band(c + f, lo, hi) = band(c, max(lo - f, 0), max(hi - f, 0)) + max(f - hi, 0)), and runs
 * kao_solve_replication on it: the path, the options it accepts and its refusals (KAO_FLAG_ROW_MAJOR, sharding and
 * KAO_FLAG_LP_BOUND above KAO_MAX_SMEM_PARTITIONS) follow from the REDUCED problem's size and rows.  A plain reduced
 * problem of at most KAO_MAX_SMEM_PARTITIONS rows whose tables do not fit the shared memory of an SM (e.g. above 7,680
 * rows at 33..64 broker slots) runs on the HBM path with uniform replication rows instead of being refused; there
 * KAO_FLAG_ROW_MAJOR and sharding are KAO_E_ARG and KAO_FLAG_LP_BOUND is computed on the plain reduced problem.  Fixed topics drop
 * out of the topic rows and the others are renumbered.
 * Result: fixed rows come back as cur lists them (-1 padded to RF); violation = V' + V0 and objective = O' + O0, where
 * V0 is what the fixed load alone exceeds (C3, C4, C6 and the cells of fixed topics) and O0 the fixed rows' objective;
 * objective_bound = bound' + O0 (every bound); moves counts the searched rows; feasible = (violation == 0), so the call
 * returns KAO_INFEASIBLE when V0 > 0 whatever the search found; optimal keeps its meaning.  key and key_obj_bits are
 * those of the reduced search.
 * KAO_E_ARG before any CUDA call, besides what kao_solve_replication refuses: a fixed row that is empty, that names a
 * broker after a -1 (a replica outside the target list cannot be kept), that names one broker twice or more than RF;
 * with topic rows a topic that is partly fixed; every partition fixed.  fixed == NULL: exactly kao_solve_replication.
 * The session API (kao_create*) and kao_eval take no mask: their callers build the problem they search.
 */
int kao_solve_fixed(const kao_problem *pb, const kao_topics *tp, const kao_replication *rp, const uint8_t *fixed,
                    const kao_options *opt, kao_result *res);
/* kao_objective_bound_replication of the reduced problem of kao_solve_fixed, plus O0: an upper bound on the objective
 * of every feasible assignment that keeps the fixed rows.  Host-side, needs no GPU.  replicas == NULL: the cheap bound;
 * else a [P*RF] assignment whose searched rows are feasible in the reduced problem (its fixed rows are not read): the
 * flow bound.  fixed == NULL: exactly kao_objective_bound_replication. */
int kao_objective_bound_fixed(const kao_problem *pb, const kao_replication *rp, const uint8_t *fixed,
                              const int32_t *replicas, int64_t *bound);

/*
 * Leaders only (docs/MODEL.md §13): "spread leadership, move no data".  Every partition keeps the replica set cur[p]
 * lists; the call chooses each one's leader among those replicas, exactly.  C1, C3, C5, C6, C7 and the C3t rows of `tp`
 * are then constants (their violation is *fixed_violation); C2 holds by construction; the free rows are C4 and the C4t
 * rows of `tp` (tp == NULL: none).  The result is the lexicographic optimum: the least violation of the free rows, then
 * the largest objective (README.md:145-146) among the choices with that violation.  fixed[p] = 1 (fixed == NULL: none)
 * keeps partition p's current leader, which still counts in C4 and C4t.  Host-side, needs no GPU; the same input gives
 * the same lists.
 * Result: res->replicas[P*RF] = per row the chosen leader, then the row's other replicas in their order in cur, -1
 * padded (a row whose leader stays comes back exactly as cur lists it); violation = the whole violation of that
 * assignment as kao_eval scores it (plus the topic rows of `tp`); moves, n_candidates, rounds_run, restarts, key and
 * device_ms = 0; objective_bound = objective, the optimum over LEADER-ONLY assignments of these replica sets, not a
 * bound on the full program (kao_solve*'s reassignments may do better); optimal = feasible = (violation == 0);
 * KAO_INFEASIBLE when violation > 0, with the result filled.
 * KAO_E_ARG before anything else, naming the partition or broker: what kao_create refuses in pb; a row with an entry
 * after a -1 (a replica on a broker outside the target list, whose data would have to move) or naming a broker not in
 * 0..B-1; a row naming one broker twice; an empty row; a row of more than RF replicas; topic rows kao_create_topics
 * refuses.  A trailing -1 is padding: that row is shorter, and C1 counts what it lacks.
 */
int kao_solve_leaders(const kao_problem *pb, const kao_topics *tp, const uint8_t *fixed, kao_result *res,
                      int64_t *fixed_violation);

int kao_destroy(kao_handle *h);
/* base <- current assignment restricted to the target brokers and completed to RF (MODEL §4) */
int kao_reset(kao_handle *h);
int kao_set_base(kao_handle *h, const int32_t *replicas);
int kao_get_base(kao_handle *h, int32_t *replicas, int64_t *violation, int64_t *objective,
                 int32_t *moves);

/* rounds first_round .. first_round+rounds-1 on this GPU alone; round_keys (optional, host,
 * [rounds]) receives each round's winning key; device_ms (optional) the CUDA-event time. */
int kao_search(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
               uint32_t round_size, uint64_t *round_keys, double *device_ms);

/* SURVEY.md 8(f)3 — the same search with DELTA evaluation: every candidate's key is derived from
 * the base's totals and its <= 3 patched rows (one thread per candidate) instead of a full pass
 * over its bit-plane.  Keys, winners and trajectory are bit-identical to kao_search; throughput
 * is reported separately (it is not the "full evaluation per candidate" metric).  Every row width; the only
 * search above KAO_MAX_SMEM_PARTITIONS partitions (base in HBM, DESIGN.md 7.1). */
int kao_search_delta(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                     uint32_t round_size, uint64_t *round_keys, double *device_ms);
int kao_candidate_keys_delta(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                             uint32_t idx_begin, uint32_t count, uint64_t *keys);

/* early stop for every later search on this handle: leave after `n` rounds without a better
 * (violation, objective); 0 = run all rounds.  The decision depends only on the round keys, so all
 * ranks of a sharded search stop together.  kao_last_rounds: rounds the last search actually ran. */
int kao_set_patience(kao_handle *h, uint32_t rounds_without_improvement);

/* Full-evaluation kernel used by kao_search / kao_search_sharded / kao_candidate_keys of this session.
 * Both evaluate every row and column of every candidate (C1..C7 + objective, README.md:144-185) and
 * return bit-identical keys; they differ in how the base is laid out in shared memory:
 *   KAO_EVAL_COLUMN_MAJOR  also one bitmap over the partitions per broker slot (replicas, leader one-hot) and the
 *                          objective as term planes over the partitions; needs rows of up to 64 slots, racks of up
 *                          to 8 brokers, C7 = at most one replica per rack, wL >= wF with the non-zero terms of the
 *                          objective row (README.md:145-146) fitting 8 term planes (docs/MODEL.md 3.2), and the planes fitting the
 *                          shared memory of an SM (e.g. 2,000 partitions x 64 slots, 8,160 x 32);
 *                          the DEFAULT wherever it applies; KAO_E_ARG when requested elsewhere
 *   KAO_EVAL_ROW_MAJOR     rows of the (partition x broker) bit-plane, column totals by bit-sliced
 *                          counters; every layout */
#define KAO_EVAL_ROW_MAJOR 0
#define KAO_EVAL_COLUMN_MAJOR 1
int kao_set_evaluator(kao_handle *h, int32_t evaluator);
/* Schedule of the column-major evaluator: the same arithmetic, laid out differently in time.  Two are built:
 *   (1, 0x300, 512)   the default: every sum on the tensor cores, one binary MMA over a batch of 32 candidates
 *                     (kao_device_mma.cuh), with every CTA's candidates of a round sorted by the class of their control
 *                     word first, so that the 32 candidates of a batch mostly take one generator body, a generator whose
 *                     later operations share their steps across link kinds, and an MMA epilogue that scores two
 *                     candidates per instruction (16 x 2 halfword pairs); 512 threads per CTA
 *   (4, 0x22, 1024)   one warp per candidate: the column loop unrolled by four (sync 4) and, in each popcount stream
 *                     (column totals in the low hex digit of pop, leader totals in the next), two POPC per four words
 *                     with carry-save adders doing the rest; 1024 threads per CTA
 * Any other (sync, pop, threads) is refused (KAO_E_ARG).  The default is the fastest measured on an H100 (config 3;
 * (4, 0x22, 1024) is the fastest popcount one).  Results never depend on it.  The environment variable
 * KAO_SCHEDULE="sync,pop(hex),threads" sets it for every session (and kao_solve); KAO_EVALUATOR=row forces
 * the row-major evaluator. */
int kao_set_schedule(kao_handle *h, int32_t sync, int32_t pop, int32_t threads);
/* what kao_search of this session runs right now: evaluator (KAO_EVAL_*) and the schedule of the column-major one */
int kao_get_evaluator(kao_handle *h, int32_t *evaluator, int32_t *sync, int32_t *pop, int32_t *threads);
int kao_last_rounds(kao_handle *h, uint32_t *rounds_run);

/* keys of candidates idx_begin .. idx_begin+count-1 of `round` against the current base (host
 * buffer) — the per-candidate parity vector. */
int kao_candidate_keys(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                       uint32_t idx_begin, uint32_t count, uint64_t *keys);

/* sharded round, asynchronous on `stream` (a cudaStream_t, 0 = default):
 *   kao_round_launch  evaluates idx_lo..idx_hi-1 and atomically min-reduces the packed key into
 *                     *d_key (DEVICE pointer, caller pre-sets it to KAO_KEY_NONE);
 *   [caller min-all-reduces *d_key across ranks: one 8-byte collective]
 *   kao_round_apply   re-materialises the winning candidate from (seed, round, index) and makes
 *                     it the base.  Every rank applies the same key => identical bases. */
int kao_round_launch(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                     uint32_t idx_lo, uint32_t idx_hi, uint64_t *d_key, void *stream);
int kao_round_apply(kao_handle *h, uint64_t seed, uint32_t round, uint32_t round_size,
                    const uint64_t *d_key, void *stream);

/* sharded search with the reduction INSIDE the kernel, one PROCESS per GPU (kao_solve with n_gpus > 1 does
 * the same inside one process): every rank owns a mailbox in its HBM that the peers map through CUDA IPC;
 * per round every rank stores its 8-byte key into its slot of every mailbox over NVLink and takes the
 * minimum of the slots of its own (no host, no NCCL in the loop).  Setup, once per session:
 *   kao_p2p_export   -> 64 opaque bytes; all-gather them across the ranks (any transport);
 *   kao_p2p_connect  <- the world's handles in rank order.
 * kao_search_sharded must then be called by every rank with identical arguments; each evaluates
 * its contiguous slice of every round and all end with the same base and the same round_keys. */
#define KAO_IPC_HANDLE_BYTES 64
int kao_p2p_export(kao_handle *h, uint8_t *handle_out /* [KAO_IPC_HANDLE_BYTES] */);
int kao_p2p_connect(kao_handle *h, int32_t rank, int32_t world, const uint8_t *handles /* [world][64] */);
int kao_search_sharded(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                       uint32_t round_size, uint64_t *round_keys, double *device_ms);
/* the same with delta evaluation (see kao_search_delta) */
int kao_search_sharded_delta(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                             uint32_t round_size, uint64_t *round_keys, double *device_ms);

/* introspection for benchmarks: kernel launches issued by this handle so far, words per row */
int kao_stats(kao_handle *h, uint64_t *kernel_launches, int32_t *words_per_row,
              int32_t *slots, int32_t *dense_weights);

/* benchmark aid: `rounds` rounds with CUDA events around every kernel; sums per kernel kind */
int kao_profile_rounds(kao_handle *h, uint64_t seed, uint32_t first_round, uint32_t rounds,
                       uint32_t round_size, double *search_ms, double *apply_ms);

/* key layout, smaller is better: violation | (objmax - objective) | index(24).  The cost field is `ob`
 * bits wide, ob = bit length of P * RF * (largest weight) = kao_key_obj_bits(problem) (also reported in
 * kao_result.key_obj_bits), objmax = 2^ob - 1; the violation field takes the remaining 63 - 24 - ob bits
 * (15..38, at most 31 used) and saturates; bit 63 is always 0, so keys order the same as signed int64.
 * KAO_KEY_NONE = "no candidate evaluated". */
#define KAO_KEY_NONE 0x7FFFFFFFFFFFFFFFull
#define KAO_KEY_VIOLATION(k, ob) ((uint32_t)((k) >> (24 + (ob))))
#define KAO_KEY_OBJECTIVE(k, ob) (((1u << (ob)) - 1u) - ((uint32_t)((k) >> 24) & ((1u << (ob)) - 1u)))
#define KAO_KEY_INDEX(k) ((uint32_t)((k) & 0xFFFFFFu))
/* width of the cost field of this problem's keys; < 0 on a bad problem */
int kao_key_obj_bits(const kao_problem *pb);

#ifdef __cplusplus
}
#endif
#endif /* KAO_H_ */
