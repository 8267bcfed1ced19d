/*
 * b2_planner.h -- C ABI of libb2planner.so, the H100 (sm_90a) planning engine
 * behind the rl-agents plugin surface.
 *
 * Every entry point replaces the inner loop of one reference method (cited as
 * file:line under /root/reference).  Conventions (SURVEY.md section 8b):
 *   - plain C, no allocation, no ownership: every buffer is caller-owned device
 *     memory (e.g. torch.Tensor.data_ptr()) unless the name ends in _host;
 *   - `stream` is a cudaStream_t passed as void*; calls enqueue work and return
 *     without synchronising; the caller synchronises before reading results;
 *   - return 0 on success, otherwise a non-zero code; b2_last_error() gives the
 *     message for the calling thread;
 *   - distinct handles / buffers are independent: safe from different host
 *     threads or processes (scripts/experiments.py:105 forks worker processes).
 */
#ifndef B2_PLANNER_H
#define B2_PLANNER_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_OK 0
#define B2_ERR_INVALID 1   /* bad argument */
#define B2_ERR_CUDA 2      /* CUDA runtime error, see b2_last_error() */
#define B2_ERR_UNSUPPORTED 3

const char* b2_last_error(void);
int b2_version(void);
/* number of SMs / device name of the current device (diagnostics for bench.py) */
int b2_device_info(int* sm_count, int* cc_major, int* cc_minor, char* name, int name_len);

/* ------------------------------------------------------------------------
 * Environment models (the batched transition the planners call)
 * ---------------------------------------------------------------------- */
#define B2_ENV_FINITE 0   /* finite MDP tables (deterministic, except for sparse sampling) */
#define B2_ENV_HIGHWAY 1  /* HighwayLite, docs/HIGHWAY_LITE_SPEC.md         */

#define B2_ENV_INTERSECTION 2 /* IntersectionLite, docs/INTERSECTION_LITE_SPEC.md (wavefront OPD, MCTS, OLOP + b2_intersection_step) */

#define B2_HW_STATE_WORDS 136 /* 32-bit words of one HighwayLite / IntersectionLite state */
#define B2_HW_ACTIONS 5
#define B2_IL_ACTIONS 3

typedef struct b2_finite_mdp {
    int32_t n_states;
    int32_t n_actions;
    const int32_t* transition; /* [S, A] next state (deterministic mode)     */
    const double* reward;      /* [S, A]                                     */
    const uint8_t* terminal;   /* [S]                                        */
} b2_finite_mdp;

/* A finite MDP as the sampled env steps it (FiniteMDPEnv.step): r = reward[s, a]; k = searchsorted(cdf[s, a], u,
 * "right") for u = default_rng(seed).random(); s' = next[s, a, k]. */
typedef struct b2_finite_mdp_sampled {
    int32_t n_states;
    int32_t n_actions;
    int32_t n_next;          /* B: 1 "deterministic", S "stochastic" (next[s, a, k] = k), next's width "sparse" */
    int32_t reserved;
    const double* cdf;       /* [S, A, B] p.cumsum(); cdf /= cdf[-1], as Generator.choice computes it (host numpy) */
    const int32_t* next;     /* [S, A, B]                                                                       */
    const double* reward;    /* [S, A]                                                                          */
    const uint8_t* row_ok;   /* [S, A] 1 when Generator.choice accepts p[s, a] (no NaN, none negative, Kahan sum
                                within sqrt(eps) of 1); sampling a row with 0 is the reference's ValueError       */
} b2_finite_mdp_sampled;

/* One decision step of n_envs HighwayLite states (15 physics sub-steps each).
 * Replaces `env.step(a)` on a deep-copied env: deterministic.py:36-43,
 * mcts.py:145,173.  states: [n_envs, 136] words, updated in place.
 * actions: [n_envs] int32.  reward: [n_envs] float; flags: [n_envs] int32,
 * bit0 terminated, bit1 truncated.  avail_mask (nullable): [n_envs] int32
 * bitmask of get_available_actions() in the NEW state. */
int b2_highway_step(int32_t* states, const int32_t* actions, float* reward, int32_t* flags,
                    int32_t* avail_mask, int32_t n_envs, void* stream);

/* ValueIterationAgent on HighwayLite scenes, batched: per scene, the time-to-collision grid MDP that
 * `env.unwrapped.to_finite_mdp()` hands the reference's agent (rl_agents/agents/dynamic_programming/
 * value_iteration.py:17,32; docs/HIGHWAY_LITE_SPEC.md section 9: 3 speeds x 4 lanes x 10 s = 120 states, 5 actions,
 * deterministic) is built and the agent's fixed-point iteration (value_iteration.py:42-73, incl. the np.allclose early
 * exit that returns the previous iterate) is run by one warp in shared memory.
 * states [n_envs,136] i32; q_out [n_envs,120,5] f64 or NULL; action_out [n_envs] i32 = argmax_a Q[state] (:35);
 * mdp_state_out [n_envs] i32 (the scene's cell, `mdp.state`) or NULL; sweeps_out [n_envs] i32 or NULL. */
#define B2_TTC_STATES 120
int b2_highway_ttc_vi(const int32_t* states, int32_t n_envs, double gamma, int32_t iterations, double rtol,
                      double atol, double* q_out, int32_t* action_out, int32_t* mdp_state_out, int32_t* sweeps_out,
                      void* stream);

/* The same for IntersectionLite (BASELINE config C5's env model): 3 actions (0 SLOWER, 1 IDLE, 2 FASTER),
 * states [n_envs, 136] words, avail_mask in the NEW state. */
int b2_intersection_step(int32_t* states, const int32_t* actions, float* reward, int32_t* flags,
                         int32_t* avail_mask, int32_t n_envs, void* stream);

/* FiniteMDPEnv.step on a batch of n episodes of one finite MDP in any mode (the `finite_mdp` package's MDP.step),
 * one thread per episode, with the sampled planners' own step (lane_env.cuh, SampledFiniteEnv::step).  For every
 * episode i with alive[i] != 0, from s = states[i] and a = actions[i]: reward[i] = reward[s, a]; flags[i] bit0 =
 * terminal[s] (done is read on the state the action is taken in); states[i] = next[s, a, k] with k = 0 when
 * env_draws == 0 ("deterministic"), else k = Generator.choice(p.size, p=p[s, a]) of the episode's env generator,
 * env_rng [n, 6] words (pcg64_words), advanced in place; bad_row[i] = -1.  A row Generator.choice rejects (row_ok 0)
 * leaves states[i] and the generator unchanged, sets reward[i] = 0, flags[i] = 0 and reports the row s * A + a in
 * bad_row[i].  Episodes with alive[i] == 0 are not touched.  env_rng may be NULL when env_draws == 0.
 * The states and actions of the live episodes are checked on the device first, and the call synchronises `stream`
 * to read that check: a state outside [0, n_states) or an action outside [0, n_actions) steps no episode and returns
 * B2_ERR_INVALID. */
int b2_finite_step(const struct b2_finite_mdp_sampled* mdp, const uint8_t* terminal, int32_t env_draws,
                   int32_t* states, const int32_t* actions, const uint8_t* alive, uint64_t* env_rng, double* reward,
                   int32_t* flags, int32_t* bad_row, int32_t n, void* stream);

/* Self-test (tests/test_gpu_engines.py): the HighwayLite kernel divides by two constants of the spec with a
 * 3-instruction sequence instead of the full IEEE division; this compares both, exhaustively over every fp32
 * mantissa, both signs and exponents -60..60, and writes the number of differing results (must be 0). */
int b2_selftest_const_division(unsigned long long* mismatches_dev, void* stream);

/* Self-test (tests/test_gpu_highway_step_paths.py): the HighwayLite step in the per-group mode of the
 * one-tree-per-group planners -- scene s on its own 16-lane group (HighwayEnv::step, that group's mask),
 * n_steps[s] <= max_steps decisions.  actions [n_scenes, max_steps]; every intermediate state to
 * trace [n_scenes, max_steps, 136]; reward [n_scenes, max_steps]; flags [n_scenes, max_steps] = bit0 terminated,
 * bit1 truncated, available-action mask of the new state << 2.  Entries past n_steps[s] are left as they were. */
int b2_selftest_highway_step_groups(const int32_t* states, const int32_t* actions, const int32_t* n_steps,
                                    int32_t* trace, float* reward, int32_t* flags, int32_t n_scenes,
                                    int32_t max_steps, void* stream);

/* Self-tests of the device primitives the planners share (tests/test_gpu_device_primitives.py), one thread per
 * stream or case, each calling the planners' own inline functions. */

/* numpy's PCG64 (pcg64.cuh): stream s loads words [n_streams, 6] and runs ops[s, 0 .. n_ops-1] with args:
 * 0 next64, 1 next32, 2 random (out = the double's bits), 3 integers(arg) (Generator.integers(0, arg), 1 <= arg < 2^32),
 * 4 skip32(arg) and 5 seed_from(arg) (both: out = the low 64 bits of the LCG state after the op), any other code: no op,
 * out left as it was.  out [n_streams, n_ops]; words_out [n_streams, 6] the words after the last op. */
int b2_selftest_pcg64(const uint64_t* words, const int32_t* ops, const uint64_t* args, uint64_t* out,
                      uint64_t* words_out, int32_t n_streams, int32_t n_ops, void* stream);

/* kl_bound.cuh: kl[i] = bernoulli_kl(p[i], q[i]) for i < n_kl; bound[i] = kl_bound(sum[i], count[i], threshold[i],
 * lower[i] != 0) for i < n_bound.  Either part may be empty. */
int b2_selftest_kl(const double* p, const double* q, int32_t n_kl, double* kl, const double* sum,
                   const int32_t* count, const double* threshold, const int32_t* lower, int32_t n_bound, double* bound,
                   void* stream);

/* lane_env.cuh: k[i] = searchsorted_right(cdf + u_row[i] * n_next, n_next, u[i]) for i < n_u (cdf rows of n_next
 * entries); and for i < n_steps, sampled_next(*mdp, rows[i], draw[i] != 0, g) with g loaded from words [n_steps, 6]:
 * next [n_steps] and the words afterwards, words_out [n_steps, 6].  Either part may be empty. */
int b2_selftest_sampled_next(const double* cdf, int32_t n_next, const double* u, const int32_t* u_row, int32_t n_u,
                             int32_t* k, const struct b2_finite_mdp_sampled* mdp, const int64_t* rows,
                             const int32_t* draw, const uint64_t* words, int32_t n_steps, int32_t* next,
                             uint64_t* words_out, void* stream);

/* mdp_gape.cu's backup expectations: case i is a chance node whose children 0 .. K[i]-1 sit at i * max_k + j of
 * f, neg_f (= -f), counts and zeros (max_k * n_cases zeros), valued with gamma = 1.  n[i] == 0: gape_expectation (one
 * observed child, child 0, with p_hat qp[i]); n[i] >= 1: gape_expectation_kl with children 0 .. n[i]-1 observed,
 * p_hat = counts / cnt[i].  out [n_cases, 2]: the upper side (values f), then the lower side (values -f). */
int b2_selftest_gape_expectation(const double* f, const double* neg_f, const int32_t* counts, const double* zeros,
                                 int32_t max_k, const int32_t* K, const int32_t* n, const int32_t* cnt,
                                 const double* qp, const double* c, int32_t n_cases, double* out, void* stream);

/* ------------------------------------------------------------------------
 * Value iteration -- rl_agents/agents/dynamic_programming/value_iteration.py
 * ---------------------------------------------------------------------- */
#define B2_VI_DETERMINISTIC 0 /* next_v = V[T]                (:52-53)       */
#define B2_VI_STOCHASTIC 1    /* next_v = sum_s' P[s,a,s']V[s'] (:54-55)     */
#define B2_VI_SPARSE 2        /* next_v = sum_b P[s,a,b]V[N[s,a,b]] (:56-59) */

typedef struct b2_vi_problem {
    int32_t mode;
    int32_t n_actions;   /* A                                                */
    int32_t n_next;      /* B (sparse), S (stochastic), ignored otherwise    */
    int32_t reserved;    /* must be 0                                        */
    int64_t n_states;    /* S of the whole MDP (length of V)                 */
    int64_t row_begin;   /* state slab [row_begin, row_end) owned by the call */
    int64_t row_end;
    double gamma;
    double rtol, atol;   /* np.allclose tolerances (1e-5, 1e-8)              */
    /* slab-local tables: row 0 is state row_begin */
    const void* transition; /* int32 [rows,A] | double [rows,A,S] | double [rows,A,B] */
    const int32_t* next;    /* int32 [rows,A,B] (sparse only)                */
    const double* reward;   /* [rows, A]                                     */
    const uint8_t* terminal;/* [rows]                                        */
} b2_vi_problem;

/* One Bellman sweep  Q' = R + gamma * E[V(s')]  fused with V' = max_a Q' and the
 * np.allclose(Q, Q') test of fixed_point_iteration (value_iteration.py:51-63,
 * 65-73).  v_in/v_out: [S] (v_out rows of the slab are written); q_old/q_new:
 * slab-local [rows, A].  viol: int32 [>= sweep_index+1] device counters,
 * zero-initialised by the caller: the sweep adds the number of elements that
 * break allclose to viol[sweep_index]; if sweep_index > 0 and
 * viol[sweep_index-1] == 0 (previous sweep converged) the launch does nothing,
 * so a whole fixed-point loop can be enqueued without a host round trip. */
int b2_vi_sweep(const b2_vi_problem* p, const double* v_in, const double* q_old, double* q_new,
                double* v_out, int32_t* viol, int32_t sweep_index, void* stream);

/* get_state_action_value (value_iteration.py:42-45): `iterations` sweeps
 * ping-ponging q[0]/q[1] and v[0]/v[1] (q[0], v[0] must hold the initial
 * zeros).  After synchronising, the first k with viol[k]==0 marks convergence:
 * the result (the OLD iterate, :70-72) is q[k%2]; without one it is
 * q[iterations%2].  Single device (row slab = all states). */
int b2_vi_solve(const b2_vi_problem* p, double* q0, double* q1, double* v0, double* v1,
                int32_t* viol, int32_t iterations, void* stream);

/* ---- slab-sharded value iteration with the exchange fused into the sweep over NVLink peer memory ----
 * Replaces "sweep; ncclAllGather(V); ncclAllReduce(violations)" of the sharded fixed-point loop
 * (value_iteration.py:42-73 over G GPUs, one process per GPU): every rank keeps the V ping-pong buffers, an
 * arrival-flag array [world] and a violation table [iterations, world] in CUDA-IPC shared device memory
 * (b2_p2p_alloc / export / import); the sweep kernel stores V' into every rank's copy and publishes its count and
 * flag when its last CTA retires; the next sweep acquires the flags.  No NCCL call inside the loop. */
#define B2_MAX_PEERS 8
int b2_p2p_alloc(int64_t bytes, void** ptr);                          /* zeroed, IPC-exportable device memory */
int b2_p2p_free(void* ptr);
int b2_p2p_export(void* ptr, unsigned char* handle64);                /* cudaIpcGetMemHandle (64 bytes)        */
int b2_p2p_import(const unsigned char* handle64, void** peer_ptr);    /* cudaIpcOpenMemHandle + peer access    */
int b2_p2p_close(void* peer_ptr);
int b2_p2p_memset(void* ptr, int32_t value, int64_t bytes, void* stream);
int b2_p2p_read(void* dst_host, const void* src_dev, int64_t bytes, void* stream);   /* synchronous D2H */

typedef struct b2_vi_p2p {
    int32_t world, rank;
    double* v[2][B2_MAX_PEERS];      /* v[i][r]: V ping-pong buffer i ([S] doubles) in rank r's memory          */
    int32_t* flags[B2_MAX_PEERS];    /* flags[r]: rank r's [world] arrival flags; this rank writes flags[r][rank] */
    int32_t* parts[B2_MAX_PEERS];    /* parts[r]: rank r's [iterations, world] violation table                   */
    int32_t* viol_local;             /* [iterations] this rank's own counters (local scratch, zeroed)            */
    uint32_t* done;                  /* [iterations] retired-CTA counters (local scratch, zeroed)                */
    int32_t* status;                 /* [1] local scratch, zeroed: set to 1 when a peer's flag did not arrive within
                                        ~1 s (the sweep then proceeds on stale data instead of hanging the GPU)    */
} b2_vi_p2p;

/* Sweep `sweep_index` of the slab [row_begin, row_end): reads v[sweep&1][rank] and q_old, writes q_new and
 * V' into v[(sweep+1)&1][r] of every rank r.  Sparse / deterministic mode, A a power of two <= 32,
 * B in {1,2,4,8}.  After synchronising, sum_r parts[rank][k*world + r] is sweep k's allclose violation count
 * (same convergence protocol as b2_vi_sweep). */
int b2_vi_sweep_p2p(const b2_vi_problem* p, const b2_vi_p2p* x, const double* q_old, double* q_new,
                    int32_t sweep_index, void* stream);

/* Robust value iteration (rl_agents/agents/dynamic_programming/robust_value_iteration.py:39-58):
 * Q' = min over n_models models of R_m + gamma * E_m[V(s')], no terminal handling.
 * p->transition: int32 [M,S,A] (deterministic) or double [M,S,A,S] (stochastic);
 * p->reward: double [M,S,A]; p->terminal / p->next unused; rows = all states.
 * Same viol / early-exit protocol as b2_vi_sweep. */
int b2_vi_robust_sweep(const b2_vi_problem* p, int32_t n_models, const double* v_in, const double* q_old,
                       double* q_new, double* v_out, int32_t* viol, int32_t sweep_index, void* stream);

/* ------------------------------------------------------------------------
 * OPD -- rl_agents/agents/tree_search/deterministic.py
 * A batch of n_trees independent decisions, one tree per CTA, strict
 * best-first order inside each tree (bit-exact node order).
 * ---------------------------------------------------------------------- */
typedef struct b2_opd_config {
    int32_t env_kind;       /* B2_ENV_*                                      */
    int32_t n_trees;
    int32_t n_actions;      /* action_space.n: budget divisor (:118) and max branching */
    int32_t n_expansions;   /* budget // n_actions (:118)                    */
    int32_t node_capacity;  /* per tree, >= 1 + n_expansions * n_actions     */
    int32_t plan_capacity;  /* per tree, >= n_expansions + 1                 */
    int32_t keys_in_smem;   /* 1: frontier keys in shared memory when they fit */
    int32_t reserved;       /* must be 0                                     */
    double terminal_reward; /* config["terminal_reward"] (:60-63)            */
    const double* gamma_pow;     /* [n_expansions+2] gamma**d   (host floats) */
    const double* gamma_pow_div; /* [n_expansions+2] gamma**d / (1 - gamma)   */
    b2_finite_mdp mdp;      /* env_kind == FINITE                            */
    const double* terminal_bonus;/* [n_expansions+2] (terminal_reward * gamma**d) / (1 - gamma), the
                                    reference's association (:60-63), host floats */
} b2_opd_config;

/* Node arrays, each [n_trees, node_capacity] (struct-of-arrays in HBM) */
typedef struct b2_opd_tree {
    int32_t* parent;       /* -1 for the root                                */
    int32_t* first_child;  /* -1 for a leaf                                  */
    int32_t* depth;
    int32_t* count;        /* DeterministicNode.count (:18,:64-65)           */
    int32_t* meta;         /* action | n_children << 8 | done << 16          */
    double* reward;
    double* lower;         /* value_lower                                    */
    double* upper;         /* value_upper                                    */
    int32_t* state;        /* FINITE: [n_trees, cap] state ids;
                              HIGHWAY: [n_trees, cap, 136] words             */
} b2_opd_tree;

#define B2_OPD_RESULT_WORDS 16
/* per tree int32 result record:
 * [0] n_nodes [1] n_leaves [2] max_depth [3] terminal_expansions
 * [4] error (1: reward outside [0,1], deterministic.py:46-47)
 * [5] plan_len [6] tie_node (-1, or the node where get_plan met a tie that the
 *     host must break with the planner RNG, abstract.py:304-311) */

/* bytes of scratch the call needs (frontier keys + tournament + expansion order) */
int64_t b2_opd_workspace_bytes(const b2_opd_config* cfg);

/* OptimisticDeterministicPlanner.plan (:116-122): root_states [n_trees] int32
 * state ids or [n_trees,136] words.  plan: int8 [n_trees, plan_capacity]
 * greedy value_lower path (abstract.py:143-156); result: int32
 * [n_trees, B2_OPD_RESULT_WORDS]. */
int b2_opd_plan(const b2_opd_config* cfg, const int32_t* root_states, const b2_opd_tree* tree,
                void* workspace, int8_t* plan, int32_t* result, void* stream);

/* ------------------------------------------------------------------------
 * Wavefront OPD: ONE decision searched by the whole GPU.  Per wave the
 * k = min(width, expansions left, frontier size) best leaves -- in the
 * reference's arg-max order (value_upper descending, node id ascending,
 * deterministic.py:110) -- are expanded in increasing node-id order and all their
 * children simulated at once.  width = 1 is the reference's algorithm
 * (deterministic.py:106-122); for any width the result is bit-identical with the
 * specification oracle/planners.py::opd_plan_wavefront.
 * ---------------------------------------------------------------------- */
#define B2_MAX_MODELS 8
typedef struct b2_opd_wave_config {
    int32_t env_kind;       /* B2_ENV_*                                      */
    int32_t n_actions;      /* action_space.n (:118)                         */
    int32_t n_expansions;   /* budget // n_actions (:118)                    */
    int32_t node_capacity;  /* >= 1 + n_expansions * n_actions, < 2^28       */
    int32_t plan_capacity;
    int32_t width;          /* leaves expanded per wave (>= 1)               */
    int32_t max_ctas;       /* 0: one CTA per SM                             */
    int32_t n_models;       /* 0: plain OPD.  M >= 1: DROP, the joint env of M models (rl_agents/agents/robust/
                               robust.py:9-47): root_state / tree.state hold M states per node ([M] ids or
                               [M,136] words), children follow the union of the models' available actions in
                               ascending order, a node's bounds are the minima over the models of the per-model
                               path bounds (deterministic.py:52-59 with vector rewards).  Finite MDPs,
                               HighwayLite and IntersectionLite; b2_opd_plan_spec takes 0 only     */
    const double* gamma_pow;      /* [n_expansions+2] gamma**d               */
    const double* gamma_pow_div;  /* [n_expansions+2] gamma**d / (1 - gamma) */
    const double* terminal_bonus; /* [n_expansions+2] terminal_reward * gamma**d / (1 - gamma) (:60-63) */
    b2_finite_mdp mdp;
    b2_finite_mdp model_mdps[8];  /* env_kind FINITE and n_models > 0: one deterministic MDP per model */
} b2_opd_wave_config;

int64_t b2_opd_wave_workspace_bytes(const b2_opd_wave_config* cfg);
/* tree: node arrays of ONE tree ([node_capacity] each, state [node_capacity(,136)]); root_state: [1] state id
 * or [136] words; plan: int8 [plan_capacity]; result: int32 [B2_OPD_RESULT_WORDS] as for b2_opd_plan, plus
 * [7] number of waves.  Cooperative launch on `stream` (one CTA per SM). */
int b2_opd_plan_wave(const b2_opd_wave_config* cfg, const int32_t* root_state, const b2_opd_tree* tree,
                     void* workspace, int8_t* plan, int32_t* result, void* stream);

/* Speculative strict search: the reference's own one-leaf-per-iteration order (deterministic.py:106-114) -- the
 * tree is bit-identical with b2_opd_plan / width 1 -- searched by the whole GPU.  Per wave the `width` best
 * frontier leaves (value_upper descending, node id ascending) are simulated on every SM unless already cached,
 * and the longest prefix the strict order would have expanded is committed.  Same config struct (width in
 * 1..256, n_models = 0, node_capacity <= 24576); tree->state is an ARENA of b2_opd_spec_arena_slots(cfg)
 * states (a node's state is not at its own index); result as for b2_opd_plan_wave. */
int64_t b2_opd_spec_workspace_bytes(const b2_opd_wave_config* cfg);
int64_t b2_opd_spec_arena_slots(const b2_opd_wave_config* cfg);
int b2_opd_plan_spec(const b2_opd_wave_config* cfg, const int32_t* root_state, const b2_opd_tree* tree,
                     void* workspace, int8_t* plan, int32_t* result, void* stream);

/* ------------------------------------------------------------------------
 * GBOP-T -- rl_agents/agents/tree_search/state_aware.py (StateAwarePlanner), deterministic finite MDPs:
 * OPD whose leaf bounds share one value table per STATE (:66-68), tightened by a breadth-first backup through
 * the nodes aggregated by state (:42-64), with pruning of dominated leaves after every expansion (:28-40).
 * A batch of n_trees independent decisions, one warp per tree, node order / leaves / state values exactly
 * the reference's.
 * ---------------------------------------------------------------------- */
typedef struct b2_gbop_config {
    int32_t n_trees;
    int32_t n_actions;
    int32_t n_expansions;        /* budget // n_actions (deterministic.py:118)      */
    int32_t node_capacity;       /* per tree, >= 1 + n_expansions * n_actions       */
    int32_t plan_capacity;
    int32_t queue_capacity;      /* entries of the backup FIFO (result[7] = 1 on overflow) */
    int32_t backup_aggregated_nodes;   /* config key of the same name (:80-85)      */
    int32_t prune_suboptimal_leaves;
    double gamma;
    double default_value;        /* 1 / (1 - gamma), host float (:76-77)            */
    double accuracy_scale;       /* accuracy * (1 - gamma), host float (:61)        */
    const double* gamma_pow;     /* [n_expansions+2] gamma**d                       */
    const double* terminal_bonus;/* [n_expansions+2] terminal_reward * gamma**d / (1 - gamma) */
    b2_finite_mdp mdp;
} b2_gbop_config;

typedef struct b2_gbop_tree {    /* [n_trees, node_capacity] each */
    int32_t* parent;
    int32_t* first_child;
    int32_t* depth;
    int32_t* count;
    int32_t* meta;               /* action | n_children << 8 | done << 16 | still-a-leaf << 17 */
    double* reward;
    double* lower;               /* value_lower (the path sum: GBOP-T never backs it up) */
    int32_t* obs;                /* the state the node reached                      */
} b2_gbop_tree;

int64_t b2_gbop_workspace_bytes(const b2_gbop_config* cfg);
/* The first 8 * n_states bytes of every tree's workspace slice hold the state value table afterwards.
 * result: int32 [n_trees, B2_OPD_RESULT_WORDS]: [0] n_nodes [1] n_leaves [4] error [5] plan_len [6] tie_node
 * [7] queue overflow [8] expansions done. */
int b2_gbop_plan(const b2_gbop_config* cfg, const int32_t* root_states, const b2_gbop_tree* tree, void* workspace,
                 int8_t* plan, int32_t* result, void* stream);

/* GBOP-D -- rl_agents/agents/tree_search/graph_based.py (GraphBasedPlanner), deterministic finite MDPs: one graph
 * node per state with value_lower / value_upper, optimistic descent to an unexpanded state, breadth-first partial
 * value iteration through the expanded parents (pushed in ascending state id; the reference iterates a Python set).
 * n_trees independent decisions, one warp each; rng: numpy PCG64 states [n_trees, 6] consumed by the tie-breaks of
 * sampling_rule (:22-30) exactly as Generator.choice does, advanced in place. */
typedef struct b2_gbopd_config {
    int32_t n_trees;
    int32_t n_actions;
    int32_t n_epochs;            /* budget // n_actions (:119)                       */
    int32_t sampling_timeout;    /* config["sampling_timeout"] (default 100)         */
    int32_t plan_capacity;       /* >= sampling_timeout                              */
    int32_t queue_capacity;      /* per tree; result[7] = 1 on overflow              */
    double gamma;
    double default_value;        /* 1 / (1 - gamma) (:17)                            */
    double accuracy;             /* config["accuracy"] (default 1e-2, :74)           */
    b2_finite_mdp mdp;           /* terminal unused: GBOP-D ignores `done` (:46)     */
    const int32_t* rev_ptr;      /* [S+1] reverse transitions: states p with T[p, a] == s for some a, */
    const int32_t* rev_idx;      /* ascending, unique                                */
} b2_gbopd_config;
/* lower / upper: double [n_trees, S]; flags: uint8 [n_trees, S] (bit0 node exists, bit1 expanded); queue: int32
 * [n_trees, queue_capacity] scratch; plan: int8 [n_trees, plan_capacity]; result: [0] nodes [1] expansions
 * [2] epochs that found no sink [5] plan_len [7] queue overflow. */
int b2_gbopd_plan(const b2_gbopd_config* cfg, const int32_t* root_states, double* lower, double* upper, uint8_t* flags,
                  int32_t* queue, uint64_t* rng, int8_t* plan, int32_t* result, void* stream);

/* Host-buffer convenience API (callers that do not manage CUDA memory: plain C, cgo, JNI ...).
 * A handle owns the device arena of a batch of trees; *_host pointers are ordinary host memory
 * (pinned memory makes the copies asynchronous); b2_opd_plan_host is synchronous. */
typedef struct b2_opd_handle b2_opd_handle;
typedef struct b2_opd_host_config {
    int32_t env_kind, n_trees, n_actions;
    int32_t budget;          /* config["budget"]; n_expansions = budget / n_actions (:118) */
    int32_t keys_in_smem;
    int32_t kernel;          /* copied to b2_opd_config.reserved: must be 0         */
    double gamma;            /* config["gamma"], 0 <= gamma < 1                     */
    double terminal_reward;
    b2_finite_mdp mdp;       /* HOST tables when env_kind == B2_ENV_FINITE          */
} b2_opd_host_config;
int b2_opd_create(const b2_opd_host_config* cfg, b2_opd_handle** out);
void b2_opd_destroy(b2_opd_handle* h);
int32_t b2_opd_plan_capacity(const b2_opd_handle* h);   /* bytes per tree in plan_host */
/* root_states_host: [n_trees] state ids or [n_trees,136] words; plan_host: int8
 * [n_trees, plan_capacity]; result_host: int32 [n_trees, B2_OPD_RESULT_WORDS]. */
int b2_opd_plan_host(b2_opd_handle* h, const int32_t* root_states_host, int8_t* plan_host, int32_t* result_host);
/* Node arrays of one tree (first n_nodes entries) to host buffers; any pointer may be NULL. */
int b2_opd_copy_tree(b2_opd_handle* h, int32_t tree, int32_t n_nodes, int32_t* parent, int32_t* first_child,
                     int32_t* count, int32_t* meta, double* reward, double* lower, double* upper);

/* ------------------------------------------------------------------------
 * MCTS -- rl_agents/agents/tree_search/mcts.py (open loop)
 * ---------------------------------------------------------------------- */
typedef struct b2_mcts_config {
    int32_t env_kind;
    int32_t n_trees;
    int32_t n_actions;
    int32_t episodes;        /* config["episodes"] (:180)                    */
    int32_t horizon;         /* config["horizon"]                            */
    int32_t node_capacity;   /* per tree, >= 1 + episodes * n_actions        */
    int32_t rollout_policy;  /* 0 random_available, 1 random, 2 preference (:46-97) */
    int32_t prior_policy;    /* idem, for expansion priors                   */
    double temperature;      /* config["temperature"] (:127)                 */
    const double* gamma_pow; /* [horizon+1] gamma**d                         */
    const double* uniform_cdf; /* [(n_actions+1), n_actions]: row n = cumsum(ones(n)/n)/last,
                                  the cdf Generator.choice(a, 1, p) searches (host numpy)  */
    b2_finite_mdp mdp;
    /* "preference" policies (mcts.py:76-97): the preferred action label and, for n available actions with the
     * preferred one at position k-1 of the env's action order (k = 0: not available -> uniform), row
     * [(n * (n_actions+1) + k) * n_actions ..] of a host-made table: probabilities (prior policy) / the cdf
     * Generator.choice searches (rollout policy).  Only read when the policy is 2. */
    int32_t prior_pref_action, rollout_pref_action;
    const double* pref_prior;    /* [(n_actions+1), (n_actions+1), n_actions] */
    const double* pref_cdf;      /* [(n_actions+1), (n_actions+1), n_actions] */
    const int32_t* resume_nodes; /* nullable [n_trees]: > 0 -> the tree arrays already hold that many nodes
                                    (a re-rooted sub-tree, step_strategy "subtree", abstract.py:195-206,
                                    mcts.py:129-130) and the search continues from them; the caller sizes
                                    node_capacity >= resume + episodes * n_actions                      */
} b2_mcts_config;

typedef struct b2_mcts_tree {
    int32_t* parent;
    int32_t* first_child;
    int32_t* count;        /* MCTSNode.count (:248-255)                      */
    int32_t* meta;         /* action | n_children << 8                       */
    double* value;         /* MCTSNode.value                                 */
    double* prior;
} b2_mcts_tree;

#define B2_PCG64_STATE_WORDS 6 /* uint64: state hi,lo, inc hi,lo, has_uint32, uinteger */
#define B2_MCTS_RESULT_WORDS 8
/* per tree int32 result: [0] n_nodes [1] plan_len [2] env steps taken
 * [3] b2_mcts_plan_sampled: error (1: a reached probability row that Generator.choice rejects)
 * [4] b2_mcts_plan_sampled: that row s * n_actions + a, else -1.  [3] and [4] are not written by b2_mcts_plan.
 *     An error stops its own tree only. */

/* MCTS.plan (:179-184) for n_trees independent decisions, strict episode order
 * inside each tree, consuming each tree's numpy PCG64 stream exactly as
 * Generator.choice does (abstract.py:304-311, mcts.py:172).  rng: uint64
 * [n_trees, 6] numpy bit-generator states, advanced in place.  plan: int8 [n_trees, horizon].
 * env_kind: B2_ENV_FINITE, B2_ENV_HIGHWAY (5 actions) or B2_ENV_INTERSECTION (3 actions). */
int b2_mcts_plan(const b2_mcts_config* cfg, const int32_t* root_states, const b2_mcts_tree* tree,
                 uint64_t* rng, int8_t* plan, int32_t* result, void* stream);

/* MCTS.plan on a finite MDP in any mode.
 * cfg->env_kind must be B2_ENV_FINITE; cfg->mdp is not read.  The reference never reseeds its env copies, so every
 * episode's deep copy (:183) starts from the live env's generator: env_rng, uint64 [n_trees, 6] in the layout of rng,
 * read only.  With env_draws = 1 ("stochastic" / "sparse") every step an episode takes, selection or rollout, draws
 * once from that copy (Generator.choice), so step k of every episode uses the k-th double of the same stream; with
 * 0 (a "deterministic" table, n_next = 1) none.  terminal: uint8 [n_states]; done = terminal[state before the step].
 * The tree is the same open-loop tree as b2_mcts_plan's; resume_nodes ("subtree") works as there. */
int b2_mcts_plan_sampled(const b2_mcts_config* cfg, const struct b2_finite_mdp_sampled* mdp, const uint8_t* terminal,
                         int32_t env_draws, const uint64_t* env_rng, const int32_t* root_states,
                         const b2_mcts_tree* tree, uint64_t* rng, int8_t* plan, int32_t* result, void* stream);

/* step_strategy "subtree" (abstract.py:195-206) for a batch of trees, out of place: destination tree j receives the
 * sub-tree of source tree s = src_tree[j] (src_tree NULL: s = j) under that tree's root child of action action[j],
 * re-indexed breadth first with the children of a node contiguous and in order; parent / first_child are remapped,
 * count, meta, value and prior copied, and the new root's action byte set to 0xff.  Bit for bit
 * engine/mcts.py::reroot_arrays.  One launch can also gather trees into a smaller arena.
 * src / dst: arenas of [n_src, src_capacity] and [n_dst, dst_capacity] nodes; they must not share an array.
 * src_nodes[s * src_nodes_stride]: the node count of source tree s (word 0 of the last b2_mcts_plan result, stride
 * B2_MCTS_RESULT_WORDS).  kept: int32 [n_dst], the nodes written -- resume_nodes for the next b2_mcts_plan, which
 * then needs dst_capacity >= kept + episodes * n_actions:
 *   0  when action[j] < 0, when the root has no child of that action, or when kept + reserve > dst_capacity (the
 *      caller starts a new tree; destination tree j may have been partly written);
 *  -1  when s is outside [0, n_src) or its node count outside [1, src_capacity] (destination tree j untouched), or
 *      when a child range of the source leaves [1, node count).
 * Refused (B2_ERR_INVALID, nothing launched): a null pointer (src_tree excepted), n_dst < 1, n_src, a capacity or
 * src_nodes_stride < 1, arenas sharing an array, reserve < 0. */
int b2_mcts_reroot(const b2_mcts_tree* src, int32_t n_src, int32_t src_capacity, const int32_t* src_nodes,
                   int32_t src_nodes_stride, const b2_mcts_tree* dst, int32_t n_dst, int32_t dst_capacity,
                   const int32_t* src_tree, const int32_t* action, int32_t reserve, int32_t* kept, void* stream);

/* ------------------------------------------------------------------------
 * Wavefront MCTS: ONE decision searched by the whole GPU.  The reference's episode (selection mcts.py:141-149,
 * expansion :151-154, rollout :160-177, backup :257-265, recommendation :212-218) run in waves of `width`
 * episodes: selections in episode order with virtual counts, counter-based randomness, exact fixed-point
 * value sums.  Bit-identical with the specification oracle/planners.py::mcts_plan_wavefront.
 * ---------------------------------------------------------------------- */
typedef struct b2_mcts_wave_config {
    int32_t env_kind;
    int32_t n_actions;
    int32_t episodes;        /* config["episodes"]                              */
    int32_t horizon;         /* config["horizon"] (<= 64)                       */
    int32_t node_capacity;   /* >= 1 + episodes * n_actions (episode e owns ids 1 + e*n_actions ..) */
    int32_t width;           /* episodes per wave, 1..1024                      */
    int32_t rollout_policy;  /* 0 random_available (the only one implemented)   */
    int32_t prior_policy;
    double temperature;      /* config["temperature"] (:127)                    */
    uint64_t seed;           /* counter-based generator seed                    */
    const double* gamma_pow; /* [horizon+1] gamma**h                            */
    b2_finite_mdp mdp;
    int32_t max_ctas;        /* 0: one CTA per SM                               */
    int32_t reserved;
} b2_mcts_wave_config;

typedef struct b2_mcts_wave_tree {   /* [node_capacity] each; unused ids keep parent == -2 */
    int32_t* parent;
    int32_t* first_child;
    int32_t* count;
    int32_t* meta;           /* action | n_children << 8                        */
    int64_t* vsum;           /* sum of the returns backed up through the node, 2^-40 units */
    double* value;           /* vsum * 2^-40 / count (written at the end)       */
} b2_mcts_wave_tree;

int64_t b2_mcts_wave_workspace_bytes(const b2_mcts_wave_config* cfg);
/* root_state: [1] state id or [136] words; plan: int8 [horizon]; result: int32 [B2_MCTS_RESULT_WORDS]:
 * [0] node_capacity [1] plan_len [2] env steps [3] waves [4..7] phase clocks.  Cooperative launch. */
int b2_mcts_plan_wave(const b2_mcts_wave_config* cfg, const int32_t* root_state, const b2_mcts_wave_tree* tree,
                      void* workspace, int8_t* plan, int32_t* result, void* stream);

/* b2_mcts_plan_wave on a finite MDP in any mode.
 * cfg->env_kind must be B2_ENV_FINITE; cfg->mdp is not read.  mdp, terminal and env_draws as in b2_mcts_plan_sampled;
 * env_rng: uint64 [6], the live env's generator, which every episode's env copy starts from, so step h of every
 * episode draws the same double of its stream.  rejected: int32 [2], the lowest episode that reaches a probability
 * row Generator.choice rejects and that row s * n_actions + a, else -1 -1; the search stops after that episode's
 * wave.  result as for b2_mcts_plan_wave. */
int b2_mcts_plan_wave_sampled(const b2_mcts_wave_config* cfg, const struct b2_finite_mdp_sampled* mdp,
                              const uint8_t* terminal, int32_t env_draws, const uint64_t* env_rng,
                              const int32_t* root_state, const b2_mcts_wave_tree* tree, void* workspace, int8_t* plan,
                              int32_t* result, int32_t* rejected, void* stream);

/* ------------------------------------------------------------------------
 * OLOP / KL-OLOP -- rl_agents/agents/tree_search/olop.py
 * ---------------------------------------------------------------------- */
typedef struct b2_olop_config {
    int32_t env_kind;
    int32_t n_trees;
    int32_t n_actions;
    int32_t episodes;        /* config["episodes"] (OLOP.allocation, :50-62)  */
    int32_t horizon;         /* config["horizon"]                            */
    int32_t node_capacity;   /* per tree, >= 1 + episodes*horizon*n_actions   */
    int32_t kl;              /* 1: upper_bound.type == "kullback-leibler"; 0: the
                                reference leaves mu_ucb = inf (:153-163)      */
    int32_t continuation;    /* 0 "zeros", 1 "uniform" (:79-82)               */
    double gamma;
    const double* thresholds;/* [episodes] eval(upper_bound.threshold) per episode (:160) */
    const double* init_upper;/* [horizon+2] (1 - gamma**(L+1-d)) / (1 - gamma) (:118-119) */
    b2_finite_mdp mdp;
} b2_olop_config;

typedef struct b2_olop_tree {
    int32_t* parent;
    int32_t* first_child;
    int32_t* count;
    int32_t* meta;           /* action | n_children << 8 | done << 16          */
    double* cumulative;      /* OLOPNode.cumulative_reward                     */
    double* mu_ucb;
    double* upper;           /* value_upper                                    */
} b2_olop_tree;

#define B2_OLOP_RESULT_WORDS 8
/* per tree int32 result: [0] n_nodes [1] plan_len
 * [2] error (1: reward outside [0,1], olop.py:133-134; 2: "zeros" continuation
 *     with action 0 unavailable -- a KeyError in the reference, :82,:88; sampled
 *     only -- 3: a reached probability row that Generator.choice rejects)
 * [3] b2_olop_plan_sampled: the rejected row s * n_actions + a of error 3, else -1;
 *     not written by b2_olop_plan.  An error stops its own tree only. */

/* OLOP.plan (:94-100); rng and env_kind as in b2_mcts_plan; plan: int8 [n_trees, horizon]. */
int b2_olop_plan(const b2_olop_config* cfg, const int32_t* root_states, const b2_olop_tree* tree,
                 uint64_t* rng, int8_t* plan, int32_t* result, void* stream);

/* OLOP.plan on a finite MDP in any mode.
 * cfg->env_kind must be B2_ENV_FINITE; cfg->mdp is not read.  Every episode seeds the env copy's generator with
 * default_rng(np_random.randint(2**30)) (:73); with env_draws = 1 ("stochastic" / "sparse") each of the horizon
 * steps draws once from it (Generator.choice), after a terminal state too; with 0 (a "deterministic" table,
 * n_next = 1) none.  terminal: uint8 [n_states]; done = terminal[state before the step].  The tree is the same
 * open-loop tree as b2_olop_plan's; mu_ucb and upper differ from the host's only through CUDA's log. */
int b2_olop_plan_sampled(const b2_olop_config* cfg, const struct b2_finite_mdp_sampled* mdp, const uint8_t* terminal,
                         int32_t env_draws, const int32_t* root_states, const b2_olop_tree* tree, uint64_t* rng,
                         int8_t* plan, int32_t* result, void* stream);

/* ------------------------------------------------------------------------
 * MDP-GapE -- rl_agents/agents/tree_search/mdp_gape.py (KL upper bound).  b2_mdp_gape_plan runs the deterministic
 * env models, where a chance node only ever observes one next state; b2_mdp_gape_plan_sampled runs finite MDPs in
 * every mode, where a chance node observes up to max_next_states distinct next states and its backup solves the
 * KL-constrained expectation (utils.py:292-342) by Newton's method.
 * ---------------------------------------------------------------------- */
typedef struct b2_mdp_gape_config {
    int32_t env_kind;
    int32_t n_trees;
    int32_t n_actions;
    int32_t episodes;        /* config["episodes"]; the stopping rule runs at most episodes + 2 (:94-110) */
    int32_t horizon;         /* config["horizon"]                            */
    int32_t node_capacity;   /* per tree, >= 1 + (episodes+2)*horizon*(n_actions+max_next_states) */
    int32_t max_next_states; /* config["max_next_states_count"]: placeholders per chance node (:267-270) */
    int32_t continuation;    /* 0 "zeros", 1 "uniform" (:194-196)              */
    double gamma;
    double accuracy;         /* stopping rule: challenger.upper - best.lower < accuracy (:101) */
    const double* thresholds;            /* [episodes+3] eval(upper_bound.threshold) by count (:200-212) */
    const double* transition_thresholds; /* [episodes+3] eval(upper_bound.transition_threshold) by count (:307-313) */
    const double* init_upper;/* [horizon+1] (1 - gamma**(H-d)) / (1 - gamma) by depth d (:145-147) */
    b2_finite_mdp mdp;
} b2_mdp_gape_config;

/* One arena for decision and chance nodes; node id = creation order (placeholders in index order, chance nodes in
 * available-action order).  The children of a chance node are its placeholders fc .. fc+K-1.  The i-th distinct next
 * state observed takes placeholder fc+i, so a chance node with n observed states orders its children as the reference
 * does: fc+n .. fc+K-1, then fc .. fc+n-1 (b2_mdp_gape_plan: n = 1). */
typedef struct b2_mdp_gape_tree {
    int32_t* parent;
    int32_t* first_child;
    int32_t* count;
    int32_t* meta;           /* label | n_children << 8 | done << 16 | kind << 17; label = action (chance node),
                                placeholder index (decision node), 0xff (root); kind 0 decision, 1 chance */
    double* cumulative;      /* DecisionNode.cumulative_reward                 */
    double* mu_ucb;          /* KL upper / lower bound of the mean reward      */
    double* mu_lcb;
    double* upper;           /* value_upper                                    */
    double* lower;           /* value_lower                                    */
} b2_mdp_gape_tree;

#define B2_MDP_GAPE_RESULT_WORDS 8
/* per tree int32 result: [0] n_nodes [1] episodes run [2] error (1: reward outside [0,1], olop.py:133-134;
 * 2: a single available action at the root -- max() of an empty list in the reference, :247; sampled only --
 * 3: a chance node observed more than max_next_states distinct next states, the reference's "No more placeholder
 * nodes available" ValueError, :283-285; 4: a reached probability row that Generator.choice rejects) [3] recommended
 * action [4] best [5] challenger (root children's node ids, UGapE :238-249) [6] sampled: the rejected row
 * s * n_actions + a of error 4, else -1; 0 for b2_mdp_gape_plan.  An error stops its own tree only. */

/* MDPGapE.plan (:94-110); rng as in b2_mcts_plan; plan: int8 [n_trees], the recommended action (-1 on error). */
int b2_mdp_gape_plan(const b2_mdp_gape_config* cfg, const int32_t* root_states, const b2_mdp_gape_tree* tree,
                     uint64_t* rng, int8_t* plan, int32_t* result, void* stream);

/* MDPGapE.plan on a finite MDP in any mode.
 * cfg->env_kind must be B2_ENV_FINITE; cfg->mdp is not read.  Every episode seeds the env copy's generator with
 * default_rng(np_random.randint(2**30)) (:67); with env_draws = 1 ("stochastic" / "sparse") every step draws once
 * from it (Generator.choice), with 0 (a "deterministic" table, n_next = 1) none.  terminal: uint8 [n_states]; done =
 * terminal[state before the step].  keys: int32 [n_trees, node_capacity], written: the state id a decision node was
 * observed under, -1 on unobserved placeholders, the root and chance nodes.  Floats are fp64 in the reference's order,
 * its dot products as fma chains; only CUDA's log / exp differ from the host's. */
int b2_mdp_gape_plan_sampled(const b2_mdp_gape_config* cfg, const struct b2_finite_mdp_sampled* mdp,
                             const uint8_t* terminal, int32_t env_draws, const int32_t* root_states,
                             const b2_mdp_gape_tree* tree, int32_t* keys, uint64_t* rng, int8_t* plan, int32_t* result,
                             void* stream);

/* ------------------------------------------------------------------------
 * BRUE -- rl_agents/agents/tree_search/brue.py (deterministic env models, so every chance node has exactly one
 * next-state child).  Incremental means, host gamma**d and arg-maxes only: the trees equal the reference's bit for bit.
 * ---------------------------------------------------------------------- */
typedef struct b2_brue_config {
    int32_t env_kind;
    int32_t n_trees;
    int32_t n_actions;       /* action_space.n: rollout actions are randint(n_actions), available or not (:27) */
    int32_t budget;          /* config["budget"] >= 1: env steps; the last rollout runs to its end (:66-71) */
    int32_t horizon;         /* config["horizon"] >= 1                         */
    int32_t node_capacity;   /* per tree, >= 1 + 2 * (budget + horizon - 1)    */
    double gamma;
    const double* gamma_pow; /* [horizon] gamma**d (host Python floats, :63)   */
    b2_finite_mdp mdp;
} b2_brue_config;

/* One arena for decision and chance nodes; node id = creation order.  A decision node's chance children form a list
 * first_child -> next_sibling -> ... in creation order (the reference's dict order); a chance node's first_child is
 * its one decision child. */
typedef struct b2_brue_tree {
    int32_t* parent;
    int32_t* first_child;
    int32_t* next_sibling;   /* -1 at the end of a list                       */
    int32_t* count;
    int32_t* meta;           /* action | kind << 8; action 0xff on decision nodes; kind 0 decision, 1 chance */
    double* value;           /* ChanceNode.value / DecisionNode.reward (:82-86, :104-108) */
    int32_t* path;           /* [n_trees, horizon] scratch: the chance nodes of the current rollout */
    double* path_reward;     /* [n_trees, horizon] scratch: their rewards      */
} b2_brue_tree;

#define B2_BRUE_RESULT_WORDS 8
/* per tree int32 result: [0] n_nodes [1] rollouts run [2] env steps taken (budget - available_budget)
 * [3] recommended action [4] error (1: node_capacity exhausted -- cannot happen at the documented capacity) */

/* BRUE.plan (:66-75); rng as in b2_mcts_plan; plan: int8 [n_trees], the recommended action (-1 on error). */
int b2_brue_plan(const b2_brue_config* cfg, const int32_t* root_states, const b2_brue_tree* tree, uint64_t* rng,
                 int8_t* plan, int32_t* result, void* stream);

/* ------------------------------------------------------------------------
 * Sparse sampling -- rl_agents/agents/tree_search/sparse_sampling.py.  Finite MDPs in all three modes (the sampled
 * env's `seed(np_random.randint(2**30))` and `Generator.choice(p.size, p=p)` replayed on the device) and HighwayLite.
 * The values are the reference's fp64 operations in its order: every node equals the reference's bit for bit.
 * ---------------------------------------------------------------------- */
typedef struct b2_sparse_sampling_config {
    int32_t env_kind;        /* B2_ENV_FINITE or B2_ENV_HIGHWAY                                                 */
    int32_t n_trees;
    int32_t n_actions;       /* finite: action_space.n, every action is expanded (the AttributeError fallback of
                                estimateV, :40-43); HighwayLite: 5, its available actions in env order          */
    int32_t horizon;         /* config["horizon"] >= 1 (0 leaves the root childless, :45-46)                    */
    int32_t C;               /* config["C"] >= 1: samples per chance node (:76)                                 */
    int32_t reserved;
    double gamma;            /* config["gamma"]: value = reward + gamma * S / C (:87-88)                        */
    b2_finite_mdp_sampled mdp;   /* env_kind == FINITE                                                          */
} b2_sparse_sampling_config;

/* Optional creation-order dump of every tree ([n_trees, capacity] each); pass NULL to plan without it. */
typedef struct b2_sparse_sampling_tree {
    int32_t capacity;        /* nodes per tree; running out sets error 1                                        */
    int32_t reserved;
    int32_t* parent;         /* -1 for the root                                                                 */
    int32_t* kind;           /* 0 DecisionNode, 1 ChanceNode                                                    */
    int32_t* key;            /* chance: the action; decision: the next state (finite), -1 (HighwayLite, root)   */
    int32_t* depth;          /* Node.depth: a chance node has its parent's depth (:34, :68)                     */
    int32_t* count;          /* DecisionNode.count: samples that reached it (:83); 0 on chance nodes            */
    double* value;           /* DecisionNode / ChanceNode.value (:51, :87-88)                                   */
} b2_sparse_sampling_tree;

#define B2_SPARSE_SAMPLING_RESULT_WORDS 8
/* per tree int32 result: [0] nodes created [1] chance nodes [2] samples drawn (C per chance node) [3] recommended
 * action (-1 on error) [4] error (1: tree capacity exhausted; 2: a sampled probability row that Generator.choice
 * rejects) [5] that row, s * n_actions + a (-1 otherwise) */

/* Bytes of scratch the call needs: the depth-first search's stack of `horizon` frames per tree (and, on HighwayLite,
 * the horizon + 1 env states along the current path). */
int64_t b2_sparse_sampling_workspace_bytes(const b2_sparse_sampling_config* cfg);

/* SparseSampling.plan (:21-28) for n_trees independent decisions, one tree per lane (finite) or per 16-lane group
 * (HighwayLite).  Strict depth-first order: per chance node C draws of randint(2**30), the distinct next states in
 * first-visit order, then their estimateV; the root's tie-break draws choice(indices) (abstract.py:304-311).
 * rng: uint64 [n_trees, 6] numpy PCG64 states, advanced in place; root_states: [n_trees] state ids or [n_trees, 136]
 * words; root_q: double [n_trees, n_actions], the root's chance values (NaN for unavailable actions); plan: int8
 * [n_trees]; tree: NULL or the dump. */
int b2_sparse_sampling_plan(const b2_sparse_sampling_config* cfg, const int32_t* root_states,
                            const b2_sparse_sampling_tree* tree, void* workspace, uint64_t* rng, double* root_q,
                            int8_t* plan, int32_t* result, void* stream);

/* Bytes of scratch b2_sparse_sampling_plan_levels needs, sized for the worst case in which every decision node has
 * all n_actions actions: per-node ints and fp64 values for every level and, on HighwayLite, two levels of
 * n_actions^(horizon - 1) scenes.  0 for a config that call refuses. */
int64_t b2_sparse_sampling_levels_workspace_bytes(const b2_sparse_sampling_config* cfg);

/* The same decision as b2_sparse_sampling_plan -- every output bit for bit, the dump's creation order included -- for
 * ONE tree on a deterministic model (HighwayLite, or a finite MDP with mdp.n_next == 1), searched by the whole GPU
 * level by level in one cooperative launch: level d's chance nodes are numbered by a prefix sum of its available-
 * action counts and stepped in parallel, values are backed up level by level, and the planner's stream is skipped by
 * C halves per chance node in closed form.  Refused (B2_ERR_INVALID): n_trees != 1, n_next != 1, horizon < 1,
 * C < 1, null pointers, and a worst-case tree that does not fit int32 node ids.  mdp.cdf and mdp.row_ok are not
 * read: a one-entry row always samples its one next state.  A dump capacity below the node count sets error 1; the
 * other outputs are then unspecified. */
int b2_sparse_sampling_plan_levels(const b2_sparse_sampling_config* cfg, const int32_t* root_states,
                                   const b2_sparse_sampling_tree* tree, void* workspace, uint64_t* rng, double* root_q,
                                   int8_t* plan, int32_t* result, void* stream);

/* ------------------------------------------------------------------------
 * MCTS with double progressive widening -- rl_agents/agents/tree_search/mcts_dpw.py (MCTSDPW).  Finite MDPs in all
 * three modes (the env copy's `seed(np_random.randint(2**30))` once per run, then Generator.choice(p.size, p=p) per
 * step, replayed on the device) and HighwayLite.  Widening thresholds and the exploration bonus come from host tables
 * built with the reference's own expressions, so every node equals the reference's bit for bit.
 * ---------------------------------------------------------------------- */
typedef struct b2_mcts_dpw_config {
    int32_t env_kind;        /* B2_ENV_FINITE or B2_ENV_HIGHWAY                                                 */
    int32_t n_trees;
    int32_t n_actions;       /* 1..8; finite: every action is available; HighwayLite: 5                         */
    int32_t episodes;        /* config["episodes"] >= 1: runs per tree (mcts.py:179-184)                         */
    int32_t horizon;         /* config["horizon"] >= 1                                                          */
    int32_t node_capacity;   /* per tree, >= 1 + 2 * episodes (a run adds at most a chance and a decision node)  */
    int32_t rollout_policy;  /* 0 random_available, 1 random, 2 preference (mcts.py:46-97), as b2_mcts_config    */
    int32_t rollout_pref_action;
    int32_t closed_loop;     /* config["closed_loop"]: key a chance node's children on the observation (:79)     */
    int32_t open_key;        /* the key of every observation in open loop: sha1("None")[:5] as a 20-bit integer  */
    int32_t env_draws;       /* finite: 1 when the MDP is not "deterministic" (every step draws from the env's own
                                generator, a width-1 row included)                                             */
    int32_t reserved;
    double temperature;      /* config["temperature"]: UCB index value + temperature * bonus (:150)              */
    const double* gamma_pow; /* [horizon] gamma**d (host Python floats)                                          */
    const double* uniform_cdf;   /* [(n_actions+1), n_actions], as b2_mcts_config                               */
    const double* pref_cdf;      /* [(n_actions+1), (n_actions+1), n_actions], read when rollout_policy == 2     */
    const int32_t* action_widen; /* [episodes+1] by decision-node count N: the largest m <= n_actions for which
                                    `k_action*N**alpha_action < m` is false (-1: none); a node with m children
                                    adds an action iff m <= action_widen[N] and not every action has one (:121-127) */
    const int32_t* state_widen;  /* [episodes+1] the same for k_state / alpha_state, m <= episodes (:175)        */
    const double* bonus;         /* [episodes*(episodes+1)/2] np.sqrt(np.log(N / n)) at N (N-1)/2 + n-1,
                                    1 <= n <= N <= episodes (host numpy)                                        */
    const int32_t* obs_keys;     /* finite, closed loop: [S] sha1(str(s))[:5] as a 20-bit integer                 */
    const uint8_t* terminal;     /* finite: [S], `done` of a step taken in s                                      */
    b2_finite_mdp_sampled mdp;   /* env_kind == FINITE                                                          */
} b2_mcts_dpw_config;

/* One arena for decision and chance nodes; node id = creation order.  A node's children form a list first_child ->
 * next_sibling -> ... in creation order (the reference's dict order). */
typedef struct b2_mcts_dpw_tree {
    int32_t* parent;         /* -1 for the root                                                                  */
    int32_t* first_child;
    int32_t* next_sibling;   /* -1 at the end of a list                                                          */
    int32_t* count;          /* Node.count                                                                       */
    int32_t* kind;           /* 0 DecisionNode, 1 ChanceNode                                                     */
    int32_t* key;            /* chance: the action; decision: the observation key (closed loop: obs_keys[s] on a
                                finite MDP, the step count t on HighwayLite; open loop: open_key), -1 at the root */
    double* value;           /* MCTSNode.value (mcts.py:248-255)                                                 */
} b2_mcts_dpw_tree;

#define B2_MCTS_DPW_RESULT_WORDS 8
/* per tree int32 result: [0] n_nodes [1] runs completed [2] env steps [3] recommended action (-1 on error)
 * [4] error (1: node_capacity exhausted; 2: a sampled probability row that Generator.choice rejects; 3: a decision
 * node that can neither add an action nor select one; 4: a chance node that can neither add a state nor choose one)
 * [5] the rejected row, s * n_actions + a (-1 otherwise) */

/* MCTSDPW.plan (mcts.py:179-184, mcts_dpw.py:59-94) for n_trees independent decisions, one tree per lane (finite) or
 * per 16-lane group (HighwayLite), runs in strict order.  rng: uint64 [n_trees, 6] numpy PCG64 states of the planners'
 * streams, advanced in place; root_states: [n_trees] state ids or [n_trees, 136] words; plan: int8 [n_trees], the
 * root's selection_rule (mcts.py:212-218). */
int b2_mcts_dpw_plan(const b2_mcts_dpw_config* cfg, const int32_t* root_states, const b2_mcts_dpw_tree* tree,
                     uint64_t* rng, int8_t* plan, int32_t* result, void* stream);

/* ------------------------------------------------------------------------
 * PlaTyPOOS -- rl_agents/agents/tree_search/platypoos.py (PlaTyPOOS, PlaTyPOOSNode).  Finite MDPs in all three modes
 * and HighwayLite.  The search runs one depth layer at a time; every table that needs log2, ceil, floor or pow comes
 * from the host, evaluated with the reference's own expressions, so every node equals the reference's bit for bit.
 * ---------------------------------------------------------------------- */
typedef struct b2_platypoos_config {
    int32_t env_kind;        /* B2_ENV_FINITE or B2_ENV_HIGHWAY                                                 */
    int32_t n_trees;
    int32_t n_actions;       /* finite: action_space.n, whose actions 1..n-1 are expanded (the reference's fallback
                                range(1, n), :145-147); HighwayLite: 5, its available actions in env order      */
    int32_t horizon;         /* h_max >= 2 (config["horizon"]): the root is expanded h_max times per action      */
    int32_t node_capacity;   /* per tree; running out sets error 1                                              */
    int32_t layer_capacity;  /* the widest depth layer per tree (scene, sort and selection slots); error 1 past it  */
    int32_t max_p;           /* entries per depth in the quota tables: p_top(h) < max_p <= 32                    */
    int32_t env_draws;       /* finite: 1 when the MDP is not "deterministic" (a new child's state is drawn by
                                Generator.choice of the env copy seeded with its first sample's randint(2**30))   */
    const int32_t* p_top;        /* [horizon] p_top(h) of explore(h) (:41), entry 0 unused                      */
    const int32_t* nodes_count;  /* [horizon, max_p] at h * max_p + p (:44)                                      */
    const int32_t* evaluations;  /* [horizon, max_p] (:45)                                                       */
    const int32_t* min_visits;   /* [horizon, max_p] (:46)                                                       */
    const int32_t* cv_count;     /* [horizon] cross_validate's evaluations at a node of depth d (:75-76)          */
    const double* gamma_pow;     /* [horizon] gamma**d: a child of depth d + 1 has value parent.value + gamma**d *
                                    cumulative_reward / count (:129-130)                                         */
    const uint8_t* terminal;     /* finite: [S], `done` of a step taken in s                                      */
    b2_finite_mdp_sampled mdp;   /* env_kind == FINITE                                                          */
} b2_platypoos_config;

/* The arena, [n_trees, node_capacity] per field; node id = creation order.  A node's children are contiguous, in its
 * available-action order, from first_child. */
typedef struct b2_platypoos_tree {
    int32_t* parent;         /* -1 for the root                                                                  */
    int32_t* first_child;    /* -1 until the node is expanded with at least one sample                           */
    int32_t* action;         /* the incoming action, -1 at the root                                              */
    int32_t* depth;
    int32_t* count;          /* samples of the node's (parent state, action) (:127)                              */
    int32_t* flags;          /* bit 0 done, bit 1 to_expand                                                       */
    int32_t* state;          /* finite: the state id the first sample reached; HighwayLite: its available-action
                                mask                                                                             */
    double* cumulative;      /* cumulative_reward (:126)                                                          */
    double* value;           /* value (:128-129); the root's is 0.0                                               */
    double* reward;          /* the reward of the node's (parent state, action) step                             */
} b2_platypoos_tree;

#define B2_PLATYPOOS_RESULT_WORDS 8
/* per tree int32 result: [0] nodes [1] openings (the reference logs them, :95) [2] plan length [3] error (1: node or
 * layer capacity exhausted; 2: a sampled probability row that Generator.choice rejects, reached; 3: cross-validation
 * would create a child; 4: no candidate) [4] the rejected row, s * n_actions + a (-1 otherwise) [5] env steps (one per
 * created child) [6] candidates [7] 0 */

/* Bytes of scratch per call: per tree the two ping-pong layers of HighwayLite scenes and the sort and selection lists
 * of one layer. */
int64_t b2_platypoos_workspace_bytes(const b2_platypoos_config* cfg);

/* PlaTyPOOS.plan (:88-97) for n_trees independent decisions, one tree per CTA.  rng: uint64 [n_trees, 6] numpy PCG64
 * states of the planners' streams, advanced in place by every randint(2**30) the reference draws; root_states:
 * [n_trees] state ids or [n_trees, 136] words; plan: int8 [n_trees, horizon], the actions from the root to the best
 * candidate (result word 2 of them); candidates: int32 [n_trees, 2 * max_p], (p, node id) pairs in dict order. */
int b2_platypoos_plan(const b2_platypoos_config* cfg, const int32_t* root_states, const b2_platypoos_tree* tree,
                      void* workspace, uint64_t* rng, int8_t* plan, int32_t* candidates, int32_t* result,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2_PLANNER_H */
