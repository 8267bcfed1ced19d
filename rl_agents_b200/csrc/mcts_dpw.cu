// MCTS with double progressive widening -- MCTSDPW.plan of rl_agents/agents/tree_search/mcts_dpw.py (with the
// inherited MCTS.plan / evaluate and MCTSNode.update / selection_rule of mcts.py) for a BATCH of independent decisions.
// Runs inside one tree stay in strict order (every run reads the statistics the previous one wrote).
//
// One run (MCTSDPW.run, :59-90): `state.seed(np_random.randint(2**30))`, then the descent while depth < horizon, the
// last step was not terminal and the decision node was visited before (or is the root).
//   - Decision node (get_child, :120-127): a new action while not every available action has a chance child and
//     `k_action*N**alpha_action < len(children)` is false (host table action_widen), drawn by choice() from the
//     unexplored actions in ascending id order (list() of a small-int set, :115-118).  Otherwise the UCB index
//     value + temperature * bonus[N][n] of every child in insertion order, the first maximum picked by random_argmax
//     (abstract.py:304-311).  The bonus is the host's np.sqrt(np.log(N / n)), so only a correctly rounded multiply
//     and add run here.
//   - The env steps; the 4-tuple step drops truncation (:76).
//   - Chance node (get_child, :171-182): the child under the observation's key (closed loop) or the one key of
//     open loop; an unseen key becomes a new child while `k_state*N**alpha_state < len(children)` is false (host
//     table state_widen), otherwise choice() picks an existing child and the env keeps the state it sampled.
// A run that did not end terminal rolls out with the rollout policy (MCTS.evaluate, mcts.py:160-177), as mcts.cu
// draws it, until the horizon, a terminal or a truncated step.  The return, sum of gamma**d * r, is backed up from the
// last decision node to the root: count += 1; value += 1.0 / count * (total - value).
//
// Two streams per run: the planner's numpy PCG64 (seed, widening, tie, state-choice and rollout draws) and, on a
// stochastic finite MDP, the env copy's default_rng(seed) (Pcg64::seed_from), one random() per step.  Values are
// fp64 in the reference's order of operations and the library builds with -fmad=false, so every node equals the
// reference's bit for bit.
//
// One tree per lane (finite MDP) or per 16-lane group (HighwayLite, lane = vehicle slot, hw::step's mapping as in
// mcts.cu).  Every lane of a group runs the same search on group-uniform values and draws from its own copy of the
// planner's stream; lane 0 writes the tree.
#include <math.h>

#include "common.cuh"
#include "lane_env.cuh"
#include "pcg64.cuh"

namespace b2 {
namespace {

constexpr int KIND_DECISION = 0, KIND_CHANCE = 1;
constexpr int MAX_ACTIONS_DPW = 8;
constexpr int ERR_CAPACITY = 1, ERR_BAD_ROW = 2, ERR_NO_ACTION = 3, ERR_NO_STATE = 4;

struct DpwArgs {
    b2_mcts_dpw_config cfg;
    b2_mcts_dpw_tree tree;
    const int32_t* root_states;
    uint64_t* rng;
    int8_t* plan;
    int32_t* result;
    LaneModel model;
};

// The observation's key: the state's on the finite MDP; on HighwayLite the step count t, which the host turns into
// sha1(str(t))[:5] for the dump (the model is deterministic, so a chance node has one child either way).
template <class Env>
__device__ __forceinline__ int obs_key(const Env& env, const b2_mcts_dpw_config& c) {
    if constexpr (kSampled<Env>) return c.obs_keys[env.s]; else return env.t;
}

// DecisionNode / ChanceNode.__init__: value 0, count 0, appended to the parent's children after `last`
__device__ __forceinline__ void new_node(const b2_mcts_dpw_tree& tr, int64_t nb, int id, int parent, int last,
                                         int kind, int key) {
    tr.parent[nb + id] = parent; tr.first_child[nb + id] = -1; tr.next_sibling[nb + id] = -1;
    tr.count[nb + id] = 0; tr.kind[nb + id] = kind; tr.key[nb + id] = key; tr.value[nb + id] = 0.0;
    if (parent >= 0) {
        if (last < 0) tr.first_child[nb + parent] = id;
        else tr.next_sibling[nb + last] = id;
    }
}

template <class Env>
__global__ void __launch_bounds__(128, Env::GROUP == 16 ? 4 : 8) mcts_dpw_kernel(DpwArgs a) {
    B2_LANE_MAP_LIVE(Env, a.cfg.n_trees);          // whole lane groups: no live lane of a group leaves
    const b2_mcts_dpw_config& c = a.cfg;
    const b2_mcts_dpw_tree& tr = a.tree;
    const int A = c.n_actions, H = c.horizon;
    const int64_t nb = (int64_t)tree * c.node_capacity;

    Pcg64 rng;
    rng.load(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
    if (writer) new_node(tr, nb, 0, -1, -1, KIND_DECISION, -1);      // DecisionNode(parent=None)
    __syncwarp(gmask);
    int n_nodes = 1, runs = 0, steps = 0, error = 0, bad_row = -1;

    for (int ep = 0; ep < c.episodes; ++ep) {
        if (n_nodes + 2 > c.node_capacity) { error = ERR_CAPACITY; break; }
        Env env;
        env.load_root(a.root_states, tree, li);                       // safe_deepcopy_env(state), mcts.py:183
        env.seed(a.model, rng.integers(1u << 30));                     // state.seed(np_random.randint(2**30)), :69
        int node = 0, depth = 0;
        bool term = false, trunc = false;
        double total = 0.0;
        while (depth < H && !term && (node == 0 || tr.count[nb + node] != 0)) {
            // DecisionNode.get_child (:120-127)
            const int N = tr.count[nb + node];
            const int amask = env.avail(A, gmask);
            int n_children = 0, last = -1, explored = 0;
            for (int ch = tr.first_child[nb + node]; ch >= 0; ch = tr.next_sibling[nb + ch]) {
                ++n_children;
                last = ch;
                explored |= 1 << tr.key[nb + ch];
            }
            int chance = -1, action = 0;
            if (n_children != __popc(amask) && n_children <= c.action_widen[N]) {
                // expand (:115-118): choice(list(unexplored)), the symmetric difference in ascending action order
                const int unexplored = amask ^ explored;
                int pick = (int)rng.integers((uint32_t)__popc(unexplored));
                int m = unexplored;
                while (pick-- > 0) m &= m - 1;
                action = __ffs(m) - 1;
                chance = n_nodes++;
                if (writer) new_node(tr, nb, chance, node, last, KIND_CHANCE, action);
                __syncwarp(gmask);
            } else {
                // selection_strategy (:139-154): value + temperature * sqrt(log(N / n)), random_argmax
                const double* bonus = c.bonus + ((int64_t)N * (N - 1) / 2 - 1);
                double best = -INFINITY;
                int ties = 0;
                for (int ch = tr.first_child[nb + node]; ch >= 0; ch = tr.next_sibling[nb + ch]) {
                    const double x = tr.value[nb + ch] + c.temperature * bonus[tr.count[nb + ch]];
                    if (x > best) { best = x; ties = 1; } else if (x == best) ++ties;
                }
                if (ties == 0) { error = ERR_NO_ACTION; break; }       // no child to select
                int pick = (int)rng.integers((uint32_t)ties);           // draws only for two or more ties
                for (int ch = tr.first_child[nb + node]; ch >= 0; ch = tr.next_sibling[nb + ch]) {
                    const double x = tr.value[nb + ch] + c.temperature * bonus[tr.count[nb + ch]];
                    if (x == best && pick-- == 0) { chance = ch; break; }
                }
                action = tr.key[nb + chance];
            }
            double r;
            env.step(a.model, action, li, gmask, true, term, trunc, r, bad_row);
            if (bad_row >= 0) { error = ERR_BAD_ROW; break; }
            ++steps;
            // ChanceNode.get_child (:171-182)
            const int key = c.closed_loop ? obs_key(env, c) : c.open_key;
            int n_states = 0, lastk = -1, child = -1;
            for (int ch = tr.first_child[nb + chance]; ch >= 0; ch = tr.next_sibling[nb + ch]) {
                if (tr.key[nb + ch] == key) { child = ch; break; }
                ++n_states;
                lastk = ch;
            }
            if (child < 0) {
                if (n_states <= c.state_widen[tr.count[nb + chance]]) {
                    child = n_nodes++;                                  // expand(obs_id)
                    if (writer) new_node(tr, nb, child, chance, lastk, KIND_DECISION, key);
                    __syncwarp(gmask);
                } else {
                    // choice(list(children)): an existing child; the env keeps the state it sampled
                    if (n_states == 0) { error = ERR_NO_STATE; break; }
                    int pick = (int)rng.integers((uint32_t)n_states);
                    for (child = tr.first_child[nb + chance]; pick-- > 0;) child = tr.next_sibling[nb + child];
                }
            }
            node = child;
            total = total + c.gamma_pow[depth] * r;                      // :82
            ++depth;
        }
        if (error) break;
        if (!term) {
            // MCTS.evaluate (mcts.py:160-177): choice(actions, 1, p) of the rollout policy, as mcts.cu draws it
            for (int h = depth; h < H; ++h) {
                const int amask = env.avail(A, gmask);
                const int pm = c.rollout_policy != 1 ? amask : (1 << A) - 1;
                const int n = __popc(pm);
                const double u = rng.random();
                const double* cdf = c.rollout_policy == 2
                    ? c.pref_cdf + ((int64_t)n * (A + 1) + Env::rank_of(pm, c.rollout_pref_action) + 1) * A
                    : c.uniform_cdf + (int64_t)n * A;
                int idx = 0;
                for (int i = 0; i < n; ++i) idx += cdf[i] <= u ? 1 : 0;   // searchsorted(side='right')
                idx = min(idx, n - 1);
                const int action = c.rollout_policy != 1 ? Env::nth(pm, idx) : idx;
                double r;
                env.step(a.model, action, li, gmask, true, term, trunc, r, bad_row);
            if (bad_row >= 0) { error = ERR_BAD_ROW; break; }
                ++steps;
                total = total + c.gamma_pow[h] * r;
                if (term || trunc) break;
            }
            if (error) break;
        }
        if (writer) {                                                     // backup_to_root / update (mcts.py:248-255)
            for (int n = node; n >= 0; n = tr.parent[nb + n]) {
                const int cnt = tr.count[nb + n] + 1;
                const double v = tr.value[nb + n];
                tr.count[nb + n] = cnt;
                tr.value[nb + n] = v + 1.0 / (double)cnt * (total - v);
            }
        }
        __syncwarp(gmask);
        ++runs;
    }

    if (writer) {
        int action = -1;
        if (!error) {
            // get_plan: root.selection_rule (mcts.py:212-218), the first highest value among the most visited children
            int best = -1, bc = 0;
            double bv = 0.0;
            for (int ch = tr.first_child[nb]; ch >= 0; ch = tr.next_sibling[nb + ch]) {
                const int cnt = tr.count[nb + ch];
                const double v = tr.value[nb + ch];
                if (best < 0 || cnt > bc || (cnt == bc && v > bv)) { best = ch; bc = cnt; bv = v; }
            }
            action = best >= 0 ? tr.key[nb + best] : -1;
        }
        rng.store(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
        a.plan[tree] = (int8_t)action;
        int32_t* res = a.result + (int64_t)tree * B2_MCTS_DPW_RESULT_WORDS;
        res[0] = n_nodes;
        res[1] = runs;
        res[2] = steps;
        res[3] = action;
        res[4] = error;
        res[5] = error == ERR_BAD_ROW ? bad_row : -1;
        res[6] = 0;
        res[7] = 0;
    }
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" int b2_mcts_dpw_plan(const b2_mcts_dpw_config* cfg, const int32_t* root_states, const b2_mcts_dpw_tree* tree,
                                uint64_t* rng, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_states && tree && rng && plan && result, "null pointer");
    B2_REQUIRE(tree->parent && tree->first_child && tree->next_sibling && tree->count && tree->kind && tree->key &&
               tree->value, "tree arrays missing");
    B2_REQUIRE(cfg->n_trees > 0, "bad batch");
    // episodes < 1 or horizon < 1 leave the root childless (the reference's get_plan returns None)
    B2_REQUIRE(cfg->episodes >= 1 && cfg->horizon >= 1, "episodes and horizon must be >= 1");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions <= MAX_ACTIONS_DPW, "n_actions must be in 1..8");
    B2_REQUIRE((int64_t)cfg->node_capacity >= 1 + 2 * (int64_t)cfg->episodes, "node_capacity too small");
    B2_REQUIRE(cfg->gamma_pow && cfg->uniform_cdf && cfg->action_widen && cfg->state_widen && cfg->bonus,
               "gamma / cdf / widening / bonus tables missing");
    B2_REQUIRE(cfg->rollout_policy >= 0 && cfg->rollout_policy <= 2,
               "rollout_policy must be 0 (random_available), 1 (random) or 2 (preference)");
    B2_REQUIRE(cfg->rollout_policy != 2 || cfg->pref_cdf, "preference policy table missing");
    const int rc = check_env_kind(cfg->env_kind, cfg->n_actions);
    if (rc != B2_OK) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    DpwArgs a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.rng = rng; a.plan = plan; a.result = result;
    a.model = LaneModel{b2_finite_mdp{}, cfg->mdp, cfg->terminal, cfg->env_draws};
    if (cfg->env_kind == B2_ENV_FINITE) {
        if (check_sampled_mdp(cfg->mdp, cfg->n_actions, cfg->terminal, true) != B2_OK) return B2_ERR_INVALID;
        B2_REQUIRE(!cfg->closed_loop || cfg->obs_keys, "observation key table missing");
        mcts_dpw_kernel<SampledFiniteEnv><<<lane_grid<SampledFiniteEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    } else {
        mcts_dpw_kernel<HighwayEnv><<<lane_grid<HighwayEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    }
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
