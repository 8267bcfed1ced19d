// BRUE -- the plan() loop of rl_agents/agents/tree_search/brue.py for a BATCH of independent decisions.  Strict
// rollout order inside each tree; the planner's numpy PCG64 stream is consumed exactly as the reference does:
// `np_random.randint(2**30)` to seed the env copy and `randint(action_space.n)` per step (:25-27), then, in the
// reverse update, one `random()` per level estimate() walks (`np_random.choice(next_states, p=...)` draws one
// double even over a single next state, :62), and `choice(indices)` for a tie of the root recommendation
// (random_argmax, abstract.py:304-311).
//
// The statistics are incremental means ((count-1)/count * v + x/count, one IEEE op per Python op; the library builds
// with -fmad=false), host gamma**d products and first-maximum arg-maxes, so every fp64 field equals the reference's
// bit for bit.
//
// Same lane-group mapping as mdp_gape.cu: one tree per 16-lane group (HighwayLite, lane = vehicle slot) or per lane
// (finite MDP).  Every lane of a group holds a copy of the tree's RNG and draws the rollout actions itself; only
// lane 0 touches the tree.  It runs the reverse update alone, and the group then takes its RNG position.  A tree
// whose budget is spent leaves its loop; hw::step only synchronises the 16 lanes of one group, so the other tree
// of the warp carries on.
#include "common.cuh"
#include "lane_env.cuh"
#include "pcg64.cuh"

namespace b2 {
namespace {

constexpr int KIND_DECISION = 0, KIND_CHANCE = 1, NO_ACTION = 0xff;

struct BrueArgs {
    b2_brue_config cfg;
    b2_brue_tree tree;
    const int32_t* root_states;
    uint64_t* rng;
    int8_t* plan;
    int32_t* result;
    LaneModel model;
};

__device__ __forceinline__ void new_node(const b2_brue_tree& tr, int64_t nb, int id, int parent, int action, int kind) {
    tr.parent[nb + id] = parent; tr.first_child[nb + id] = -1; tr.next_sibling[nb + id] = -1; tr.count[nb + id] = 0;
    tr.meta[nb + id] = action | (kind << 8);
    tr.value[nb + id] = 0.0;
}

// DecisionNode.update / ChanceNode.update (:84-86, :106-108): (count - 1) / count * v + x / count
__device__ __forceinline__ void update(const b2_brue_tree& tr, int64_t nb, int id, double x) {
    const int c = tr.count[nb + id] + 1;
    tr.count[nb + id] = c;
    const double dc = (double)c;
    tr.value[nb + id] = (double)(c - 1) / dc * tr.value[nb + id] + x / dc;
}

// BRUE.estimate (:52-64) below decision node `node`, at most `levels` levels: the first maximum of the chance
// children's value in creation order, one random() for the choice of the (single) next state, its reward discounted
__device__ double estimate(const b2_brue_tree& tr, int64_t nb, int node, int levels, const double* gamma_pow,
                           Pcg64& rng) {
    double ret = 0.0;
    for (int d = 0; d < levels; ++d) {
        int c = tr.first_child[nb + node];
        if (c < 0) break;
        int best = c;
        double bv = tr.value[nb + c];
        for (c = tr.next_sibling[nb + c]; c >= 0; c = tr.next_sibling[nb + c]) {
            const double v = tr.value[nb + c];
            if (v > bv) { bv = v; best = c; }
        }
        rng.random();
        node = tr.first_child[nb + best];
        ret = ret + gamma_pow[d] * tr.value[nb + node];
    }
    return ret;
}

template <class Env>
__global__ void __launch_bounds__(128, 8) brue_kernel(BrueArgs a) {
    B2_LANE_MAP_LIVE(Env, a.cfg.n_trees);          // whole lane groups: no live lane of a group leaves
    const int H = a.cfg.horizon;
    const int64_t nb = (int64_t)tree * a.cfg.node_capacity;
    const b2_brue_tree& tr = a.tree;
    int32_t* path = tr.path + (int64_t)tree * H;
    double* path_reward = tr.path_reward + (int64_t)tree * H;

    Pcg64 rng;
    rng.load(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
    if (writer) new_node(tr, nb, 0, -1, NO_ACTION, KIND_DECISION);     // DecisionNode(parent=None)
    int n_nodes = 1, rollouts = 0, error = 0, budget = a.cfg.budget;   // n_nodes: lane 0 only

    while (budget > 0) {                            // BRUE.plan (:66-71)
        // a rollout creates at most 2 * horizon nodes; never short at the documented capacity
        if (writer) error = n_nodes + 2 * H > a.cfg.node_capacity;
        if (G > 1) error = __shfl_sync(gmask, error, 0, G);
        if (error) break;
        Env env;
        env.load_root(a.root_states, tree, li);      // safe_deepcopy_env(state), :69
        rng.integers(1u << 30);                      // state.seed(np_random.randint(2**30)), :25
        int node = 0, len = 0;
        for (int h = 0; h < H; ++h) {                // rollout (:24-33)
            const int action = (int)rng.integers((uint32_t)a.cfg.n_actions);
            bool term, trunc;
            double r;
            int bad_row;
            env.step(a.model, action, li, gmask, true, term, trunc, r, bad_row);
            if (writer) {                            // update's forward pass (:39-44)
                // DecisionNode.get_child: the chance child of this action, appended to the list on the first visit
                int c = tr.first_child[nb + node], last = -1;
                while (c >= 0 && (tr.meta[nb + c] & 0xff) != action) { last = c; c = tr.next_sibling[nb + c]; }
                if (c < 0) {
                    c = n_nodes++;
                    new_node(tr, nb, c, node, action, KIND_CHANCE);
                    if (last < 0) tr.first_child[nb + node] = c;
                    else tr.next_sibling[nb + last] = c;
                }
                // ChanceNode.get_child(str(obs)): a deterministic env model gives a chance node one next state
                int d = tr.first_child[nb + c];
                if (d < 0) {
                    d = n_nodes++;
                    new_node(tr, nb, d, c, NO_ACTION, KIND_DECISION);
                    tr.first_child[nb + c] = d;
                }
                path[h] = c;
                path_reward[h] = r;
                node = d;
            }
            ++len;
            --budget;                                // available_budget -= 1, also for the step that ends it
            if (term) break;
        }
        ++rollouts;
        if (writer) {                                // update's reverse pass (:46-50)
            for (int h = len - 1; h >= 0; --h) {
                const int c = path[h], d = tr.first_child[nb + c];
                const double r = path_reward[h];
                update(tr, nb, d, r);                                           // R(s, a, s')
                const double est = estimate(tr, nb, d, H - (h + 1), a.cfg.gamma_pow, rng);   // depth of d: h + 1
                update(tr, nb, c, r + a.cfg.gamma * est);
            }
        }
        if (G > 1) {                                 // random() leaves the buffered 32-bit half alone
            uint64_t hi = (uint64_t)(rng.state >> 64), lo = (uint64_t)rng.state;
            hi = __shfl_sync(gmask, (unsigned long long)hi, 0, G);
            lo = __shfl_sync(gmask, (unsigned long long)lo, 0, G);
            rng.state = ((unsigned __int128)hi << 64) | lo;
        }
    }

    if (writer) {
        int action = -1;
        if (!error) {                                // get_plan: root.selection_rule, random_argmax (:73-91)
            const int c0 = tr.first_child[nb];
            double m = tr.value[nb + c0];
            int ties = 1;
            for (int c = tr.next_sibling[nb + c0]; c >= 0; c = tr.next_sibling[nb + c]) {
                const double v = tr.value[nb + c];
                if (v > m) { m = v; ties = 1; } else if (v == m) ++ties;
            }
            int pick = (int)rng.integers((uint32_t)ties);                   // draws only for two or more ties
            for (int c = c0; c >= 0; c = tr.next_sibling[nb + c])
                if (tr.value[nb + c] == m && pick-- == 0) { action = tr.meta[nb + c] & 0xff; break; }
        }
        rng.store(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
        a.plan[tree] = (int8_t)action;
        int32_t* res = a.result + (int64_t)tree * B2_BRUE_RESULT_WORDS;
        res[0] = n_nodes;
        res[1] = rollouts;
        res[2] = a.cfg.budget - budget;
        res[3] = action;
        res[4] = error;
        res[5] = 0;
        res[6] = 0;
        res[7] = 0;
    }
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" int b2_brue_plan(const b2_brue_config* cfg, const int32_t* root_states, const b2_brue_tree* tree,
                            uint64_t* rng, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_states && tree && rng && plan && result, "null pointer");
    B2_REQUIRE(tree->path && tree->path_reward, "rollout path scratch missing");
    B2_REQUIRE(cfg->n_trees > 0, "bad batch");
    // budget < 1 leaves the root without children (the reference's get_plan raises); horizon < 1 never spends budget
    B2_REQUIRE(cfg->budget >= 1 && cfg->horizon >= 1, "budget and horizon must be >= 1");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions < NO_ACTION, "n_actions must be in 1..254");
    B2_REQUIRE((int64_t)cfg->node_capacity >= 1 + 2 * ((int64_t)cfg->budget + cfg->horizon - 1),
               "node_capacity too small");
    B2_REQUIRE(cfg->gamma_pow, "gamma**d table missing");
    const int rc = check_lane_env(cfg->env_kind, cfg->n_actions, cfg->mdp);
    if (rc != B2_OK) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    BrueArgs a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.rng = rng; a.plan = plan; a.result = result;
    a.model = LaneModel{cfg->mdp};
    if (cfg->env_kind == B2_ENV_FINITE)
        brue_kernel<FiniteEnv><<<lane_grid<FiniteEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    else
        brue_kernel<HighwayEnv><<<lane_grid<HighwayEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
