// MCTS / UCT -- the plan() loop of rl_agents/agents/tree_search/mcts.py for a
// BATCH of independent decisions.  Episodes inside one tree stay strictly
// sequential (every episode reads the statistics the previous one wrote) and
// consume that tree's numpy PCG64 stream exactly as the reference does, so
// tree indices, visit counts and values are bit-identical; the batch dimension
// (thousands of trees / root-parallel replicas) is what fills the GPU.
//
// One tree per lane group: 16 lanes for HighwayLite and IntersectionLite (lane = vehicle slot, the
// scene lives in registers and is "deep-copied" from the root once per episode,
// mcts.py:183), 1 lane for finite MDPs.  Tree bookkeeping is group-uniform
// scalar code; lane 0 of the group performs the stores.
//
// SampledFiniteEnv (b2_mcts_plan_sampled) steps a finite MDP in any mode as FiniteMDPEnv.step does.  The reference
// never reseeds its env copies, so every episode's deep copy starts from the live env's generator: each episode loads
// the tree's env words, and step k of every episode draws the k-th double of that one stream.  Only the steps the
// reference takes draw or check a row; a reached row Generator.choice rejects stops its own tree.
#include "common.cuh"
#include "lane_env.cuh"
#include "pcg64.cuh"

namespace b2 {

constexpr int MAX_BRANCH_MCTS = 8;
constexpr int ERR_BAD_ROW = 1;

struct MctsArgs {
    b2_mcts_config cfg;
    b2_mcts_tree tree;
    const int32_t* root_states;
    uint64_t* rng;
    int8_t* plan;
    int32_t* result;
    const uint64_t* env_rng;   // SampledFiniteEnv: the env generator's words of each tree
    LaneModel model;
};

// --------------------------------------------------------------- kernel ---
#ifndef B2_MCTS_MIN_BLOCKS
#define B2_MCTS_MIN_BLOCKS 8   // 64 registers, 32 warps/SM
#endif
template <class Env>
__global__ void __launch_bounds__(128, B2_MCTS_MIN_BLOCKS) mcts_kernel(MctsArgs a) {
    B2_LANE_MAP(Env, a.cfg.n_trees);
    const int A = a.cfg.n_actions, H = a.cfg.horizon;
    const int64_t nb = (int64_t)tree * a.cfg.node_capacity;
    const b2_mcts_tree& tr = a.tree;

    Pcg64 rng;
    rng.load(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
    const int resume = a.cfg.resume_nodes ? a.cfg.resume_nodes[tree] : 0;
    if (writer && resume <= 0) {   // MCTSNode(parent=None) (mcts.py:129-130, :207-210)
        tr.parent[nb] = -1; tr.first_child[nb] = -1; tr.count[nb] = 0; tr.meta[nb] = 0xff;
        tr.value[nb] = 0.0; tr.prior[nb] = 1.0;
    }
    __syncwarp(gmask);
    int n_nodes = resume > 0 ? resume : 1, env_steps = 0;   // resume: a re-rooted sub-tree is already in place
    int error = 0, bad_row = -1;

    for (int ep = 0; ep < a.cfg.episodes; ++ep) {
        if (error) break;
        Env env;
        env.load_root(a.root_states, tree, li);     // safe_deepcopy_env(state), mcts.py:183
        env.load_rng(a.env_rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
        int node = 0;
        bool in_sel = true, active = live;
        double total = 0.0;
        for (int h = 0; h < H; ++h) {
            // the 16 lanes of a group leave the episode together (terminal / truncated); the
            // other half of the warp keeps stepping its own scene under its half mask
            if (!active) break;
            // what a group that left its episode steps (the result is dropped): IDLE, action 1 on HighwayLite and
            // IntersectionLite alike (il::A_IDLE == hw::A_IDLE), always available there
            int action = hw::A_IDLE < A ? hw::A_IDLE : 0, child = -1;
            const int amask = env.avail(a.cfg.n_actions, gmask);
            if (active && in_sel && tr.first_child[nb + node] < 0) {
                // expansion (mcts.py:151-154, :237-246): children for the policy's actions
                const int pm = a.cfg.prior_policy != 1 ? amask : (1 << A) - 1;
                const int n = __popc(pm);
                if (writer) {
                    const double p = 1.0 / (double)n;
                    const double* pt = nullptr;       // preference_policy (:76-97): host-made probabilities
                    if (a.cfg.prior_policy == 2)
                        pt = a.cfg.pref_prior + ((int64_t)n * (A + 1) + Env::rank_of(pm, a.cfg.prior_pref_action) + 1) * A;
                    for (int i = 0; i < n; ++i) {
                        const int c = n_nodes + i;
                        tr.parent[nb + c] = node; tr.first_child[nb + c] = -1; tr.count[nb + c] = 0;
                        tr.meta[nb + c] = a.cfg.prior_policy != 1 ? Env::nth(pm, i) : i;
                        tr.value[nb + c] = 0.0; tr.prior[nb + c] = pt ? pt[i] : p;
                    }
                    tr.first_child[nb + node] = n_nodes;
                    tr.meta[nb + node] = (tr.meta[nb + node] & 0xff) | (n << 8);
                }
                n_nodes += n;
                in_sel = false;
                __syncwarp(gmask);
            }
            if (active) {
                if (in_sel) {
                    // sampling_rule / selection_strategy (mcts.py:220-235, :275-286)
                    const int fc = tr.first_child[nb + node];
                    const int n = (tr.meta[nb + node] >> 8) & 0xff;
                    double best = -INFINITY;
                    int ties = 0;
                    double sc[MAX_BRANCH_MCTS];
#pragma unroll
                    for (int i = 0; i < MAX_BRANCH_MCTS; ++i) {
                        if (i < n) {
                            const double v = tr.value[nb + fc + i];
                            const double p = tr.prior[nb + fc + i];
                            const int cnt = tr.count[nb + fc + i];
                            sc[i] = v + a.cfg.temperature * (double)n * p / (double)(cnt + 1);
                            if (sc[i] > best) { best = sc[i]; ties = 1; }
                            else if (sc[i] == best) ++ties;
                        }
                    }
                    int pick = (int)rng.integers((uint32_t)ties);   // random_argmax
                    int sel = 0;
#pragma unroll
                    for (int i = 0; i < MAX_BRANCH_MCTS; ++i) {
                        if (i < n && sc[i] == best) {
                            if (pick == 0) sel = i;
                            --pick;
                        }
                    }
                    child = fc + sel;
                    action = tr.meta[nb + child] & 0xff;
                } else {
                    // rollout policy (mcts.py:171-172): choice(actions, 1, p)
                    const int pm = a.cfg.rollout_policy != 1 ? amask : (1 << A) - 1;
                    const int n = __popc(pm);
                    const double u = rng.random();
                    const double* cdf = a.cfg.rollout_policy == 2
                        ? a.cfg.pref_cdf + ((int64_t)n * (A + 1) + Env::rank_of(pm, a.cfg.rollout_pref_action) + 1) * A
                        : a.cfg.uniform_cdf + (int64_t)n * A;
                    int idx = 0;
                    for (int i = 0; i < n; ++i) idx += cdf[i] <= u ? 1 : 0;   // searchsorted(side='right')
                    idx = min(idx, n - 1);
                    action = a.cfg.rollout_policy != 1 ? Env::nth(pm, idx) : idx;
                }
            }
            bool term, trunc;
            Env next = env;
            double r;
            if (!next.step(a.model, action, li, gmask, active, term, trunc, r, bad_row)) {
                error = ERR_BAD_ROW;
                active = false;
            }
            if (active) {
                env = next;
                ++env_steps;
                total += a.cfg.gamma_pow[h] * r;          // mcts.py:146,174
                if (in_sel) {
                    node = child;
                    if (term) active = false;              // :141 loop exit, no expansion, no rollout
                } else if (term || trunc) {
                    active = false;                        // :175
                }
            }
        }
        // update_branch (mcts.py:257-265)
        if (writer && !error) {
            int n = node;
            while (n >= 0) {
                const int c = tr.count[nb + n] + 1;
                const double v = tr.value[nb + n];
                tr.count[nb + n] = c;
                tr.value[nb + n] = v + 1.0 / (double)c * (total - v);
                n = tr.parent[nb + n];
            }
        }
        __syncwarp(gmask);
    }

    if (writer) {
        rng.store(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
        // get_plan with MCTSNode.selection_rule (mcts.py:212-218)
        int8_t* plan = a.plan + (int64_t)tree * a.cfg.horizon;
        int node = 0, len = 0;
        while (tr.first_child[nb + node] >= 0) {
            const int fc = tr.first_child[nb + node];
            const int n = (tr.meta[nb + node] >> 8) & 0xff;
            int best = 0;
            for (int i = 1; i < n; ++i) {
                const int ci = tr.count[nb + fc + i], cb = tr.count[nb + fc + best];
                if (ci > cb || (ci == cb && tr.value[nb + fc + i] > tr.value[nb + fc + best])) best = i;
            }
            if (len < a.cfg.horizon) plan[len] = (int8_t)(tr.meta[nb + fc + best] & 0xff);
            ++len;
            node = fc + best;
        }
        int32_t* res = a.result + (int64_t)tree * B2_MCTS_RESULT_WORDS;
        res[0] = n_nodes;
        res[1] = len;
        res[2] = env_steps;
        if constexpr (kSampled<Env>) { res[3] = error; res[4] = bad_row; }
    }
}

}  // namespace b2

using namespace b2;

static int check_mcts_config(const b2_mcts_config* cfg) {
    B2_REQUIRE(cfg->n_trees > 0 && cfg->episodes >= 0 && cfg->horizon >= 0, "bad batch / budget");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions <= MAX_BRANCH_MCTS, "n_actions must be in 1..8");
    B2_REQUIRE((int64_t)cfg->node_capacity >= 1 + (int64_t)cfg->episodes * cfg->n_actions, "node_capacity too small");
    B2_REQUIRE(cfg->gamma_pow && cfg->uniform_cdf, "gamma / cdf tables missing");
    B2_REQUIRE(cfg->rollout_policy >= 0 && cfg->rollout_policy <= 2 && cfg->prior_policy >= 0 && cfg->prior_policy <= 2,
               "policy must be 0 (random_available), 1 (random) or 2 (preference)");
    B2_REQUIRE((cfg->prior_policy != 2 || cfg->pref_prior) && (cfg->rollout_policy != 2 || cfg->pref_cdf),
               "preference policy tables missing");
    return B2_OK;
}

extern "C" int b2_mcts_plan(const b2_mcts_config* cfg, const int32_t* root_states, const b2_mcts_tree* tree,
                            uint64_t* rng, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_states && tree && rng && plan && result, "null pointer");
    if (check_mcts_config(cfg) != B2_OK) return B2_ERR_INVALID;
    const int rc = check_lane_env_il(cfg->env_kind, cfg->n_actions, cfg->mdp);
    if (rc != B2_OK) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    MctsArgs a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.rng = rng; a.plan = plan; a.result = result;
    a.model = LaneModel{cfg->mdp};
    if (cfg->env_kind == B2_ENV_FINITE)
        mcts_kernel<FiniteEnv><<<lane_grid<FiniteEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    else if (cfg->env_kind == B2_ENV_HIGHWAY)
        mcts_kernel<HighwayEnv><<<lane_grid<HighwayEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    else
        mcts_kernel<IntersectionEnv><<<lane_grid<IntersectionEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_mcts_plan_sampled(const b2_mcts_config* cfg, const b2_finite_mdp_sampled* mdp, const uint8_t* terminal,
                                    int32_t env_draws, const uint64_t* env_rng, const int32_t* root_states,
                                    const b2_mcts_tree* tree, uint64_t* rng, int8_t* plan, int32_t* result,
                                    void* stream_) {
    B2_REQUIRE(cfg && mdp && env_rng && root_states && tree && rng && plan && result, "null pointer");
    if (check_mcts_config(cfg) != B2_OK) return B2_ERR_INVALID;
    if (check_sampled_entry(cfg->env_kind, *mdp, cfg->n_actions, terminal, env_draws) != B2_OK) return B2_ERR_INVALID;
    cudaStream_t stream = (cudaStream_t)stream_;
    MctsArgs a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.rng = rng; a.plan = plan; a.result = result;
    a.env_rng = env_rng; a.model = LaneModel{b2_finite_mdp{}, *mdp, terminal, env_draws};
    mcts_kernel<SampledFiniteEnv><<<lane_grid<SampledFiniteEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
