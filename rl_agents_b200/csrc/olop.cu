// OLOP / KL-OLOP -- the plan() loop of rl_agents/agents/tree_search/olop.py for
// a BATCH of independent decisions, strict episode order inside each tree, the
// planner's numpy PCG64 stream consumed exactly as the reference does
// (`np_random.randint(2**30)` per episode, olop.py:73; `choice(children)` for the
// "uniform" continuation, :80-81).  The KL upper confidence bound
// (rl_agents/utils.py:123-203: damped Newton iteration on the Bernoulli KL,
// kl_bound.cuh) runs in-kernel in fp64.
//
// Same lane-group mapping as mcts.cu: one tree per 16-lane group (HighwayLite and
// IntersectionLite, lane = vehicle slot) or per lane (finite MDP).
//
// SampledFiniteEnv (b2_olop_plan_sampled) steps a finite MDP in any mode as
// FiniteMDPEnv.step does: each episode seeds the env copy's generator with the
// default_rng(seed) of its randint(2**30) draw, and every one of the `horizon`
// steps draws once with Generator.choice, also after a terminal state.  The
// tree stays open-loop (keyed on action sequences), so only its statistics and
// the plan depend on the draws.
#include "common.cuh"
#include "kl_bound.cuh"
#include "lane_env.cuh"
#include "pcg64.cuh"

namespace b2 {

constexpr int ERR_BAD_ROW = 3;

struct OlopArgs {
    b2_olop_config cfg;
    b2_olop_tree tree;
    const int32_t* root_states;
    uint64_t* rng;
    int8_t* plan;
    int32_t* result;
    LaneModel model;
};

template <class Env>
__global__ void __launch_bounds__(128, 8) olop_kernel(OlopArgs a) {
    B2_LANE_MAP(Env, a.cfg.n_trees);
    const int L = a.cfg.horizon;
    const int64_t nb = (int64_t)tree * a.cfg.node_capacity;
    const b2_olop_tree& tr = a.tree;
    const double gamma = a.cfg.gamma;

    Pcg64 rng;
    rng.load(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
    if (writer) {   // OLOPNode(parent=None) (olop.py:106-124)
        tr.parent[nb] = -1; tr.first_child[nb] = -1; tr.count[nb] = 0; tr.meta[nb] = 0xff;
        tr.cumulative[nb] = 0.0; tr.mu_ucb[nb] = a.cfg.kl ? 1.0 : INFINITY; tr.upper[nb] = a.cfg.init_upper[0];
    }
    __syncwarp(gmask);
    int n_nodes = 1, error = 0, bad_row = -1;

    for (int ep = 0; ep < a.cfg.episodes; ++ep) {
        Env env;
        env.load_root(a.root_states, tree, li);     // safe_deepcopy_env(state), olop.py:98
        if (live) env.seed(a.model, rng.integers(1u << 30));    // state.seed(np_random.randint(2**30)), :73
        int node = 0;
        const double threshold = a.cfg.thresholds[ep];
        for (int h = 0; h < L; ++h) {
            int action = 0, child = 0;
            const int amask = env.avail(a.cfg.n_actions, gmask);
            if (live && !error) {
                int fc = tr.first_child[nb + node];
                if (fc < 0) {
                    // expand (olop.py:165-180): one child per available action
                    const int n = __popc(amask);
                    if (writer) {
                        for (int i = 0; i < n; ++i) {
                            const int c = n_nodes + i;
                            tr.parent[nb + c] = node; tr.first_child[nb + c] = -1; tr.count[nb + c] = 0;
                            tr.meta[nb + c] = Env::nth(amask, i);
                            tr.cumulative[nb + c] = 0.0; tr.mu_ucb[nb + c] = a.cfg.kl ? 1.0 : INFINITY;
                            tr.upper[nb + c] = a.cfg.init_upper[h + 1];
                        }
                        tr.first_child[nb + node] = n_nodes;
                        tr.meta[nb + node] = (tr.meta[nb + node] & ~0xff00) | (n << 8);
                    }
                    fc = n_nodes;
                    n_nodes += n;
                    __syncwarp(gmask);
                    if (a.cfg.continuation == 1) {           // "uniform": np_random.choice(children keys)
                        child = fc + (int)rng.integers((uint32_t)n);
                    } else {                                 // "zeros": children[0] -- KeyError when unavailable
                        child = -1;
                        for (int i = 0; i < n; ++i)
                            if (Env::nth(amask, i) == 0) child = fc + i;
                        if (child < 0) { error = 2; child = fc; }
                    }
                } else {
                    // UCB elsewhere: first arg-max of value_upper (olop.py:84)
                    const int n = (tr.meta[nb + node] >> 8) & 0xff;
                    child = fc;
                    double best = tr.upper[nb + fc];
                    for (int i = 1; i < n; ++i) {
                        const double u = tr.upper[nb + fc + i];
                        if (u > best) { best = u; child = fc + i; }
                    }
                }
                action = tr.meta[nb + child] & 0xff;
            }
            bool term, trunc;
            double r;                                                                   // olop.py:87
            if (!env.step(a.model, action, li, gmask, live && !error, term, trunc, r, bad_row)) error = ERR_BAD_ROW;
            if (live && !error) {
                node = child;
                // update (olop.py:132-142)
                if (!(r >= 0.0 && r <= 1.0)) error = 1;
                if (writer) {
                    int meta = tr.meta[nb + node];
                    if (term) meta |= 1 << 16;
                    const double rr = (meta >> 16) & 1 ? 0.0 : r;
                    const double cum = tr.cumulative[nb + node] + rr;
                    const int cnt = tr.count[nb + node] + 1;
                    tr.meta[nb + node] = meta;
                    tr.cumulative[nb + node] = cum;
                    tr.count[nb + node] = cnt;
                    if (a.cfg.kl) tr.mu_ucb[nb + node] = kl_upper_bound(cum, cnt, threshold);   // :144-163
                }
                __syncwarp(gmask);
            }
        }
        // backup_to_root (olop.py:182-193)
        if (writer && !error) {
            int n = node;
            while (n >= 0) {
                const int fc = tr.first_child[nb + n];
                if (fc >= 0) {
                    const int k = (tr.meta[nb + n] >> 8) & 0xff;
                    double m = tr.upper[nb + fc];
                    for (int i = 1; i < k; ++i) {
                        const double u = tr.upper[nb + fc + i];
                        m = u > m ? u : m;
                    }
                    tr.upper[nb + n] = tr.mu_ucb[nb + n] + gamma * m;
                } else {
                    tr.upper[nb + n] = tr.mu_ucb[nb + n];
                }
                n = tr.parent[nb + n];
            }
        }
        __syncwarp(gmask);
    }

    if (writer) {
        rng.store(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
        // get_plan with OLOPNode.selection_rule (olop.py:126-130)
        int8_t* plan = a.plan + (int64_t)tree * max(L, 1);
        int node = 0, len = 0;
        while (tr.first_child[nb + node] >= 0) {
            const int fc = tr.first_child[nb + node];
            const int n = (tr.meta[nb + node] >> 8) & 0xff;
            int best = 0;
            for (int i = 1; i < n; ++i) {
                const int ci = tr.count[nb + fc + i], cb = tr.count[nb + fc + best];
                if (ci > cb || (ci == cb && tr.upper[nb + fc + i] > tr.upper[nb + fc + best])) best = i;
            }
            if (len < L) plan[len] = (int8_t)(tr.meta[nb + fc + best] & 0xff);
            ++len;
            node = fc + best;
        }
        int32_t* res = a.result + (int64_t)tree * B2_OLOP_RESULT_WORDS;
        res[0] = n_nodes;
        res[1] = len;
        res[2] = error;
        if constexpr (kSampled<Env>) res[3] = bad_row;
    }
}

}  // namespace b2

using namespace b2;

static int check_olop_config(const b2_olop_config* cfg) {
    B2_REQUIRE(cfg->n_trees > 0 && cfg->episodes >= 0 && cfg->horizon >= 1, "bad batch / budget");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions <= 8, "n_actions must be in 1..8");
    B2_REQUIRE((int64_t)cfg->node_capacity >= 1 + (int64_t)cfg->episodes * cfg->horizon * cfg->n_actions,
               "node_capacity too small");
    B2_REQUIRE(cfg->thresholds && cfg->init_upper, "threshold / initial bound tables missing");
    return B2_OK;
}

extern "C" int b2_olop_plan(const b2_olop_config* cfg, const int32_t* root_states, const b2_olop_tree* tree,
                            uint64_t* rng, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_states && tree && rng && plan && result, "null pointer");
    if (check_olop_config(cfg) != B2_OK) return B2_ERR_INVALID;
    const int rc = check_lane_env_il(cfg->env_kind, cfg->n_actions, cfg->mdp);
    if (rc != B2_OK) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    OlopArgs a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.rng = rng; a.plan = plan; a.result = result;
    a.model = LaneModel{cfg->mdp};
    if (cfg->env_kind == B2_ENV_FINITE)
        olop_kernel<FiniteEnv><<<lane_grid<FiniteEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    else if (cfg->env_kind == B2_ENV_HIGHWAY)
        olop_kernel<HighwayEnv><<<lane_grid<HighwayEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    else
        olop_kernel<IntersectionEnv><<<lane_grid<IntersectionEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_olop_plan_sampled(const b2_olop_config* cfg, const b2_finite_mdp_sampled* mdp,
                                    const uint8_t* terminal, int32_t env_draws, const int32_t* root_states,
                                    const b2_olop_tree* tree, uint64_t* rng, int8_t* plan, int32_t* result,
                                    void* stream_) {
    B2_REQUIRE(cfg && mdp && terminal && root_states && tree && rng && plan && result, "null pointer");
    if (check_olop_config(cfg) != B2_OK) return B2_ERR_INVALID;
    if (check_sampled_entry(cfg->env_kind, *mdp, cfg->n_actions, terminal, env_draws) != B2_OK) return B2_ERR_INVALID;
    cudaStream_t stream = (cudaStream_t)stream_;
    OlopArgs a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.rng = rng; a.plan = plan; a.result = result;
    a.model = LaneModel{b2_finite_mdp{}, *mdp, terminal, env_draws};
    olop_kernel<SampledFiniteEnv><<<lane_grid<SampledFiniteEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
