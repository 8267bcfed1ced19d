// MDP-GapE -- the plan() loop of rl_agents/agents/tree_search/mdp_gape.py for a BATCH of independent
// decisions.  Strict episode order inside each tree; the planner's numpy PCG64 stream is consumed exactly as
// the reference does (`np_random.randint(2**30)` per episode, :67; `randint(n_actions)` for the "uniform"
// continuation, :195; `choice(indices)` for ties of random_argmax, abstract.py:296-311).  The KL bounds of a
// decision node (utils.py:123-203, damped Newton on the Bernoulli KL, kl_bound.cuh -- the iteration OLOP uses) run
// in-kernel in fp64.
//
// The tree alternates decision nodes (value bounds, KL statistics of the reward received on arrival) and chance
// nodes (one per available action).  A chance node's children are max_next_states_count placeholders.  On the
// deterministic env models (FiniteEnv, HighwayEnv) only placeholder 0 is ever observed, and it is moved to the END
// of the chance node's child order (mdp_gape.py:272-286) -- the order in which the backup sums.  Then
// max_expectation_under_constraint (utils.py:292-342) sees a distribution with one positive element and needs
// no Newton solve: it is restated operation by operation in gape_expectation().
//
// SampledFiniteEnv steps a finite MDP in any mode with the episode's env generator default_rng(seed), one
// Generator.choice per step.  A chance node then observes up to max_next_states_count distinct next states, keyed
// by state id (keys[]): the i-th one takes placeholder i, so the dict order is the placeholders n .. K-1, then the
// observed 0 .. n-1.  Its backup runs max_expectation_under_constraint in full (gape_expectation_kl(), the Newton
// solve included).  The reference's 1-D dot products are sequential fused multiply-add chains from 0.0 (numpy's and
// numba's `@` on the host for lengths up to 15); the library builds with -fmad=false, so they are written with
// explicit fma() and every other operation stays unfused, in the reference's order.
//
// Same lane-group mapping as olop.cu: one tree per 16-lane group (HighwayLite, lane = vehicle slot) or per lane
// (finite MDP).  Every lane of a group holds a copy of the tree's RNG and takes every selection decision
// itself from the tree arrays; lane 0 writes the tree.  A tree whose stopping rule fired leaves its episode
// loop; hw::step only synchronises the 16 lanes of one group, so the other trees of the warp carry on.
#include "common.cuh"
#include "kl_bound.cuh"
#include "lane_env.cuh"
#include "pcg64.cuh"

namespace b2 {
namespace {

constexpr int KIND_DECISION = 0, KIND_CHANCE = 1;
constexpr int DONE_BIT = 1 << 16, KIND_SHIFT = 17;
constexpr int ERR_PLACEHOLDERS = 3, ERR_BAD_ROW = 4;

struct GapeArgs {
    b2_mdp_gape_config cfg;
    b2_mdp_gape_tree tree;
    const int32_t* root_states;
    uint64_t* rng;
    int8_t* plan;
    int32_t* result;
    int32_t* keys;             // SampledFiniteEnv: the state id each decision node was observed under
    LaneModel model;
};

// ChanceNode.backup_to_root (mdp_gape.py:288-305) for one side: with f = u_next (upper) or -l_next (lower),
// p = max_expectation_under_constraint(f, p_hat, c) and the bound is p @ (u_next | l_next).  Children in the
// reference's dict order: the unobserved placeholders fc+1 .. fc+k-1, then the observed fc, whose p_hat is qp.
__device__ double gape_expectation(const b2_mdp_gape_tree& tr, int64_t nb, int fc, int k, bool upper_side,
                                   double gamma, double qp, double c) {
    auto value = [&](int id) {
        return upper_side ? tr.mu_ucb[nb + id] + gamma * tr.upper[nb + id] : tr.mu_lcb[nb + id] + gamma * tr.lower[nb + id];
    };
    const double fp = upper_side ? value(fc) : -value(fc);
    double f_star = fp, f_zero_max = -INFINITY;
    for (int i = 1; i < k; ++i) {
        const double f = upper_side ? value(fc + i) : -value(fc + i);
        f_star = f > f_star ? f : f_star;
        f_zero_max = f > f_zero_max ? f : f_zero_max;
    }
    // utils.py:317-323: move the mass z = 1 - exp(theta(f*)) to the best unobserved entries when theta(f*) < 0,
    // theta(l) = q_p @ log(l - f_p) + log(q_p @ (1 / (l - f_p))) - c (theta_func, :279-282)
    double z = 0.0, d = 0.0;
    bool moved = false;
    if (f_star > fp) {
        d = f_star - fp;
        const double theta = qp * log(d) + log(qp * (1.0 / d)) - c;
        if (theta < 0.0) {
            moved = true;
            z = 1.0 - exp(theta);
        }
    }
    double p_obs = qp, share = 0.0;
    if (moved) {
        int n_max = 0;
        for (int i = 1; i < k; ++i) n_max += (upper_side ? value(fc + i) : -value(fc + i)) == f_zero_max;
        share = z / (double)n_max;
        const double beta = (1.0 - z) / (qp * (1.0 / d));          // :335, lambda = f*
        p_obs = beta != 0.0 ? (beta * qp) / d : 0.0;               // :336-341 (no observed entry reaches f*)
    }
    // p @ next in the dict order
    double s = 0.0;
    for (int i = 1; i < k; ++i) {
        const double v = value(fc + i);
        const double p = moved ? (((upper_side ? v : -v) == f_zero_max) ? 1.0 : 0.0) * share : 0.0;
        s = s + p * v;
    }
    return s + p_obs * value(fc);
}

// ChanceNode.backup_to_root (mdp_gape.py:288-305) for one side, in full: f = u_next (upper) or -l_next (lower),
// p = max_expectation_under_constraint(f, p_hat, c) (utils.py:292-342) and the bound is p @ (u_next | l_next).
// The K children fc .. fc+K-1 hold the observed next states 0 .. n-1 (n >= 1, the positive entries of p_hat in the
// reference's order) and the unobserved placeholders n .. K-1, which come first in the dict order.
__device__ double gape_expectation_kl(const b2_mdp_gape_tree& tr, int64_t nb, int fc, int K, int n, bool upper_side,
                                      double gamma, int cnt, double c) {
    auto value = [&](int i) {
        const int64_t id = nb + fc + i;
        return upper_side ? tr.mu_ucb[id] + gamma * tr.upper[id] : tr.mu_lcb[id] + gamma * tr.lower[id];
    };
    auto f = [&](int i) { return upper_side ? value(i) : -value(i); };
    auto q = [&](int i) { return (double)tr.count[nb + fc + i] / (double)cnt; };
    // theta_func (:279-282): q_p @ log(l - f_p) + log(q_p @ (1 / (l - f_p))) - c
    auto theta = [&](double l) {
        double s1 = 0.0, s2 = 0.0;
        for (int i = 0; i < n; ++i) {
            const double d = l - f(i), qi = q(i);
            s1 = fma(qi, log(d), s1);
            s2 = fma(qi, 1.0 / d, s2);
        }
        return s1 + log(s2) - c;
    };
    double fp_max = f(0);
    for (int i = 1; i < n; ++i) {
        const double fi = f(i);
        fp_max = fi > fp_max ? fi : fp_max;
    }
    double f_star = fp_max;
    for (int i = n; i < K; ++i) {
        const double fi = f(i);
        f_star = fi > f_star ? fi : f_star;
    }
    double lambda = 0.0, z = 0.0, share = 0.0;
    bool moved = false, solved = false;
    if (f_star > fp_max) {                                   // :317-323: mass z to the best unobserved entries
        const double theta_star = theta(f_star);
        if (theta_star < 0.0) {
            moved = solved = true;
            lambda = f_star;
            z = 1.0 - exp(theta_star);
            int n_max = 0;
            for (int i = n; i < K; ++i) n_max += f(i) == f_star;
            share = z / (double)n_max;
        }
    }
    bool close = false;
    if (!solved) {
        // np.isclose(f_p, f_p[0]).all() (atol 1e-8, rtol 1e-5): p = q
        const double f0 = f(0);
        close = true;
        for (int i = 1; i < n; ++i) {
            const double fi = f(i);
            close = close && ((fabs(fi - f0) <= 1e-8 + 1e-5 * fabs(f0) && isfinite(f0)) || fi == f0);
        }
    }
    if (!solved && !close) {
        // newton_iteration(theta, d_theta_dl, 1e-2, x0=f_star + 1, a=f_star) (utils.py:150-203), weight 0.9
        double x = INFINITY, x_next = f_star + 1.0;
        for (int it = 0; fabs(x - x_next) > 1e-2 && it < 100; ++it) {
            x = x_next;
            const double f_x = theta(x);
            double s1 = 0.0, s2 = 0.0;                       // d_theta_dl_func (:285-289)
            for (int i = 0; i < n; ++i) {
                const double inv = 1.0 / (x - f(i)), qi = q(i);
                s1 = fma(qi, inv, s1);
                s2 = fma(qi, inv * inv, s2);
            }
            // numba's scalar division by zero raises ZeroDivisionError: the finite difference
            const double df_x = s1 != 0.0 ? s1 - s2 / s1 : (f_x - theta(x - 1e-2)) / 1e-2;
            if (df_x != 0.0) x_next = x - f_x / df_x;
            if (x_next < f_star) x_next = 0.9 * f_star + (1.0 - 0.9) * x;
        }
        lambda = x_next < f_star ? f_star : x_next;
    }
    double beta = 0.0;
    int n_uni = 0;
    if (!close) {                                            // :335: beta = (1 - z) / (q_p @ (1 / (lambda - f_p)))
        double sb = 0.0;
        for (int i = 0; i < n; ++i) sb = fma(q(i), 1.0 / (lambda - f(i)), sb);
        beta = (1.0 - z) / sb;
        if (beta == 0.0)                                     // :336-339
            for (int i = 0; i < n; ++i) n_uni += f(i) == f_star;
    }
    // p @ next in the dict order: placeholders n .. K-1, then the observed 0 .. n-1
    double s = 0.0;
    for (int j = 0; j < K; ++j) {
        const int i = j < K - n ? n + j : j - (K - n);
        double p;
        if (i >= n) p = moved && f(i) == f_star ? share : 0.0;
        else if (close) p = q(i);
        else if (beta == 0.0) p = f(i) == f_star ? (1.0 - z) / (double)n_uni : 0.0;
        else p = (beta * q(i)) / (lambda - f(i));
        s = fma(p, value(i), s);
    }
    return s;
}

// best_arm_identification_selection (mdp_gape.py:228-249) on the children fc .. fc+n-1 (n >= 2): UGapE's best
// (first minimum of the gap), challenger (first maximum of value_upper among the others) and the sampled arm
// (the wider interval of the two, best on a tie).  Node ids.
__device__ void bai(const b2_mdp_gape_tree& tr, int64_t nb, int fc, int n, int& sel, int& best, int& challenger) {
    int bi = 0;
    double best_gap = 0.0;
    for (int i = 0; i < n; ++i) {
        double g = -INFINITY;
        const double lo = tr.lower[nb + fc + i];
        for (int j = 0; j < n; ++j) {
            if (j == i) continue;
            const double x = tr.upper[nb + fc + j] - lo;
            if (x > g) g = x;
        }
        if (i == 0 || g < best_gap) { best_gap = g; bi = i; }
    }
    int ci = -1;
    double cu = 0.0;
    for (int j = 0; j < n; ++j) {
        if (j == bi) continue;
        const double u = tr.upper[nb + fc + j];
        if (ci < 0 || u > cu) { ci = j; cu = u; }
    }
    best = fc + bi;
    challenger = fc + ci;
    const double wb = tr.upper[nb + best] - tr.lower[nb + best];
    const double wc = tr.upper[nb + challenger] - tr.lower[nb + challenger];
    sel = wc > wb ? challenger : best;
}

__device__ __forceinline__ void new_node(const b2_mdp_gape_tree& tr, int64_t nb, int id, int parent, int label,
                                         int kind, double init_upper) {
    tr.parent[nb + id] = parent; tr.first_child[nb + id] = -1; tr.count[nb + id] = 0;
    tr.meta[nb + id] = label | (kind << KIND_SHIFT);
    tr.cumulative[nb + id] = 0.0; tr.mu_ucb[nb + id] = 1.0; tr.mu_lcb[nb + id] = 0.0;   // KL (mdp_gape.py:139-143)
    tr.upper[nb + id] = init_upper; tr.lower[nb + id] = 0.0;
}

template <class Env>
__global__ void __launch_bounds__(128, 8) mdp_gape_kernel(GapeArgs a) {
    B2_LANE_MAP_LIVE(Env, a.cfg.n_trees);          // whole lane groups: no live lane of a group leaves
    const int H = a.cfg.horizon, K = a.cfg.max_next_states;
    const int64_t nb = (int64_t)tree * a.cfg.node_capacity;
    const b2_mdp_gape_tree& tr = a.tree;
    const double gamma = a.cfg.gamma;

    Pcg64 rng;
    rng.load(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
    if (writer) new_node(tr, nb, 0, -1, 0xff, KIND_DECISION, a.cfg.init_upper[0]);    // DecisionNode(None)
    if constexpr (kSampled<Env>) { if (writer) a.keys[nb] = -1; }
    __syncwarp(gmask);
    int n_nodes = 1, error = 0, episode = 0, best = -1, challenger = -1, bad_row = -1;
    bool done = false;

    // expand a decision node (mdp_gape.py:162-170): one chance node per available action, env order
    auto expand_decision = [&](int node, int amask, int depth) {
        const int n = __popc(amask);
        if (writer) {
            for (int i = 0; i < n; ++i) new_node(tr, nb, n_nodes + i, node, Env::nth(amask, i), KIND_CHANCE,
                                                  a.cfg.init_upper[depth]);
            if constexpr (kSampled<Env>) { for (int i = 0; i < n; ++i) a.keys[nb + n_nodes + i] = -1; }
            tr.first_child[nb + node] = n_nodes;
            tr.meta[nb + node] = (tr.meta[nb + node] & ~0xff00) | (n << 8);
        }
        n_nodes += n;
        __syncwarp(gmask);
    };

    while (!done) {                                  // MDPGapE.plan (:94-110)
        Env env;
        env.load_root(a.root_states, tree, li);      // safe_deepcopy_env(state), :98
        env.seed(a.model, rng.integers(1u << 30));       // state.seed(np_random.randint(2**30)), :67
        if (tr.first_child[nb] < 0) expand_decision(0, env.avail(a.cfg.n_actions, gmask), 0);
        int node = 0;
        for (int h = 0; h < H; ++h) {
            const int amask = env.avail(a.cfg.n_actions, gmask);
            int fc = tr.first_child[nb + node];
            // sampling_rule (:183-198)
            int action;
            if (node == 0) {
                const int n = (tr.meta[nb] >> 8) & 0xff;
                if (n < 2) { error = 2; break; }     // max() of an empty challenger list: ValueError
                int sel;
                bai(tr, nb, fc, n, sel, best, challenger);
                action = tr.meta[nb + sel] & 0xff;
            } else if (fc >= 0) {                    // random_argmax of the chance children's value_upper
                const int n = (tr.meta[nb + node] >> 8) & 0xff;
                double m = tr.upper[nb + fc];
                int ties = 1;
                for (int i = 1; i < n; ++i) {
                    const double u = tr.upper[nb + fc + i];
                    if (u > m) { m = u; ties = 1; } else if (u == m) ++ties;
                }
                int pick = ties > 1 ? (int)rng.integers((uint32_t)ties) : 0;
                int child = fc;
                for (int i = 0; i < n; ++i)
                    if (tr.upper[nb + fc + i] == m && pick-- == 0) { child = fc + i; break; }
                action = tr.meta[nb + child] & 0xff;
            } else {                                 // leaf: "uniform" randint(n_actions) / "zeros" 0
                action = a.cfg.continuation == 1 ? (int)rng.integers((uint32_t)a.cfg.n_actions) : 0;
            }
            // get_child (:155-160): expand a leaf, fall back to the first available action
            if (fc < 0) {
                fc = n_nodes;
                expand_decision(node, amask, h);
            }
            const int n = (tr.meta[nb + node] >> 8) & 0xff;
            int chance = fc;
            for (int i = 0; i < n; ++i)
                if ((tr.meta[nb + fc + i] & 0xff) == action) { chance = fc + i; break; }
            action = tr.meta[nb + chance] & 0xff;
            bool term, trunc;
            double r;                                                                        // :82
            if (!env.step(a.model, action, li, gmask, true, term, trunc, r, bad_row)) {
                error = ERR_BAD_ROW;
                break;
            }
            // ChanceNode.get_child (:272-286): placeholders on the first visit; a deterministic env observes placeholder 0
            int child = tr.first_child[nb + chance];
            if (child < 0) {
                child = n_nodes;
                if (writer) {
                    for (int i = 0; i < K; ++i) new_node(tr, nb, n_nodes + i, chance, i, KIND_DECISION,
                                                          a.cfg.init_upper[h + 1]);
                    if constexpr (kSampled<Env>) { for (int i = 0; i < K; ++i) a.keys[nb + n_nodes + i] = -1; }
                    tr.first_child[nb + chance] = n_nodes;
                    tr.meta[nb + chance] = (tr.meta[nb + chance] & ~0xff00) | (K << 8);
                }
                n_nodes += K;
            }
            if constexpr (kSampled<Env>) {
                // the i-th distinct next state takes placeholder i: the observation's key, else the first free one;
                // none left is the reference's ValueError
                int i = 0;
                while (i < K && a.keys[nb + child + i] >= 0 && a.keys[nb + child + i] != env.s) ++i;
                if (i == K) { error = ERR_PLACEHOLDERS; break; }
                child += i;
                if (writer) a.keys[nb + child] = env.s;
            }
            if (!(r >= 0.0 && r <= 1.0)) { error = 1; break; }                 // olop.py:133-134
            if (writer) {
                tr.count[nb + chance] += 1;                                      // ChanceNode.update (:264-265)
                int meta = tr.meta[nb + child];                                  // OLOPNode.update (olop.py:132-142)
                if (term) meta |= DONE_BIT;
                const double rr = (meta & DONE_BIT) ? 0.0 : r;
                const double cum = tr.cumulative[nb + child] + rr;
                const int cnt = tr.count[nb + child] + 1;
                tr.meta[nb + child] = meta;
                tr.cumulative[nb + child] = cum;
                tr.count[nb + child] = cnt;
                const double thr = a.cfg.thresholds[cnt];                        // compute_reward_ucb (:200-212)
                tr.mu_ucb[nb + child] = kl_bound(cum, cnt, thr, false);
                tr.mu_lcb[nb + child] = kl_bound(cum, cnt, thr, true);
            }
            __syncwarp(gmask);
            node = child;
        }
        if (error) break;
        if (writer) {                                                            // backup_to_root
            int n = node;
            while (n >= 0) {
                const int meta = tr.meta[nb + n];
                const int fc = tr.first_child[nb + n];
                const int k = (meta >> 8) & 0xff;
                if (((meta >> KIND_SHIFT) & 1) == KIND_DECISION) {               // :214-226
                    double up = 0.0, lo = 0.0;                                   // a leaf (depth H): 0 / 0
                    if (fc >= 0) {
                        up = tr.upper[nb + fc];
                        lo = tr.lower[nb + fc];
                        for (int i = 1; i < k; ++i) {
                            const double u = tr.upper[nb + fc + i], l = tr.lower[nb + fc + i];
                            up = u > up ? u : up;
                            lo = l > lo ? l : lo;
                        }
                    }
                    tr.upper[nb + n] = up;
                    tr.lower[nb + n] = lo;
                } else if constexpr (kSampled<Env>) {                            // :288-305
                    const int cnt = tr.count[nb + n];
                    const double c = a.cfg.transition_thresholds[cnt] / (double)cnt;
                    int obs = 1;
                    while (obs < k && a.keys[nb + fc + obs] >= 0) ++obs;
                    tr.upper[nb + n] = gape_expectation_kl(tr, nb, fc, k, obs, true, gamma, cnt, c);
                    tr.lower[nb + n] = gape_expectation_kl(tr, nb, fc, k, obs, false, gamma, cnt, c);
                } else {
                    const int cnt = tr.count[nb + n];
                    const double qp = (double)tr.count[nb + fc] / (double)cnt;
                    const double c = a.cfg.transition_thresholds[cnt] / (double)cnt;
                    tr.upper[nb + n] = gape_expectation(tr, nb, fc, k, true, gamma, qp, c);
                    tr.lower[nb + n] = gape_expectation(tr, nb, fc, k, false, gamma, qp, c);
                }
                n = tr.parent[nb + n];
            }
        }
        __syncwarp(gmask);
        int sel;
        bai(tr, nb, tr.first_child[nb], (tr.meta[nb] >> 8) & 0xff, sel, best, challenger);
        done = tr.upper[nb + challenger] - tr.lower[nb + best] < a.cfg.accuracy;      // stopping rule (:100-102)
        done = done || episode > a.cfg.episodes;
        ++episode;
    }

    if (writer) {
        rng.store(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
        // get_plan (:129-131): the root's BAI best, unchanged since the last episode's selection
        const int action = error ? -1 : tr.meta[nb + best] & 0xff;
        a.plan[tree] = (int8_t)action;
        int32_t* res = a.result + (int64_t)tree * B2_MDP_GAPE_RESULT_WORDS;
        res[0] = n_nodes;
        res[1] = episode;
        res[2] = error;
        res[3] = action;
        res[4] = error ? -1 : best;
        res[5] = error ? -1 : challenger;
        res[6] = kSampled<Env> ? bad_row : 0;
        res[7] = 0;
    }
}

// b2_selftest_gape_expectation: case i is chance node 0 of a tree whose children fc = 0 .. K-1 hold mu_ucb = f,
// mu_lcb = -f, upper = lower = 0 and integer counts, with gamma = 1, so that value() is mu_ucb or mu_lcb exactly.
__global__ void gape_expectation_selftest_kernel(b2_mdp_gape_tree tr, int max_k, const int32_t* K, const int32_t* n,
                                                 const int32_t* cnt, const double* qp, const double* c, int n_cases,
                                                 double* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cases) return;
    const int64_t nb = (int64_t)i * max_k;
    for (int side = 0; side < 2; ++side)
        out[2 * i + side] = n[i] == 0 ? gape_expectation(tr, nb, 0, K[i], side == 0, 1.0, qp[i], c[i])
                                      : gape_expectation_kl(tr, nb, 0, K[i], n[i], side == 0, 1.0, cnt[i], c[i]);
}

}  // namespace
}  // namespace b2

using namespace b2;

static int check_mdp_gape_config(const b2_mdp_gape_config* cfg) {
    B2_REQUIRE(cfg->n_trees > 0 && cfg->episodes >= 0 && cfg->horizon >= 1, "bad batch / budget");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions <= 8, "n_actions must be in 1..8");
    B2_REQUIRE(cfg->max_next_states >= 1 && cfg->max_next_states <= 255, "max_next_states must be in 1..255");
    B2_REQUIRE((int64_t)cfg->node_capacity >= 1 + ((int64_t)cfg->episodes + 2) * cfg->horizon *
                                                      (cfg->n_actions + cfg->max_next_states),
               "node_capacity too small");
    B2_REQUIRE(cfg->thresholds && cfg->transition_thresholds && cfg->init_upper,
               "threshold / initial bound tables missing");
    return B2_OK;
}

extern "C" int b2_mdp_gape_plan(const b2_mdp_gape_config* cfg, const int32_t* root_states, const b2_mdp_gape_tree* tree,
                                uint64_t* rng, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_states && tree && rng && plan && result, "null pointer");
    if (check_mdp_gape_config(cfg) != B2_OK) return B2_ERR_INVALID;
    const int rc = check_lane_env(cfg->env_kind, cfg->n_actions, cfg->mdp);
    if (rc != B2_OK) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    GapeArgs a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.rng = rng; a.plan = plan; a.result = result;
    a.model = LaneModel{cfg->mdp};
    if (cfg->env_kind == B2_ENV_FINITE)
        mdp_gape_kernel<FiniteEnv><<<lane_grid<FiniteEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    else
        mdp_gape_kernel<HighwayEnv><<<lane_grid<HighwayEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_mdp_gape_plan_sampled(const b2_mdp_gape_config* cfg, const b2_finite_mdp_sampled* mdp,
                                        const uint8_t* terminal, int32_t env_draws, const int32_t* root_states,
                                        const b2_mdp_gape_tree* tree, int32_t* keys, uint64_t* rng, int8_t* plan,
                                        int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && mdp && terminal && root_states && tree && keys && rng && plan && result, "null pointer");
    if (check_mdp_gape_config(cfg) != B2_OK) return B2_ERR_INVALID;
    if (check_sampled_entry(cfg->env_kind, *mdp, cfg->n_actions, terminal, env_draws) != B2_OK) return B2_ERR_INVALID;
    cudaStream_t stream = (cudaStream_t)stream_;
    GapeArgs a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.rng = rng; a.plan = plan; a.result = result;
    a.keys = keys; a.model = LaneModel{b2_finite_mdp{}, *mdp, terminal, env_draws};
    mdp_gape_kernel<SampledFiniteEnv><<<lane_grid<SampledFiniteEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_selftest_gape_expectation(const double* f, const double* neg_f, const int32_t* counts,
                                            const double* zeros, int32_t max_k, const int32_t* K, const int32_t* n,
                                            const int32_t* cnt, const double* qp, const double* c, int32_t n_cases,
                                            double* out, void* stream) {
    B2_REQUIRE(f && neg_f && counts && zeros && K && n && cnt && qp && c && out, "null pointer");
    B2_REQUIRE(n_cases > 0 && max_k >= 1, "empty batch");
    b2_mdp_gape_tree tr{};
    tr.count = const_cast<int32_t*>(counts);
    tr.mu_ucb = const_cast<double*>(f);
    tr.mu_lcb = const_cast<double*>(neg_f);
    tr.upper = tr.lower = const_cast<double*>(zeros);
    gape_expectation_selftest_kernel<<<(n_cases + 127) / 128, 128, 0, (cudaStream_t)stream>>>(tr, max_k, K, n, cnt, qp,
                                                                                              c, n_cases, out);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
