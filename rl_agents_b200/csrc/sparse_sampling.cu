// Sparse sampling -- SparseSampling.plan of rl_agents/agents/tree_search/sparse_sampling.py for a BATCH of independent
// decisions.  The reference recurses: DecisionNode.estimateV (:38-51) runs ChanceNode.estimateQ (:71-88) on every
// action, which draws C samples -- a deep copy of the env, `seed(np_random.randint(2**30))`, `step(action)` -- keeps
// the distinct observations as children in first-visit order, and only then calls estimateV on each of them.  Here
// the same order runs as a depth-first search over an explicit stack of `horizon` frames (no node arena): a frame
// holds its state, its action cursor, its running maximum, and the chance node in progress with its <= C distinct
// children, their counts, the child cursor and the running sum S.
//
// The planner's numpy PCG64 stream is consumed exactly as the reference consumes it: C draws of randint(2**30) per
// chance node (2^30 divides 2^32, so every draw is one buffered 32-bit half), then choice(indices) for a tie at the
// root (random_argmax, abstract.py:304-311).  On a stochastic finite MDP every sample replays the seeded env's own
// draw: default_rng(seed) -- SeedSequence and PCG64 seeding, Pcg64::seed_from -- then Generator.choice(p.size, p=p),
// i.e. searchsorted(cdf, random(), "right") over the host-made cdf.  A deterministic model (B = 1, and HighwayLite)
// needs no env generator: the reference throws it away after one step.
//
// Values: fp64, `reward + gamma * S / C` evaluated as r + ((gamma * S) / C) with S summed left to right, and the
// first maximum of the chance values (np.amax).  The library builds with -fmad=false, so every value equals the
// reference's bit for bit.
//
// One tree per lane (finite MDP) or per 16-lane group (HighwayLite, lane = vehicle slot, hw::step's mapping as in
// brue.cu).  On HighwayLite every lane of a group runs the same search on group-uniform values; the env states along
// the current path live in the workspace, one per depth, and a (node, available action) is stepped once: the model is
// deterministic, so the reference's C samples are C identical steps, and the child gets count C.
#include <math.h>

#include "common.cuh"
#include "highway_lite.cuh"
#include "lane_env.cuh"
#include "pcg64.cuh"
#include "sparse_sampling.cuh"

namespace b2 {
namespace {

using ss::KIND_DECISION;
using ss::KIND_CHANCE;
using ss::ERR_CAPACITY;
using ss::ERR_BAD_ROW;
using ss::put;

// The search stack, tree index fastest (lanes at the same depth touch neighbouring words).  Frame d of tree t is
// entry d * n + t; child j of frame d is entry (d * C + j) * n + t.
struct Stack {
    double *best, *S, *r;              // running max of the chance values, running sum, the chance node's reward
    int32_t *state, *node, *act;       // state id (finite) / available-action mask (HighwayLite), node id, action cursor
    int32_t *chance, *nk, *kc;         // chance node id, distinct children, child cursor
    int32_t *k_state, *k_count, *k_node;
    int32_t* hw;                       // HighwayLite: [n, H + 1, WORDS] env states along the current path
};

__host__ __device__ inline char* carve(char* p, size_t bytes) { return p + ((bytes + 255) & ~(size_t)255); }

// Lays the stack out from `base`; returns the end (base = nullptr gives the size).
__host__ __device__ inline char* layout(char* base, int n, int H, int C, bool highway, Stack& s) {
    const size_t fr = (size_t)H * n, kid = fr * C;
    char* p = base;
    s.best = (double*)p; p = carve(p, fr * 8);
    s.S = (double*)p; p = carve(p, fr * 8);
    s.r = (double*)p; p = carve(p, fr * 8);
    int32_t** ints[6] = {&s.state, &s.node, &s.act, &s.chance, &s.nk, &s.kc};
    for (int i = 0; i < 6; ++i) { *ints[i] = (int32_t*)p; p = carve(p, fr * 4); }
    int32_t** kids[3] = {&s.k_state, &s.k_count, &s.k_node};
    for (int i = 0; i < 3; ++i) { *kids[i] = (int32_t*)p; p = carve(p, kid * 4); }
    s.hw = (int32_t*)p;
    if (highway) p = carve(p, (size_t)n * (H + 1) * hw::WORDS * 4);
    return p;
}

struct SsArgs {
    b2_sparse_sampling_config cfg;
    b2_sparse_sampling_tree tree;      // capacity 0: no dump
    Stack st;
    const int32_t* root_states;
    uint64_t* rng;
    double* root_q;
    int8_t* plan;
    int32_t* result;
};

struct SFiniteEnv {
    static constexpr int GROUP = 1;
    __device__ __forceinline__ int root(const SsArgs& a, int tree, int li, unsigned gmask) {
        return a.root_states[tree];
    }
    __device__ __forceinline__ int n_choices(const SsArgs& a, int state) const { return a.cfg.n_actions; }
    __device__ __forceinline__ int action(int state, int idx) const { return idx; }   // range(action_space.n), :40-43
    // estimateQ's sampling loop (:76-84) for `action` in frame d: C samples, the distinct next states in first-visit
    // order with their counts, each a new DecisionNode.  Returns the reward; sets err / bad_row on a rejected row.
    __device__ __forceinline__ double expand(const SsArgs& a, int tree, int li, unsigned gmask, int d,
                                             int state, int action, int chance, Pcg64& rng, int& n_nodes, int& nk,
                                             int& err, int& bad_row) {
        const b2_finite_mdp_sampled& m = a.cfg.mdp;
        const Stack& st = a.st;
        const int n = a.cfg.n_trees, C = a.cfg.C, B = m.n_next;
        const bool rec = a.tree.capacity > 0;
        const int64_t nb = (int64_t)tree * a.tree.capacity;
        const int64_t row = (int64_t)state * m.n_actions + action;
        nk = 0;
        for (int i = 0; i < C; ++i) {
            const uint32_t seed = rng.integers(1u << 30);           // next_state.seed(np_random.randint(2**30)), :79
            if (!m.row_ok[row]) { err = ERR_BAD_ROW; bad_row = (int)row; return 0.0; }
            int k = 0;
            if (B > 1) {                                            // Generator.choice(p.size, p=p) of the seeded env
                Pcg64 e;
                e.seed_from(seed);
                k = searchsorted_right(m.cdf + row * B, B, e.random());
            }
            const int s2 = m.next[row * B + k];
            int j = 0;
            while (j < nk && st.k_state[((int64_t)d * C + j) * n + tree] != s2) ++j;
            const int64_t kj = ((int64_t)d * C + j) * n + tree;
            if (j == nk) {                                          // get_child(observation): first visit, :93-96
                ++nk;
                st.k_state[kj] = s2;
                st.k_count[kj] = 1;
                st.k_node[kj] = n_nodes;
                if (rec) put(a.tree, nb, n_nodes, chance, KIND_DECISION, s2, d + 1);
                ++n_nodes;
            } else {
                st.k_count[kj] += 1;
            }
        }
        if (rec)
            for (int j = 0; j < nk; ++j) {
                const int64_t kj = ((int64_t)d * C + j) * n + tree;
                a.tree.count[nb + st.k_node[kj]] = st.k_count[kj];
            }
        return m.reward[row];                                       // every sample's reward is R[s, a]
    }
};

struct SHighwayEnv {
    static constexpr int GROUP = 16;
    __device__ __forceinline__ int32_t* words(const SsArgs& a, int tree, int d) const {
        return a.st.hw + ((int64_t)tree * (a.cfg.horizon + 1) + d) * hw::WORDS;
    }
    __device__ __forceinline__ int root(const SsArgs& a, int tree, int li, unsigned gmask) {
        hw::Lane L;
        int t, si;
        hw::load_state(a.root_states + (int64_t)tree * hw::WORDS, li, L, t, si);
        hw::store_state(words(a, tree, 0), li, L, t, si);
        __syncwarp(gmask);
        return hw::avail_mask(__shfl_sync(gmask, L.y, 0, 16), si);
    }
    __device__ __forceinline__ int n_choices(const SsArgs& a, int mask) const { return __popc(mask); }
    __device__ __forceinline__ int action(int mask, int idx) const { return hw::nth_action(mask, idx); }
    __device__ __forceinline__ double expand(const SsArgs& a, int tree, int li, unsigned gmask, int d,
                                             int mask, int action, int chance, Pcg64& rng, int& n_nodes, int& nk,
                                             int& err, int& bad_row) {
        const Stack& st = a.st;
        const int n = a.cfg.n_trees, C = a.cfg.C;
        for (int i = 0; i < C; ++i) rng.integers(1u << 30);        // C samples of one deterministic step
        hw::Lane L;
        int t, si;
        hw::load_state(words(a, tree, d), li, L, t, si);
        bool term, trunc;                                           // `done` is ignored (:81)
        const float r = hw::step(L, li, t, si, action, term, trunc, gmask);
        int child_mask = 0;
        if (d + 1 < a.cfg.horizon) {
            hw::store_state(words(a, tree, d + 1), li, L, t, si);
            __syncwarp(gmask);
            child_mask = hw::avail_mask(__shfl_sync(gmask, L.y, 0, 16), si);
        }
        const int64_t k0 = (int64_t)d * C * n + tree;
        nk = 1;
        st.k_state[k0] = child_mask;
        st.k_count[k0] = C;
        st.k_node[k0] = n_nodes;
        if (a.tree.capacity > 0 && li == 0) {
            const int64_t nb = (int64_t)tree * a.tree.capacity;
            put(a.tree, nb, n_nodes, chance, KIND_DECISION, -1, d + 1);
            a.tree.count[nb + n_nodes] = C;
        }
        ++n_nodes;
        return (double)r;
    }
};

template <class Env>
__global__ void __launch_bounds__(128, Env::GROUP == 16 ? 4 : 8) sparse_sampling_kernel(SsArgs a) {
    B2_LANE_MAP_LIVE(Env, a.cfg.n_trees);          // whole lane groups: no live lane of a group leaves
    const int H = a.cfg.horizon, C = a.cfg.C, n = a.cfg.n_trees, A = a.cfg.n_actions;
    const Stack& st = a.st;
    const b2_sparse_sampling_tree& tr = a.tree;
    const bool rec = tr.capacity > 0;
    const int64_t nb = (int64_t)tree * tr.capacity;
    double* root_q = a.root_q + (int64_t)tree * A;
    Env env;

    Pcg64 rng;
    rng.load(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
    if (writer) {
        for (int i = 0; i < A; ++i) root_q[i] = __longlong_as_double(0x7ff8000000000000LL);   // NaN: not available
        if (rec) put(tr, nb, 0, -1, KIND_DECISION, -1, 0);                                   // DecisionNode(None)
    }
    // Every lane of a group keeps the same counters and writes the same frame words; only lane 0 writes the dump.
    int n_nodes = 1, n_chance = 0, samples = 0, error = 0, bad_row = -1;
    const int root_choice = env.root(a, tree, li, gmask);
    st.state[tree] = root_choice;
    st.node[tree] = 0;
    st.act[tree] = 0;
    int d = 0;
    bool begin = true;                              // true: start the chance node of frame d's action cursor
    while (true) {
        if (begin) {
            const int64_t f = (int64_t)d * n + tree;
            const int s = st.state[f];
            const int action = env.action(s, st.act[f]);
            if (rec && n_nodes + 1 + C > tr.capacity) { error = ERR_CAPACITY; break; }
            const int c = n_nodes++;                // DecisionNode.get_child(action), :58-61
            ++n_chance;
            if (rec && writer) put(tr, nb, c, st.node[f], KIND_CHANCE, action, d);
            int nk = 0;
            const double r = env.expand(a, tree, li, gmask, d, s, action, c, rng, n_nodes, nk, error, bad_row);
            samples += error ? 1 : C;
            if (error) break;
            st.chance[f] = c;
            st.r[f] = r;
            st.nk[f] = nk;
            st.kc[f] = 0;
            st.S[f] = 0.0;                          // sum(...) starts from int 0: 0 + x == 0.0 + x
            if (d + 1 < H) {                        // estimateV of the first child (:85-86)
                const int64_t k0 = (int64_t)d * C * n + tree, g = f + n;
                st.state[g] = st.k_state[k0];
                st.node[g] = st.k_node[k0];
                st.act[g] = 0;
                ++d;
                continue;
            }
            begin = false;                          // children at the horizon keep value 0: S stays 0
        }
        // the chance node of frame d is complete: ChanceNode.value (:87-88), then the decision node's next action
        const int64_t f = (int64_t)d * n + tree;
        const double q = st.r[f] + a.cfg.gamma * st.S[f] / (double)C;
        int idx = st.act[f];
        if (writer) {
            if (rec) tr.value[nb + st.chance[f]] = q;
            if (d == 0) root_q[env.action(st.state[f], idx)] = q;
        }
        if (idx == 0 || q > st.best[f]) st.best[f] = q;               // np.amax: the first maximum
        st.act[f] = ++idx;
        if (idx < env.n_choices(a, st.state[f])) { begin = true; continue; }
        const double v = st.best[f];                                   // DecisionNode.value, :51
        if (rec && writer) tr.value[nb + st.node[f]] = v;
        if (d == 0) break;
        --d;                                                           // back in the parent's chance node
        const int64_t p = f - n;
        int kc = st.kc[p];
        st.S[p] = st.S[p] + v * (double)st.k_count[((int64_t)d * C + kc) * n + tree];
        st.kc[p] = ++kc;
        if (kc < st.nk[p]) {
            const int64_t kj = ((int64_t)d * C + kc) * n + tree;
            st.state[f] = st.k_state[kj];
            st.node[f] = st.k_node[kj];
            st.act[f] = 0;
            ++d;
            begin = true;
        } else {
            begin = false;
        }
    }

    if (writer) {
        int action = -1;
        if (!error)
            action = ss::root_plan(root_q, env.n_choices(a, root_choice),
                                   [&](int i) { return env.action(root_choice, i); }, rng);
        rng.store(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
        a.plan[tree] = (int8_t)action;
        int32_t* res = a.result + (int64_t)tree * B2_SPARSE_SAMPLING_RESULT_WORDS;
        res[0] = n_nodes;
        res[1] = n_chance;
        res[2] = samples;
        res[3] = action;
        res[4] = error;
        res[5] = bad_row;
        res[6] = 0;
        res[7] = 0;
    }
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" int64_t b2_sparse_sampling_workspace_bytes(const b2_sparse_sampling_config* cfg) {
    if (!cfg || cfg->n_trees <= 0 || cfg->horizon < 1 || cfg->C < 1) return 0;
    Stack s;
    return (int64_t)(size_t)layout(nullptr, cfg->n_trees, cfg->horizon, cfg->C, cfg->env_kind == B2_ENV_HIGHWAY, s);
}

extern "C" int b2_sparse_sampling_plan(const b2_sparse_sampling_config* cfg, const int32_t* root_states,
                                       const b2_sparse_sampling_tree* tree, void* workspace, uint64_t* rng,
                                       double* root_q, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_states && workspace && rng && root_q && plan && result, "null pointer");
    B2_REQUIRE(cfg->n_trees > 0, "bad batch");
    // horizon 0 leaves the root without children (the reference's selection_rule raises); C 0 never binds `reward`
    B2_REQUIRE(cfg->horizon >= 1 && cfg->C >= 1, "horizon and C must be >= 1");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions < 128, "n_actions must be in 1..127");
    SsArgs a;
    a.cfg = *cfg;
    a.tree = b2_sparse_sampling_tree{};
    if (tree) {
        B2_REQUIRE(tree->capacity >= 1 && tree->parent && tree->kind && tree->key && tree->depth && tree->count &&
                   tree->value, "tree dump arrays missing");
        a.tree = *tree;
    }
    a.root_states = root_states; a.rng = rng; a.root_q = root_q; a.plan = plan; a.result = result;
    const int rc = check_env_kind(cfg->env_kind, cfg->n_actions);
    if (rc != B2_OK) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (cfg->env_kind == B2_ENV_FINITE) {
        if (check_sampled_mdp(cfg->mdp, cfg->n_actions, nullptr, false) != B2_OK) return B2_ERR_INVALID;
        layout((char*)workspace, cfg->n_trees, cfg->horizon, cfg->C, false, a.st);
        sparse_sampling_kernel<SFiniteEnv><<<lane_grid<SFiniteEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    } else {
        layout((char*)workspace, cfg->n_trees, cfg->horizon, cfg->C, true, a.st);
        sparse_sampling_kernel<SHighwayEnv><<<lane_grid<SHighwayEnv>(cfg->n_trees), 128, 0, stream>>>(a);
    }
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
