// PlaTyPOOS -- PlaTyPOOS.plan of rl_agents/agents/tree_search/platypoos.py for a BATCH of independent decisions, one
// tree per CTA, one depth layer at a time:
//   root        expand(layer, h_max): h_max samples of every available action, each child created at its first sample.
//   explore(h)  h = 1 .. h_max-1: the layer sorted by value, descending and stable (a rank per node, ties in layer
//               order); the selection scan for p = p_top(h) .. 0 by one warp (the first node with count > min_visits
//               that is not yet flagged, the quota tested after EVERY visited node, the list cumulative over p); the
//               selected nodes expanded, their children stepped in parallel; candidates[p] updated in list order.
//   cross_validate  every candidate in dict order walked up to and including the root by one warp, expanding each node
//               cv_count[depth] times.
//   get_plan    the actions from the root to the first candidate of highest value.
//
// One env step per created child.  The reward and `done` of a step depend only on the node's state and the action on
// every model here (finite MDPs: R[s, a] and terminal[s]; HighwayLite is deterministic), and the reference keeps the
// first sample's state as the child's.  So a child of a node expanded `ev` times gets count ev and its reward added ev
// times one by one; a cross-validation expansion adds it cv_count more times.  Cross-validation only expands nodes that
// explore expanded, so it creates no child (error 3 if it would) and steps no env.
//
// The planner's stream: an expansion of a node that is not done draws ev x |available| randint(2**30) (2^30 divides
// 2^32: one buffered 32-bit half each), sample-major.  Exclusive prefix sums over a layer's selected nodes give each
// new child its first sample's position; on a stochastic finite MDP the child's state is drawn there by the env copy's
// default_rng(seed) (Pcg64::seed_from, sampled_next).  After the search the stream is advanced in closed form by every
// draw (Pcg64::skip32).
//
// Scenes (HighwayLite): only two layers are live, the one being expanded and the one being created, in two ping-pong
// buffers of layer_capacity scenes: layer h's in buffer h & 1, slot = node id - first id of the layer.
//
// Values are fp64 in the reference's order of operations and the library builds with -fmad=false, so every node equals
// the reference's bit for bit.
#include <math.h>

#include "common.cuh"
#include "highway_lite.cuh"
#include "lane_env.cuh"
#include "pcg64.cuh"

namespace b2 {
namespace {

constexpr int THREADS = 128;
constexpr int MAX_P = 32;
constexpr int FLAG_DONE = 1, FLAG_TO_EXPAND = 2;
constexpr int ERR_CAPACITY = 1, ERR_BAD_ROW = 2, ERR_CV_CHILD = 3, ERR_NO_CANDIDATE = 4;

// Per-tree scratch, tree-major: each field is [n_trees, layer_capacity (+1)].
struct Work {
    int32_t* scenes;        // HighwayLite: [n_trees, 2, layer_capacity, WORDS]
    int32_t* order;         // the layer sorted by value, descending
    int32_t* sel;           // the selected nodes, in list order
    int32_t* sel_p;         // and their p (-1: the root's expansion)
    int32_t* cbase;         // [layer_capacity + 1] exclusive prefix sum of the children each selected node creates
    int64_t* dbase;         // [layer_capacity + 1] exclusive prefix sum of its draws
};

__host__ __device__ inline char* carve(char* p, size_t bytes) { return p + ((bytes + 255) & ~(size_t)255); }

__host__ __device__ inline char* layout(char* base, int n, int W, bool highway, Work& w) {
    char* p = base;
    w.scenes = (int32_t*)p;
    if (highway) p = carve(p, (size_t)n * 2 * W * hw::WORDS * 4);
    int32_t** ints[4] = {&w.order, &w.sel, &w.sel_p, &w.cbase};
    for (int i = 0; i < 4; ++i) { *ints[i] = (int32_t*)p; p = carve(p, (size_t)n * (W + 1) * 4); }
    w.dbase = (int64_t*)p;
    p = carve(p, (size_t)n * (W + 1) * 8);
    return p;
}

struct Args {
    b2_platypoos_config cfg;
    b2_platypoos_tree tree;
    Work w;
    const int32_t* root_states;
    uint64_t* rng;
    int8_t* plan;
    int32_t* candidates;
    int32_t* result;
};

struct Shared {
    int n_nodes, layer_begin, layer_n, n_sel, error, steps, openings, n_cand;
    unsigned long long bad;            // (first-sample position << 32) | row of the first rejected row reached
    int64_t draws;                     // draws so far
    int cand[MAX_P], cand_order[MAX_P];
};

// Expand the n_sel selected nodes (sel, sel_p) of the layer starting at node layer_begin: ev[i] samples of every
// available action.  Creates the next layer [n_nodes, n_nodes + K) in list order and steps each new child once.
template <bool HW>
__device__ void expand_selected(const Args& a, Shared& sh, int tree, int depth, const int32_t* ev_of_p, int root_ev) {
    const b2_platypoos_config& c = a.cfg;
    const b2_platypoos_tree& tr = a.tree;
    const int W = c.layer_capacity, A = c.n_actions;
    const int64_t nb = (int64_t)tree * c.node_capacity, wb = (int64_t)tree * (W + 1);
    const int tid = threadIdx.x, lane = tid & 31;
    const int n_sel = sh.n_sel, n0 = sh.n_nodes;
    // ---- the prefix sums (warp 0), openings, first_child of every selected node ----
    if (tid < 32) {
        int carry = 0, opened = 0;
        int64_t dcarry = 0;
        for (int base = 0; base < n_sel; base += 32) {
            const int i = base + lane;
            int k = 0, ev = 0;
            int64_t dr = 0;
            if (i < n_sel) {
                const int node = a.w.sel[wb + i], p = a.w.sel_p[wb + i];
                ev = p < 0 ? root_ev : ev_of_p[p];
                const int navail = HW ? __popc(tr.state[nb + node]) : A - 1;
                if (!(tr.flags[nb + node] & FLAG_DONE)) {        // a done node returns before sampling (:150-151)
                    k = ev > 0 ? navail : 0;
                    dr = (int64_t)ev * navail;
                }
            }
            int x = k;
            int64_t y = dr;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int xs = __shfl_up_sync(0xffffffffu, x, o);
                const int64_t ys = __shfl_up_sync(0xffffffffu, y, o);
                if (lane >= o) { x += xs; y += ys; }
            }
            if (i < n_sel) {
                a.w.cbase[wb + i] = carry + x - k;
                a.w.dbase[wb + i] = dcarry + y - dr;
                tr.first_child[nb + a.w.sel[wb + i]] = k > 0 ? n0 + carry + x - k : -1;
            }
            carry += __shfl_sync(0xffffffffu, x, 31);
            dcarry += __shfl_sync(0xffffffffu, y, 31);
            opened += __reduce_add_sync(0xffffffffu, ev);
        }
        if (lane == 0) {
            a.w.cbase[wb + n_sel] = carry;
            a.w.dbase[wb + n_sel] = dcarry;
            sh.openings += opened;
            if (n0 + (int64_t)carry > c.node_capacity || carry > W) sh.error = ERR_CAPACITY;
        }
    }
    __syncthreads();
    if (sh.error) return;
    const int K = a.w.cbase[wb + n_sel];
    const int64_t pos0 = sh.draws;
    // ---- one step per new child ----
    auto parent_of = [&](int c_) {          // the last selected index whose cbase <= c_
        int lo = 0, hi = n_sel;             // invariant: cbase[lo] <= c_ < cbase[hi]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (a.w.cbase[wb + mid] <= c_) lo = mid; else hi = mid;
        }
        return lo;
    };
    auto write_child = [&](int id, int parent, int action, int32_t st, double r, bool done, int ev) {
        double cum = 0.0;                   // cumulative_reward starts from int 0: 0 + r == 0.0 + r
        for (int e = 0; e < ev; ++e) cum = cum + r;
        tr.parent[nb + id] = parent;
        tr.first_child[nb + id] = -1;
        tr.action[nb + id] = action;
        tr.depth[nb + id] = depth + 1;
        tr.count[nb + id] = ev;
        tr.flags[nb + id] = done ? FLAG_DONE : 0;
        tr.state[nb + id] = st;
        tr.cumulative[nb + id] = cum;
        tr.reward[nb + id] = r;
        tr.value[nb + id] = tr.value[nb + parent] + c.gamma_pow[depth] * (cum / (double)ev);
    };
    if (HW) {
        // both halves of a warp step together (an odd count is padded with a discarded item), on warp-uniform loop
        // conditions: hw::step in its full-warp mode
        const int li = lane & 15, half = lane >> 4, warp = tid >> 5;
        const int32_t* src = a.w.scenes + ((int64_t)tree * 2 + (depth & 1)) * W * hw::WORDS;
        int32_t* dst = a.w.scenes + ((int64_t)tree * 2 + ((depth + 1) & 1)) * W * hw::WORDS;
        for (int pr = warp; 2 * pr < K; pr += THREADS / 32) {
            const int item = 2 * pr + half;
            const bool live = item < K;
            const int j = live ? item : 2 * pr;
            const int i = parent_of(j);
            const int parent = a.w.sel[wb + i], p = a.w.sel_p[wb + i];
            const int action = hw::nth_action(tr.state[nb + parent], j - a.w.cbase[wb + i]);
            hw::Lane L;
            int t, si;
            hw::load_state(src + (int64_t)(parent - sh.layer_begin) * hw::WORDS, li, L, t, si);
            bool term, trunc;               // the 4-tuple step drops truncation
            const float r = hw::step(L, li, t, si, action, term, trunc, 0xffffffffu);
            if (live) hw::store_state(dst + (int64_t)j * hw::WORDS, li, L, t, si);
            const int mask = hw::avail_mask(__shfl_sync(0xffffffffu, L.y, 0, 16), si);
            if (live && li == 0)
                write_child(n0 + j, parent, action, mask, (double)r, term, p < 0 ? root_ev : ev_of_p[p]);
        }
    } else {
        const b2_finite_mdp_sampled& m = c.mdp;
        for (int j = tid; j < K; j += THREADS) {
            const int i = parent_of(j);
            const int parent = a.w.sel[wb + i], p = a.w.sel_p[wb + i];
            const int off = j - a.w.cbase[wb + i];
            const int action = off + 1;                             // range(1, n) (:147)
            const int s = tr.state[nb + parent];
            const int64_t row = (int64_t)s * A + action;
            int s2 = m.next[row * m.n_next];
            if (c.env_draws) {
                const int64_t pos = pos0 + a.w.dbase[wb + i] + off; // the child's first sample
                if (!m.row_ok[row]) {
                    atomicMin(&sh.bad, ((unsigned long long)pos << 32) | (unsigned)row);
                    continue;
                }
                Pcg64 e;                                            // the stream before the plan
                e.load(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
                e.skip32((uint64_t)pos);
                const uint32_t seed = e.integers(1u << 30);         // state.seed(np_random.randint(2**30)), :154
                Pcg64 env_rng;
                env_rng.seed_from(seed);
                s2 = sampled_next(m, row, true, env_rng);
            }
            write_child(n0 + j, parent, action, s2, m.reward[row], c.terminal[s] != 0,
                        p < 0 ? root_ev : ev_of_p[p]);
        }
    }
    __syncthreads();
    if (tid == 0) {
        if (sh.bad != ~0ull) sh.error = ERR_BAD_ROW;
        sh.draws += a.w.dbase[wb + n_sel];
        sh.steps += K;
        sh.layer_begin = n0;
        sh.layer_n = K;
        sh.n_nodes = n0 + K;
    }
    __syncthreads();
}

template <bool HW>
__global__ void __launch_bounds__(THREADS, 1) platypoos_kernel(Args a) {
    __shared__ Shared sh;
    const b2_platypoos_config& c = a.cfg;
    const b2_platypoos_tree& tr = a.tree;
    const int tree = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const int H = c.horizon, W = c.layer_capacity, A = c.n_actions;
    const int64_t nb = (int64_t)tree * c.node_capacity, wb = (int64_t)tree * (W + 1);

    // ---- the root: PlaTyPOOSNode(None) with value 0.0, the only node of layer 0 ----
    if (tid == 0) {
        sh.n_nodes = 1; sh.layer_begin = 0; sh.layer_n = 1; sh.n_sel = 1;
        sh.error = 0; sh.steps = 0; sh.openings = 0; sh.n_cand = 0;
        sh.bad = ~0ull;
        sh.draws = 0;
        tr.parent[nb] = -1; tr.first_child[nb] = -1; tr.action[nb] = -1; tr.depth[nb] = 0; tr.count[nb] = 0;
        tr.flags[nb] = 0; tr.cumulative[nb] = 0.0; tr.value[nb] = 0.0; tr.reward[nb] = 0.0;
        if (!HW) tr.state[nb] = a.root_states[tree];
        a.w.sel[wb] = 0;
        a.w.sel_p[wb] = -1;
    }
    if (tid < MAX_P) sh.cand[tid] = -1;
    if (HW && tid < 16) {
        hw::Lane L;
        int t, si;
        hw::load_state(a.root_states + (int64_t)tree * hw::WORDS, tid, L, t, si);
        hw::store_state(a.w.scenes + (int64_t)tree * 2 * W * hw::WORDS, tid, L, t, si);
        const int mask = hw::avail_mask(__shfl_sync(0xFFFFu, L.y, 0, 16), si);
        if (tid == 0) tr.state[nb] = mask;
    }
    __syncthreads();
    expand_selected<HW>(a, sh, tree, 0, nullptr, H);                // root.expand(layer, h_max), :91

    // ---- explore(h), h = 1 .. h_max - 1 ----
    for (int h = 1; h < H && !sh.error; ++h) {
        const int lb = sh.layer_begin, L = sh.layer_n;
        // sorted(layer, key=value, reverse=True): stable, so equal values keep layer order
        for (int i = tid; i < L; i += THREADS) {
            const double v = tr.value[nb + lb + i];
            int rank = 0;
            for (int j = 0; j < L; ++j) {
                const double u = tr.value[nb + lb + j];
                rank += (u > v || (u == v && j < i)) ? 1 : 0;
            }
            a.w.order[wb + rank] = lb + i;
        }
        __syncthreads();
        const int32_t* nc_h = c.nodes_count + (int64_t)h * c.max_p;
        const int32_t* ev_h = c.evaluations + (int64_t)h * c.max_p;
        const int32_t* mv_h = c.min_visits + (int64_t)h * c.max_p;
        if (tid < 32) {
            // the selection scan (:47-55): after every visited node, stop once the list holds nodes_count entries
            int n_sel = 0;
            for (int p = c.p_top[h]; p >= 0; --p) {
                const int nc = nc_h[p], mv = mv_h[p];
                for (int base = 0; base < L; base += 32) {
                    const int idx = base + lane;
                    const bool valid = idx < L;
                    const int node = valid ? a.w.order[wb + idx] : 0;
                    const bool elig = valid && tr.count[nb + node] > mv && !(tr.flags[nb + node] & FLAG_TO_EXPAND);
                    unsigned e = __ballot_sync(0xffffffffu, elig);
                    const unsigned upto = 0xffffffffu >> (31 - lane);        // lanes 0..lane
                    const unsigned stop = __ballot_sync(0xffffffffu, valid && n_sel + __popc(e & upto) >= nc);
                    if (stop) e &= 0xffffffffu >> (31 - (__ffs(stop) - 1));
                    if ((e >> lane) & 1) {
                        const int at = n_sel + __popc(e & (upto >> 1));
                        a.w.sel[wb + at] = node;
                        a.w.sel_p[wb + at] = p;
                        tr.flags[nb + node] |= FLAG_TO_EXPAND;
                    }
                    n_sel += __popc(e);
                    __syncwarp();
                    if (stop) break;
                }
            }
            if (lane == 0) sh.n_sel = n_sel;
        }
        __syncthreads();
        expand_selected<HW>(a, sh, tree, h, ev_h, 0);
        if (tid == 0) {
            // candidates (:62-64): a new p is inserted, an existing one replaced by a strictly higher value
            for (int i = 0; i < sh.n_sel; ++i) {
                const int node = a.w.sel[wb + i], p = a.w.sel_p[wb + i];
                if (sh.cand[p] < 0) {
                    sh.cand[p] = node;
                    sh.cand_order[sh.n_cand++] = p;
                } else if (tr.value[nb + node] > tr.value[nb + sh.cand[p]]) {
                    sh.cand[p] = node;
                }
            }
        }
        __syncthreads();
    }

    // ---- cross_validate (:66-76), one warp ----
    if (tid < 32 && !sh.error) {
        int opened = 0, err = 0;
        int64_t draws = 0;
        for (int k = 0; k < sh.n_cand && !err; ++k) {
            for (int node = sh.cand[sh.cand_order[k]]; node >= 0; node = tr.parent[nb + node]) {
                const int d = tr.depth[nb + node], cnt = c.cv_count[d];
                opened += cnt;
                if ((tr.flags[nb + node] & FLAG_DONE) || cnt <= 0) continue;
                const int navail = HW ? __popc(tr.state[nb + node]) : A - 1;
                const int fc = tr.first_child[nb + node];
                if (navail > 0 && fc < 0) { err = ERR_CV_CHILD; break; }
                draws += (int64_t)cnt * navail;
                for (int j = lane; j < navail; j += 32) {          // a finite MDP may have more than 33 actions
                    const int ch = fc + j;
                    double cum = tr.cumulative[nb + ch];
                    const double r = tr.reward[nb + ch];
                    for (int e = 0; e < cnt; ++e) cum = cum + r;
                    const int count = tr.count[nb + ch] + cnt;
                    tr.cumulative[nb + ch] = cum;
                    tr.count[nb + ch] = count;
                    tr.value[nb + ch] = tr.value[nb + node] + c.gamma_pow[d] * (cum / (double)count);
                }
                __syncwarp();
            }
        }
        if (lane == 0) {
            sh.openings += opened;
            sh.draws += draws;
            if (err) sh.error = err;
        }
    }
    __syncthreads();

    // ---- get_plan (:78-86), the stream, the result words ----
    if (tid == 0) {
        int len = 0;
        if (!sh.error) {
            int best = -1;
            for (int k = 0; k < sh.n_cand; ++k) {           // max(): the first maximum in dict order
                const int node = sh.cand[sh.cand_order[k]];
                if (best < 0 || tr.value[nb + node] > tr.value[nb + best]) best = node;
            }
            if (best < 0) {
                sh.error = ERR_NO_CANDIDATE;
            } else {
                len = tr.depth[nb + best];
                for (int node = best, k = len - 1; node > 0; node = tr.parent[nb + node], --k)
                    a.plan[(int64_t)tree * H + k] = (int8_t)tr.action[nb + node];
            }
        }
        Pcg64 rng;
        rng.load(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
        rng.skip32((uint64_t)sh.draws);
        rng.store(a.rng + (int64_t)tree * B2_PCG64_STATE_WORDS);
        int32_t* cand = a.candidates + (int64_t)tree * 2 * c.max_p;
        for (int k = 0; k < c.max_p; ++k) {
            cand[2 * k] = k < sh.n_cand ? sh.cand_order[k] : -1;
            cand[2 * k + 1] = k < sh.n_cand ? sh.cand[sh.cand_order[k]] : -1;
        }
        int32_t* res = a.result + (int64_t)tree * B2_PLATYPOOS_RESULT_WORDS;
        res[0] = sh.n_nodes;
        res[1] = sh.openings;
        res[2] = len;
        res[3] = sh.error;
        res[4] = sh.error == ERR_BAD_ROW ? (int)(sh.bad & 0xffffffffu) : -1;
        res[5] = sh.steps;
        res[6] = sh.n_cand;
        res[7] = 0;
    }
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" int64_t b2_platypoos_workspace_bytes(const b2_platypoos_config* cfg) {
    if (!cfg || cfg->n_trees <= 0 || cfg->layer_capacity < 1) return 0;
    Work w;
    return (int64_t)(size_t)layout(nullptr, cfg->n_trees, cfg->layer_capacity, cfg->env_kind == B2_ENV_HIGHWAY, w);
}

extern "C" int b2_platypoos_plan(const b2_platypoos_config* cfg, const int32_t* root_states,
                                 const b2_platypoos_tree* tree, void* workspace, uint64_t* rng, int8_t* plan,
                                 int32_t* candidates, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_states && tree && workspace && rng && plan && candidates && result, "null pointer");
    B2_REQUIRE(tree->parent && tree->first_child && tree->action && tree->depth && tree->count && tree->flags &&
               tree->state && tree->cumulative && tree->value && tree->reward, "tree arrays missing");
    B2_REQUIRE(cfg->n_trees > 0, "bad batch");
    // h_max < 2 runs no explore(), so the reference's get_plan takes max() of no candidate
    B2_REQUIRE(cfg->horizon >= 2, "horizon must be >= 2");
    B2_REQUIRE(cfg->n_actions >= 2 && cfg->n_actions < 128, "n_actions must be in 2..127");
    B2_REQUIRE(cfg->node_capacity >= 1 && cfg->layer_capacity >= 1, "node and layer capacities must be >= 1");
    B2_REQUIRE(cfg->max_p >= 1 && cfg->max_p <= MAX_P, "max_p must be in 1..32");
    B2_REQUIRE(cfg->p_top && cfg->nodes_count && cfg->evaluations && cfg->min_visits && cfg->cv_count &&
               cfg->gamma_pow, "quota / cross-validation / gamma tables missing");
    const int rc = check_env_kind(cfg->env_kind, cfg->n_actions);
    if (rc != B2_OK) return rc;
    Args a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.rng = rng; a.plan = plan;
    a.candidates = candidates; a.result = result;
    layout((char*)workspace, cfg->n_trees, cfg->layer_capacity, cfg->env_kind == B2_ENV_HIGHWAY, a.w);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (cfg->env_kind == B2_ENV_FINITE) {
        if (check_sampled_mdp(cfg->mdp, cfg->n_actions, cfg->terminal, true) != B2_OK) return B2_ERR_INVALID;
        platypoos_kernel<false><<<cfg->n_trees, THREADS, 0, stream>>>(a);
    } else {
        platypoos_kernel<true><<<cfg->n_trees, THREADS, 0, stream>>>(a);
    }
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
