// Sparse sampling, ONE decision on the whole GPU, level by level (b2_sparse_sampling_plan_levels).
//
// On a deterministic model (HighwayLite; a finite MDP with one next state per row) the reference's tree is fixed by the
// root state alone: the C samples of a chance node reach one observation, so every chance node has one decision
// child of count C, and a decision node above the horizon has one chance child per available action.  The draws only
// move the planner's stream: C halves of randint(2**30) per chance node (2^30 divides 2^32: no rejection).  So the
// tree that the depth-first lane kernel (sparse_sampling.cu) builds one step after another is built here level by
// level, in one cooperative persistent launch whose phases are separated by grid barriers:
//   expand, d = 0..H-1  exclusive prefix sum of level d's available-action counts -> chance node j of level d, whose
//                       decision child is node j of level d + 1; then one 16-lane group (HighwayLite) or one thread
//                       (finite) per chance node steps the parent's state with the action.  Scenes of two levels are
//                       resident: level d's are read from buffer d & 1, level d + 1's written to the other.
//   values, d = H-1..0  the lane kernel's expressions in its order (-fmad=false): S = 0.0 + V(child) * C (0.0 at the
//                       horizon), q = r + gamma * S / C, the decision value the first maximum over the chance
//                       children in available-action order; subtree sizes on the way up.
//   ids, d = 0..H-1     (with a tree dump only) the depth-first creation order from the sizes: a decision node D,
//                       then per action its chance node, that node's decision child and the child's subtree.
//   finish (1 thread)   the stream skipped by C * (chance nodes) halves in closed form (Pcg64::skip32), then the
//                       root's tie-break as the lane kernel draws it.
// Every field -- the dump, root_q, plan, result words, RNG words -- equals the lane kernel's bit for bit.
#include <math.h>

#include "common.cuh"
#include "highway_lite.cuh"
#include "pcg64.cuh"
#include "sparse_sampling.cuh"

namespace b2 {
namespace sslev {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int MAX_CTAS = 1024;

struct Control {                // head of the workspace; zeroed by the launch wrapper
    unsigned bar_count, bar_gen;
};

// The worst case (every decision node has all A actions), level-major: decision node j of level d is entry
// off(d) + j, off(d) = A^0 + ... + A^(d-1); its incoming chance node shares the entry.
struct Nodes {
    int32_t* st;                // finite: state id; HighwayLite: available-action mask
    int32_t* nch;               // chance children (0 at the horizon)
    int32_t* first;             // first chance child, an index into the next level
    int32_t* par;               // parent, an index into the previous level
    int32_t* act;               // incoming action
    int32_t* size;              // nodes of the subtree (decision node included)
    int32_t* id;                // creation-order id
    double* rew;                // the incoming chance node's reward
    double* val;                // DecisionNode.value
    double* q;                  // the incoming ChanceNode.value
};

struct Layout {
    size_t ctl, part, lvl_n, nodes[10], scenes, total;
    int64_t n_entries, scene_level;
};

__host__ __device__ inline int64_t level_off(int A, int d) {
    int64_t off = 0, p = 1;
    for (int k = 0; k < d; ++k) { off += p; p *= A; }
    return off;
}

inline size_t up(size_t b) { return (b + 255) & ~(size_t)255; }

inline Layout make_layout(const b2_sparse_sampling_config* cfg) {
    Layout l;
    const int A = cfg->n_actions, H = cfg->horizon;
    l.n_entries = level_off(A, H + 1);
    l.scene_level = level_off(A, H) - level_off(A, H - 1);            // A^(H-1)
    size_t p = 0;
    l.ctl = p; p += up(sizeof(Control));
    l.part = p; p += up((size_t)MAX_CTAS * 4);
    l.lvl_n = p; p += up((size_t)(H + 1) * 4);
    for (int i = 0; i < 10; ++i) { l.nodes[i] = p; p += up((size_t)l.n_entries * (i < 7 ? 4 : 8)); }
    l.scenes = p;
    if (cfg->env_kind == B2_ENV_HIGHWAY) p += up((size_t)2 * l.scene_level * hw::WORDS * 4);
    l.total = p;
    return l;
}

struct Args {
    b2_sparse_sampling_config cfg;
    b2_sparse_sampling_tree tree;       // capacity 0: no dump
    Nodes n;
    Control* ctl;
    int32_t* part;                      // [grid] per-CTA sums of the level scan
    int32_t* lvl_n;                     // [H + 1] decision nodes per level
    int32_t* scenes;                    // HighwayLite: [2, A^(H-1), WORDS]
    int64_t scene_level;
    const int32_t* root_states;
    uint64_t* rng;
    double* root_q;
    int8_t* plan;
    int32_t* result;
};

template <bool HW>
__device__ __forceinline__ int action_of(int choice, int idx) {
    return HW ? hw::nth_action(choice, idx) : idx;
}

// Block-wide sum; every thread gets it.  red: [WARPS + 1] shared ints.
__device__ __forceinline__ int block_sum(int v, int* red) {
    v = __reduce_add_sync(0xffffffffu, v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    int s = 0;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) s += red[w];
    return s;
}

// Block-wide exclusive scan; `total` gets the sum.
__device__ __forceinline__ int block_scan(int v, int* red, int& total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    __syncthreads();
    if (lane == 31) red[w] = x;
    __syncthreads();
    int before = 0;
    total = 0;
#pragma unroll
    for (int k = 0; k < WARPS; ++k) {
        before += k < w ? red[k] : 0;
        total += red[k];
    }
    return before + x - v;
}

__device__ __forceinline__ void barrier(const Args& a) { grid_barrier(a.ctl, gridDim.x); }

template <bool HW>
__global__ void __launch_bounds__(THREADS, 2) sparse_sampling_levels_kernel(Args a) {
    __shared__ int red[WARPS + 1];
    const int tid = threadIdx.x, bid = blockIdx.x, G = gridDim.x;
    const int gtid = bid * THREADS + tid, n_threads = G * THREADS;
    const int H = a.cfg.horizon, C = a.cfg.C, A = a.cfg.n_actions;
    const Nodes& nd = a.n;
    const b2_sparse_sampling_tree& tr = a.tree;

    // ---- the root: DecisionNode(None) ----
    if (bid == 0) {
        if (HW) {
            if (tid < 16) {
                hw::Lane L;
                int t, si;
                hw::load_state(a.root_states, tid, L, t, si);
                hw::store_state(a.scenes, tid, L, t, si);
                const int mask = hw::avail_mask(__shfl_sync(0xFFFFu, L.y, 0, 16), si);
                if (tid == 0) { nd.st[0] = mask; nd.nch[0] = __popc(mask); a.lvl_n[0] = 1; }
            }
        } else if (tid == 0) {
            nd.st[0] = a.root_states[0];
            nd.nch[0] = A;                          // range(action_space.n), :40-43
            a.lvl_n[0] = 1;
        }
        if (tid < A) a.root_q[tid] = __longlong_as_double(0x7ff8000000000000LL);   // NaN: not available
    }
    barrier(a);

    // ---- expand, level by level ----
    int n = 1;                                      // decision nodes of level d
    int n_chance = 0;
    int64_t off = 0, width = 1;                     // off(d), A^d
    for (int d = 0; d < H; ++d) {
        const int64_t off1 = off + width;
        // the scan: per-CTA sums over contiguous slices, then each slice rescanned from its CTA's base
        const int L = (n + G - 1) / G, lo = min(bid * L, n), hi = min(lo + L, n);
        int s = 0;
        for (int i = lo + tid; i < hi; i += THREADS) s += __ldcg(nd.nch + off + i);
        s = block_sum(s, red);
        if (tid == 0) a.part[bid] = s;
        barrier(a);
        int base = 0, m = 0;
        for (int b = tid; b < G; b += THREADS) {
            const int v = __ldcg(a.part + b);
            base += b < bid ? v : 0;
            m += v;
        }
        base = block_sum(base, red);
        m = block_sum(m, red);
        if (gtid == 0) a.lvl_n[d + 1] = m;
        for (int i0 = lo; i0 < hi; i0 += THREADS) {
            const int i = i0 + tid;
            const int k = i < hi ? __ldcg(nd.nch + off + i) : 0;
            int tile;
            const int e = base + block_scan(k, red, tile);
            if (i < hi) {
                nd.first[off + i] = e;
                const int choice = __ldcg(nd.st + off + i);
                for (int c = 0; c < k; ++c) {
                    nd.par[off1 + e + c] = i;
                    nd.act[off1 + e + c] = action_of<HW>(choice, c);
                }
            }
            base += tile;
        }
        barrier(a);
        // one transition per chance node: ChanceNode.estimateQ's C samples, all of which reach the same child
        const bool inner = d + 1 < H;
        if (HW) {
            // both halves of a warp step together (an odd count is padded with a discarded item) on warp-uniform
            // loop conditions: the step runs in its full-warp mode (two scenes, one mask), with no divergence guard
            // on its collectives
            const int lane = tid & 31, li = lane & 15, half = lane >> 4;
            const int32_t* src = a.scenes + (int64_t)(d & 1) * a.scene_level * hw::WORDS;
            int32_t* dst = a.scenes + (int64_t)((d + 1) & 1) * a.scene_level * hw::WORDS;
            const int w0 = gtid >> 5, nw = n_threads >> 5;
            for (int p = w0; __all_sync(0xffffffffu, 2 * p < m); p += nw) {
                const int item = 2 * p + half;
                const bool live = item < m;
                const int j = live ? item : 2 * p;
                const int parent = __ldcg(nd.par + off1 + j), action = __ldcg(nd.act + off1 + j);
                hw::Lane Ln;
                int t, si;
                hw::load_state(src + (int64_t)parent * hw::WORDS, li, Ln, t, si);
                bool term, trunc;                   // `done` is ignored (:81)
                const float r = hw::step(Ln, li, t, si, action, term, trunc, 0xffffffffu);
                int mask = 0;
                if (inner) {
                    if (live) hw::store_state(dst + (int64_t)j * hw::WORDS, li, Ln, t, si);
                    mask = hw::avail_mask(__shfl_sync(0xffffffffu, Ln.y, 0, 16), si);
                }
                if (live && li == 0) {
                    nd.rew[off1 + j] = (double)r;
                    nd.st[off1 + j] = mask;
                    nd.nch[off1 + j] = __popc(mask);
                }
            }
        } else {
            const b2_finite_mdp_sampled& mdp = a.cfg.mdp;
            for (int j = gtid; j < m; j += n_threads) {
                const int64_t row = (int64_t)__ldcg(nd.st + off + __ldcg(nd.par + off1 + j)) * A +
                                    __ldcg(nd.act + off1 + j);
                nd.st[off1 + j] = mdp.next[row];
                nd.rew[off1 + j] = mdp.reward[row];      // every sample's reward is R[s, a]
                nd.nch[off1 + j] = inner ? A : 0;
            }
        }
        barrier(a);
        n_chance += m;
        n = m;
        off = off1;
        width *= A;
    }

    // ---- values and subtree sizes, bottom-up ----
    for (int d = H - 1; d >= 0; --d) {
        const int64_t off_d = level_off(A, d), off1 = level_off(A, d + 1);
        const bool inner = d + 1 < H;
        const int n_d = __ldcg(a.lvl_n + d);
        for (int i = gtid; i < n_d; i += n_threads) {
            const int k = __ldcg(nd.nch + off_d + i), f = __ldcg(nd.first + off_d + i);
            double best = 0.0;
            int size = 1;
            for (int c = 0; c < k; ++c) {
                const int64_t j = off1 + f + c;
                double S = 0.0;                     // sum(...) starts from int 0: 0 + x == 0.0 + x
                int sub = 1;
                if (inner) {
                    S = 0.0 + __ldcg(nd.val + j) * (double)C;
                    sub = __ldcg(nd.size + j);
                }
                const double q = __ldcg(nd.rew + j) + a.cfg.gamma * S / (double)C;   // ChanceNode.value, :87-88
                nd.q[j] = q;
                if (d == 0) a.root_q[__ldcg(nd.act + j)] = q;
                if (c == 0 || q > best) best = q;   // np.amax: the first maximum
                size += 1 + sub;
            }
            nd.val[off_d + i] = best;               // DecisionNode.value, :51
            nd.size[off_d + i] = size;
        }
        barrier(a);
    }
    const int total = __ldcg(nd.size);
    const bool rec = tr.capacity > 0, fits = !rec || total <= tr.capacity;

    // ---- finish: the stream after every sample, then get_plan's tie-break ----
    if (gtid == 0) {
        Pcg64 rng;
        rng.load(a.rng);
        rng.skip32((uint64_t)C * (uint64_t)n_chance);
        int action = -1;
        if (fits) {
            const int root_choice = nd.st[0];
            action = ss::root_plan(a.root_q, nd.nch[0], [&](int i) { return action_of<HW>(root_choice, i); }, rng);
        }
        rng.store(a.rng);
        a.plan[0] = (int8_t)action;
        int32_t* res = a.result;
        res[0] = total;
        res[1] = n_chance;
        res[2] = C * n_chance;
        res[3] = action;
        res[4] = fits ? 0 : ss::ERR_CAPACITY;
        res[5] = -1;
        res[6] = 0;
        res[7] = 0;
    }
    if (!rec || !fits) return;

    // ---- creation-order ids and the dump, top-down ----
    if (gtid == 0) {
        ss::put(tr, 0, 0, -1, ss::KIND_DECISION, -1, 0);
        tr.value[0] = nd.val[0];
        nd.id[0] = 0;
    }
    for (int d = 0; d < H; ++d) {
        barrier(a);
        const int64_t off_d = level_off(A, d), off1 = level_off(A, d + 1);
        const bool inner = d + 1 < H;
        const int n_d = __ldcg(a.lvl_n + d);
        for (int i = gtid; i < n_d; i += n_threads) {
            const int k = __ldcg(nd.nch + off_d + i), f = __ldcg(nd.first + off_d + i);
            const int D = __ldcg(nd.id + off_d + i);
            int c = D + 1;
            for (int x = 0; x < k; ++x) {
                const int64_t j = off1 + f + x;
                ss::put(tr, 0, c, D, ss::KIND_CHANCE, __ldcg(nd.act + j), d);
                tr.value[c] = __ldcg(nd.q + j);
                ss::put(tr, 0, c + 1, c, ss::KIND_DECISION, HW ? -1 : __ldcg(nd.st + j), d + 1);
                tr.count[c + 1] = C;
                if (inner) {
                    tr.value[c + 1] = __ldcg(nd.val + j);
                    nd.id[j] = c + 1;
                }
                c += 1 + (inner ? __ldcg(nd.size + j) : 1);         // the chance node, then the child's subtree
            }
        }
    }
}

}  // namespace sslev
}  // namespace b2

using namespace b2;

// The worst case fits int32 node ids: A^0 + ... + A^H decision and A^1 + ... + A^H chance nodes.
static bool levels_config_ok(const b2_sparse_sampling_config* cfg) {
    if (!cfg || cfg->n_trees != 1 || cfg->horizon < 1 || cfg->C < 1 || cfg->n_actions < 1 || cfg->n_actions >= 128)
        return false;
    int64_t nodes = 0, p = 1;
    for (int d = 0; d <= cfg->horizon; ++d) {
        nodes += d == 0 ? 1 : 2 * p;
        if (nodes > INT32_MAX) return false;
        if (d < cfg->horizon) p *= cfg->n_actions;
    }
    return (int64_t)cfg->C * (nodes / 2) <= INT32_MAX;      // samples drawn
}

extern "C" int64_t b2_sparse_sampling_levels_workspace_bytes(const b2_sparse_sampling_config* cfg) {
    if (!levels_config_ok(cfg)) return 0;
    return (int64_t)sslev::make_layout(cfg).total;
}

extern "C" int b2_sparse_sampling_plan_levels(const b2_sparse_sampling_config* cfg, const int32_t* root_states,
                                              const b2_sparse_sampling_tree* tree, void* workspace, uint64_t* rng,
                                              double* root_q, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_states && workspace && rng && root_q && plan && result, "null pointer");
    B2_REQUIRE(cfg->n_trees == 1, "the level-synchronous search plans one decision (n_trees 1)");
    B2_REQUIRE(cfg->horizon >= 1 && cfg->C >= 1, "horizon and C must be >= 1");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions < 128, "n_actions must be in 1..127");
    const int rc = check_env_kind(cfg->env_kind, cfg->n_actions);
    if (rc != B2_OK) return rc;
    B2_REQUIRE(levels_config_ok(cfg), "the worst-case tree does not fit int32 node ids");
    sslev::Args a;
    a.cfg = *cfg;
    a.tree = b2_sparse_sampling_tree{};
    if (tree) {
        B2_REQUIRE(tree->capacity >= 1 && tree->parent && tree->kind && tree->key && tree->depth && tree->count &&
                   tree->value, "tree dump arrays missing");
        a.tree = *tree;
    }
    if (cfg->env_kind == B2_ENV_FINITE) {
        const b2_finite_mdp_sampled& m = cfg->mdp;
        B2_REQUIRE(m.next && m.reward, "finite MDP tables missing");
        B2_REQUIRE(m.n_actions == cfg->n_actions && m.n_states > 0, "bad finite MDP shape");
        B2_REQUIRE(m.n_next == 1, "the level-synchronous search needs a deterministic finite MDP (n_next 1)");
    }
    const sslev::Layout l = sslev::make_layout(cfg);
    char* ws = (char*)workspace;
    a.ctl = (sslev::Control*)(ws + l.ctl);
    a.part = (int32_t*)(ws + l.part);
    a.lvl_n = (int32_t*)(ws + l.lvl_n);
    int32_t** ints[7] = {&a.n.st, &a.n.nch, &a.n.first, &a.n.par, &a.n.act, &a.n.size, &a.n.id};
    for (int i = 0; i < 7; ++i) *ints[i] = (int32_t*)(ws + l.nodes[i]);
    a.n.rew = (double*)(ws + l.nodes[7]);
    a.n.val = (double*)(ws + l.nodes[8]);
    a.n.q = (double*)(ws + l.nodes[9]);
    a.scenes = (int32_t*)(ws + l.scenes);
    a.scene_level = l.scene_level;
    a.root_states = root_states; a.rng = rng; a.root_q = root_q; a.plan = plan; a.result = result;
    cudaStream_t stream = (cudaStream_t)stream_;
    B2_CUDA_CHECK(cudaMemsetAsync(a.ctl, 0, sizeof(sslev::Control), stream));
    const void* fn = cfg->env_kind == B2_ENV_HIGHWAY ? (const void*)sslev::sparse_sampling_levels_kernel<true>
                                                     : (const void*)sslev::sparse_sampling_levels_kernel<false>;
    int per_sm = 0;
    B2_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, sslev::THREADS, 0));
    B2_REQUIRE(per_sm >= 1, "level kernel does not fit on an SM");
    int grid = per_sm * sm_count();
    if (grid > sslev::MAX_CTAS) grid = sslev::MAX_CTAS;
    void* params[] = {&a};
    B2_CUDA_CHECK(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(sslev::THREADS), params, 0, stream));
    return B2_OK;
}
