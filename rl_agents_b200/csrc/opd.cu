// OPD (optimistic planning for deterministic systems) -- the plan() loop of
// OptimisticDeterministicPlanner (rl_agents/agents/tree_search/deterministic.py)
// for a BATCH of independent decisions: one search tree per CTA, the node
// order inside each tree exactly the reference's (strict best-first).
//
// GPU-first restructuring of the reference loop (:106-122):
//   * the frontier `max(self.leaves, key=upper)` (:110, O(n) per expansion,
//     65 % of the reference's time) becomes a radix-32 tournament tree over
//     value_upper keyed by node id: select = one descent, update = three
//     leaf-to-root refreshes.  Python's max() returns the FIRST maximal leaf in
//     list order, which is creation order = lowest node id: the descent takes
//     the lowest lane among equal maxima at every level.
//   * `safe_deepcopy_env` + `env.step` for every child (:36-43) is the batched
//     transition kernel (finite-MDP table gather, or hw::step with the scene in
//     registers); child states live in an HBM arena indexed by node id.
//   * backup_to_root (:74-79) and the count walk (:64-65) never influence which
//     leaf is expanded (only leaf bounds do, and they are final at creation),
//     so they leave the sequential loop: one bottom-up pass in reverse
//     expansion order reproduces value_lower / value_upper / count of every
//     node exactly (max and integer sums are order independent).
#include "common.cuh"
#include "highway_lite.cuh"
#include "lane_env.cuh"

namespace b2 {

constexpr int MAX_LEVELS = 6;          // 32^6 nodes
constexpr int MAX_BRANCH = 8;

struct LevelLayout {
    int n_levels;                      // keys = level 0
    int size[MAX_LEVELS];              // entries per level
    int64_t offset[MAX_LEVELS];        // in doubles, inside smem or the per-tree workspace
    int in_smem[MAX_LEVELS];
    int64_t ws_doubles;                // per-tree workspace doubles (global levels)
    int64_t ws_bytes_per_tree;         // + expansion order
    int smem_doubles;
};

struct OpdArgs {
    b2_opd_config cfg;
    b2_opd_tree tree;
    const int32_t* root_states;
    char* workspace;
    int8_t* plan;
    int32_t* result;
    LevelLayout lay;
};

struct Tournament {
    double* lvl[MAX_LEVELS];
    int size[MAX_LEVELS];
    int n_levels;

    __device__ __forceinline__ double get(int l, int i) const { return i < size[l] ? lvl[l][i] : -INFINITY; }

    // lowest node id among the leaves of maximal key (warp-collective)
    __device__ int select(int lane) const {
        const int top = n_levels - 1;
        double v = get(top, lane);
        const double m = warp_max_f64(v);
        int idx = __ffs(__ballot_sync(0xffffffffu, v == m)) - 1;
        for (int l = top - 1; l >= 0; --l) {
            v = get(l, idx * 32 + lane);
            idx = idx * 32 + __ffs(__ballot_sync(0xffffffffu, v == m)) - 1;
        }
        return idx;
    }

    // refresh the ancestors of key i after it changed (warp-collective)
    __device__ void update(int i, int lane) {
        for (int l = 0; l + 1 < n_levels; ++l) {
            const int g = i >> 5;
            const double m = warp_max_f64(get(l, g * 32 + lane));
            if (lane == 0) lvl[l + 1][g] = m;
            __syncwarp();
            i = g;
        }
    }
};

struct Shared {
    int leaf, depth, error, done_parent;
    double lower;
    int child_action[MAX_BRANCH];
    int child_done[MAX_BRANCH];
    double child_reward[MAX_BRANCH];
};

__device__ __forceinline__ void setup_tournament(Tournament& T, const LevelLayout& lay, double* smem_d, double* ws_d) {
    T.n_levels = lay.n_levels;
    for (int l = 0; l < lay.n_levels; ++l) {
        T.size[l] = lay.size[l];
        T.lvl[l] = (lay.in_smem[l] ? smem_d : ws_d) + lay.offset[l];
    }
}

// Writes the node records of the new children, retires the expanded leaf from
// the frontier and refreshes the tournament.  Called by warp 0 only.
__device__ __forceinline__ void commit_expansion(const OpdArgs& a, Tournament& T, Shared& sh, int64_t nb, int leaf,
                                                 int c0, int n, int it, int32_t* exp_order, int lane) {
    const b2_opd_tree& tr = a.tree;
    const int d = sh.depth + 1;
    if (lane < n) {
        const int c = c0 + lane;
        const double r = sh.child_reward[lane];
        const bool done = sh.child_done[lane] != 0;
        // DeterministicNode.update (deterministic.py:52-63)
        double lo = sh.lower + a.cfg.gamma_pow[d - 1] * r;
        double up = lo + a.cfg.gamma_pow_div[d];
        if (done) {
            lo = lo + a.cfg.terminal_bonus[d];
            up = lo;
        }
        tr.parent[nb + c] = leaf;
        tr.first_child[nb + c] = -1;
        tr.depth[nb + c] = d;
        tr.count[nb + c] = 2;   // 1 at creation (:18) + 1 for its own update (:64-65)
        tr.meta[nb + c] = sh.child_action[lane] | (done ? 1 << 16 : 0);
        tr.reward[nb + c] = r;
        tr.lower[nb + c] = lo;
        tr.upper[nb + c] = up;
        T.lvl[0][c] = up;
        if (!(r >= 0.0 && r <= 1.0)) sh.error = 1;   // :46-47
    }
    if (lane == 0) {
        T.lvl[0][leaf] = -INFINITY;
        tr.first_child[nb + leaf] = c0;
        tr.meta[nb + leaf] |= n << 8;
        exp_order[it] = leaf;
    }
    __syncwarp();
    T.update(leaf, lane);
    T.update(c0, lane);
    if (((c0 + n - 1) >> 5) != (c0 >> 5)) T.update(c0 + n - 1, lane);
}

// Bottom-up pass in reverse expansion order + greedy plan.  Warp 0 only.
__device__ void finish_tree(const OpdArgs& a, int64_t nb, int tree_id, int n_nodes, int n_exp, int max_depth,
                            int term_exp, int error, const int32_t* exp_order, int lane) {
    const b2_opd_tree& tr = a.tree;
    for (int k = n_exp - 1; k >= 0; --k) {
        const int p = exp_order[k];
        const int fc = tr.first_child[nb + p];
        const int n = (tr.meta[nb + p] >> 8) & 0xff;
        double lo = -INFINITY, up = -INFINITY;
        int desc = 0;
        if (lane < n) {
            lo = tr.lower[nb + fc + lane];
            up = tr.upper[nb + fc + lane];
            desc = tr.count[nb + fc + lane] - 1;
        }
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {   // MAX_BRANCH = 8 lanes
            const double lo2 = __shfl_xor_sync(0xffffffffu, lo, o);
            const double up2 = __shfl_xor_sync(0xffffffffu, up, o);
            lo = lo2 > lo ? lo2 : lo;
            up = up2 > up ? up2 : up;
            desc += __shfl_xor_sync(0xffffffffu, desc, o);
        }
        if (lane == 0) {
            tr.lower[nb + p] = lo;       // backup_to_root (:74-79)
            tr.upper[nb + p] = up;
            tr.count[nb + p] = (p == 0 ? 1 : 2) + desc;
        }
        __syncwarp();
    }
    // get_plan (abstract.py:143-156) on value_lower; a tie needs the planner RNG
    // (abstract.py:304-311): stop there and let the host finish the walk.
    int8_t* plan = a.plan + (int64_t)tree_id * a.cfg.plan_capacity;
    int node = 0, len = 0, tie_node = -1;
    while (true) {
        const int fc = tr.first_child[nb + node];
        if (fc < 0) break;
        const int n = (tr.meta[nb + node] >> 8) & 0xff;
        double lo = lane < n ? tr.lower[nb + fc + lane] : -INFINITY;
        const double m = warp_max_f64(lo);
        const unsigned eq = __ballot_sync(0xffffffffu, lane < n && lo == m);
        if (__popc(eq) > 1) { tie_node = node; break; }
        const int c = fc + __ffs(eq) - 1;
        if (lane == 0 && len < a.cfg.plan_capacity) plan[len] = (int8_t)(tr.meta[nb + c] & 0xff);
        ++len;
        node = c;
    }
    if (lane == 0) {
        int32_t* res = a.result + (int64_t)tree_id * B2_OPD_RESULT_WORDS;
        res[0] = n_nodes;
        res[1] = n_nodes - n_exp;
        res[2] = max_depth;
        res[3] = term_exp;
        res[4] = error;
        res[5] = len;
        res[6] = tie_node;
    }
}

__device__ __forceinline__ void init_tree(const OpdArgs& a, Tournament& T, int64_t nb, int tid, int nthreads) {
    for (int l = 0; l < T.n_levels; ++l)
        for (int i = tid; i < T.size[l]; i += nthreads) T.lvl[l][i] = (i == 0) ? 0.0 : -INFINITY;
    if (tid == 0) {   // DeterministicNode.__init__ (:10-19)
        const b2_opd_tree& tr = a.tree;
        tr.parent[nb] = -1;
        tr.first_child[nb] = -1;
        tr.depth[nb] = 0;
        tr.count[nb] = 1;
        tr.meta[nb] = 0xff;   // no action
        tr.reward[nb] = 0.0;
        tr.lower[nb] = 0.0;
        tr.upper[nb] = 0.0;
    }
}

// ---------------------------------------------------------------------------
// finite deterministic MDP: one warp per tree, lane a expands action a
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(32) opd_finite_kernel(OpdArgs a) {
    extern __shared__ double smem_d[];
    __shared__ Shared sh;
    const int tree_id = blockIdx.x, lane = threadIdx.x;
    const int64_t nb = (int64_t)tree_id * a.cfg.node_capacity;
    char* ws = a.workspace + (int64_t)tree_id * a.lay.ws_bytes_per_tree;
    Tournament T;
    setup_tournament(T, a.lay, smem_d, (double*)ws);
    int32_t* exp_order = (int32_t*)(ws + a.lay.ws_doubles * 8);
    init_tree(a, T, nb, lane, 32);
    if (lane == 0) {
        a.tree.state[nb] = a.root_states[tree_id];
        sh.error = 0;
    }
    __syncwarp();
    const b2_finite_mdp& m = a.cfg.mdp;
    const int A = a.cfg.n_actions;
    int n_nodes = 1, max_depth = 0, term_exp = 0, it = 0;
    for (; it < a.cfg.n_expansions; ++it) {
        const int leaf = T.select(lane);
        const int s = a.tree.state[nb + leaf];
        if (lane == 0) {
            sh.depth = a.tree.depth[nb + leaf];
            sh.lower = a.tree.lower[nb + leaf];
            sh.done_parent = (a.tree.meta[nb + leaf] >> 16) & 1;
        }
        if (lane < A) {   // deterministic.py:36-43 for action `lane`
            const int s2 = m.transition[(int64_t)s * A + lane];
            sh.child_reward[lane] = m.reward[(int64_t)s * A + lane];
            sh.child_done[lane] = m.terminal[s];   // finite_mdp's MDP.step: done = terminal[state BEFORE the transition]
            sh.child_action[lane] = lane;
            a.tree.state[nb + n_nodes + lane] = s2;
        }
        __syncwarp();
        term_exp += sh.done_parent;
        max_depth = max(max_depth, sh.depth + 1);
        commit_expansion(a, T, sh, nb, leaf, n_nodes, A, it, exp_order, lane);
        n_nodes += A;
        __syncwarp();
        if (sh.error) { ++it; break; }
    }
    finish_tree(a, nb, tree_id, n_nodes, it, max_depth, term_exp, sh.error, exp_order, lane);
}

// ---------------------------------------------------------------------------
// HighwayLite: 3 warps per tree; each 16-lane group simulates one child
// ---------------------------------------------------------------------------
constexpr int HW_THREADS = 96;

__global__ void __launch_bounds__(HW_THREADS) opd_highway_kernel(OpdArgs a) {
    extern __shared__ double smem_d[];
    __shared__ Shared sh;
    const int tree_id = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int grp = tid >> 4, li = tid & 15;
    const int64_t nb = (int64_t)tree_id * a.cfg.node_capacity;
    char* ws = a.workspace + (int64_t)tree_id * a.lay.ws_bytes_per_tree;
    Tournament T;
    setup_tournament(T, a.lay, smem_d, (double*)ws);
    int32_t* exp_order = (int32_t*)(ws + a.lay.ws_doubles * 8);
    int32_t* states = a.tree.state + nb * hw::WORDS;
    init_tree(a, T, nb, tid, HW_THREADS);
    for (int i = tid; i < hw::WORDS; i += HW_THREADS) states[i] = a.root_states[(int64_t)tree_id * hw::WORDS + i];
    if (tid == 0) sh.error = 0;
    __syncthreads();
    int n_nodes = 1, max_depth = 0, term_exp = 0, it = 0;
    for (; it < a.cfg.n_expansions; ++it) {
        if (warp == 0) {
            const int leaf = T.select(lane);
            if (lane == 0) {
                sh.leaf = leaf;
                sh.depth = a.tree.depth[nb + leaf];
                sh.lower = a.tree.lower[nb + leaf];
                sh.done_parent = (a.tree.meta[nb + leaf] >> 16) & 1;
            }
        }
        __syncthreads();
        const int leaf = sh.leaf;
        // "deep copy" of the parent scene into registers (deterministic.py:38)
        hw::Lane L;
        int t, si;
        hw::load_state(states + (int64_t)leaf * hw::WORDS, li, L, t, si);
        const float ego_y = __shfl_sync(0xffffffffu, L.y, 0, 16);
        const int mask = hw::avail_mask(ego_y, si);
        const int n = __popc(mask);
        const int action = grp < n ? hw::nth_action(mask, grp) : hw::A_IDLE;
        bool term, trunc;
        const float r = hw::step(L, li, t, si, action, term, trunc, 0xffffffffu);
        if (grp < n) {
            hw::store_state(states + (int64_t)(n_nodes + grp) * hw::WORDS, li, L, t, si);
            if (li == 0) {
                sh.child_reward[grp] = (double)r;
                sh.child_done[grp] = term ? 1 : 0;
                sh.child_action[grp] = action;
            }
        }
        __syncthreads();
        term_exp += sh.done_parent;
        max_depth = max(max_depth, sh.depth + 1);
        if (warp == 0) commit_expansion(a, T, sh, nb, leaf, n_nodes, n, it, exp_order, lane);
        n_nodes += n;
        __syncthreads();
        if (sh.error) { ++it; break; }
    }
    if (warp == 0) finish_tree(a, nb, tree_id, n_nodes, it, max_depth, term_exp, sh.error, exp_order, lane);
}

// ---------------------------------------------------------------------------
// HighwayLite, batched: 8 trees per CTA (one warp owns one tree for select /
// commit / finish); the children of all 8 expansions of an iteration are packed
// densely onto the CTA's 16 half-warp groups, so that ~94 % of the simulation
// slots do real work (a lone tree fills 3.8 of its 6 slots).  Node order inside
// every tree is unchanged: the trees are independent, only the slots are shared.
// ---------------------------------------------------------------------------
#ifndef B2_MT_TREES
#define B2_MT_TREES 8
#endif
constexpr int MT_TREES = B2_MT_TREES;
constexpr int MT_THREADS = 32 * MT_TREES;
constexpr int MT_GROUPS = MT_THREADS / 16;

struct MultiShared {
    Shared sh[MT_TREES];
    int n[MT_TREES];          // children of this iteration's expansion (0: tree idle / dead)
    int mask[MT_TREES];       // available-action mask of the expanded leaf
    int n_nodes[MT_TREES], max_depth[MT_TREES], term_exp[MT_TREES], n_exp[MT_TREES], dead[MT_TREES];
};

#ifndef B2_MT_MIN_BLOCKS
#define B2_MT_MIN_BLOCKS 4   // 64 registers: 4 CTAs = 32 warps per SM (H100: 43.4M vs 42.0M expansions/s at 3)
#endif
__global__ void __launch_bounds__(MT_THREADS, B2_MT_MIN_BLOCKS) opd_highway_multi_kernel(OpdArgs a) {
    extern __shared__ double smem_d[];
    __shared__ MultiShared ms;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, li = tid & 15;
    int grp = tid >> 4;
    asm volatile("" : "+r"(grp));   // keep in a register (else re-derived from SR_TID.X)
    const int tree0 = blockIdx.x * MT_TREES;
    const int n_local = min(MT_TREES, a.cfg.n_trees - tree0);
    // the warp's own tree
    const int my_tree = tree0 + warp;
    // warp-uniform conditions are taken through votes: ptxas then knows the branches cannot split the warp and drops the
    // divergence guards (BRA.DIV / WARPSYNC) around every collective in the regions they control
    const bool owner = __all_sync(0xffffffffu, warp < n_local);
    const int64_t my_nb = (int64_t)my_tree * a.cfg.node_capacity;
    char* my_ws = a.workspace + (int64_t)(owner ? my_tree : tree0) * a.lay.ws_bytes_per_tree;
    Tournament T;
    setup_tournament(T, a.lay, smem_d + (size_t)warp * a.lay.smem_doubles, (double*)my_ws);
    int32_t* my_exp_order = (int32_t*)(my_ws + a.lay.ws_doubles * 8);
    if (owner) {
        init_tree(a, T, my_nb, lane, 32);
        int32_t* st = a.tree.state + my_nb * hw::WORDS;
        for (int i = lane; i < hw::WORDS; i += 32) st[i] = a.root_states[(int64_t)my_tree * hw::WORDS + i];
    }
    if (lane == 0) {
        ms.sh[warp].error = 0;
        ms.n[warp] = 0;
        ms.n_nodes[warp] = 1; ms.max_depth[warp] = 0; ms.term_exp[warp] = 0; ms.n_exp[warp] = 0;
        ms.dead[warp] = owner ? 0 : 1;
    }
    __syncthreads();
    for (int it = 0; it < a.cfg.n_expansions; ++it) {
        // ---- phase 1: every warp selects the leaf of its own tree ----
        const bool alive = __all_sync(0xffffffffu, ms.dead[warp] == 0);
        if (alive) {
            const int leaf = T.select(lane);
            if (lane == 0) {
                Shared& sh = ms.sh[warp];
                sh.leaf = leaf;
                sh.depth = a.tree.depth[my_nb + leaf];
                sh.lower = a.tree.lower[my_nb + leaf];
                sh.done_parent = (a.tree.meta[my_nb + leaf] >> 16) & 1;
                const int32_t* w = a.tree.state + (my_nb + leaf) * hw::WORDS;
                const int mask = hw::avail_mask(__int_as_float(w[hw::V]), w[8 * hw::V + 1]);
                ms.mask[warp] = mask;
                ms.n[warp] = __popc(mask);
            }
        } else if (lane == 0) {
            ms.n[warp] = 0;
        }
        __syncthreads();
        // ---- phase 2: pack the children of all trees onto the groups ----
        int offs[MT_TREES + 1];
        offs[0] = 0;
#pragma unroll
        for (int u = 0; u < MT_TREES; ++u) offs[u + 1] = offs[u] + ms.n[u];
        const int total = offs[MT_TREES];
        for (int base = 0; base < total; base += MT_GROUPS) {
            if (__all_sync(0xffffffffu, base + 2 * warp >= total)) continue;   // neither group of this warp has work (vote: provably warp-uniform branch)
            const int slot = base + grp;
            const bool real = slot < total;
            int tr = 0;
#pragma unroll
            for (int u = 1; u < MT_TREES; ++u) tr += (real && slot >= offs[u]) ? 1 : 0;
            const int k = real ? slot - offs[tr] : 0;
            const int64_t nb = (int64_t)(tree0 + tr) * a.cfg.node_capacity;
            int32_t* states = a.tree.state + nb * hw::WORDS;
            const Shared& sh = ms.sh[tr];
            hw::Lane L;
            int t, si;
            hw::load_state(states + (int64_t)sh.leaf * hw::WORDS, li, L, t, si);
            const int action = real ? hw::nth_action(ms.mask[tr], k) : hw::A_IDLE;
            bool term, trunc;
            const float r = hw::step(L, li, t, si, action, term, trunc, 0xffffffffu);
            if (real) {
                hw::store_state(states + (int64_t)(ms.n_nodes[tr] + k) * hw::WORDS, li, L, t, si);
                if (li == 0) {
                    ms.sh[tr].child_reward[k] = (double)r;
                    ms.sh[tr].child_done[k] = term ? 1 : 0;
                    ms.sh[tr].child_action[k] = action;
                }
            }
        }
        __syncthreads();
        // ---- phase 3: every warp commits its own tree ----
        if (alive) {
            Shared& sh = ms.sh[warp];
            const int n = ms.n[warp], c0 = ms.n_nodes[warp];
            commit_expansion(a, T, sh, my_nb, sh.leaf, c0, n, ms.n_exp[warp], my_exp_order, lane);
            __syncwarp();
            if (lane == 0) {
                ms.term_exp[warp] += sh.done_parent;
                ms.max_depth[warp] = max(ms.max_depth[warp], sh.depth + 1);
                ms.n_nodes[warp] = c0 + n;
                ms.n_exp[warp] += 1;
                if (sh.error) ms.dead[warp] = 1;      // deterministic.py:46-47 raises: stop this tree
            }
            __syncwarp();
        }
    }
    if (owner)
        finish_tree(a, my_nb, my_tree, ms.n_nodes[warp], ms.n_exp[warp], ms.max_depth[warp], ms.term_exp[warp],
                    ms.sh[warp].error, my_exp_order, lane);
}

// ---------------------------------------------------------------------------
// batched env transition (b2_highway_step): one scene per 16-lane group
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(128) highway_step_kernel(int32_t* states, const int32_t* actions, float* reward,
                                                           int32_t* flags, int32_t* avail, int n_envs) {
    const int g = (blockIdx.x * 128 + threadIdx.x) >> 4, li = threadIdx.x & 15;
    const bool live = g < n_envs;
    const int e = live ? g : n_envs - 1;
    hw::Lane L;
    int t, si;
    hw::load_state(states + (int64_t)e * hw::WORDS, li, L, t, si);
    bool term, trunc;
    const float r = hw::step(L, li, t, si, actions[e], term, trunc, 0xffffffffu);
    const float ego_y = __shfl_sync(0xffffffffu, L.y, 0, 16);
    if (live) {
        hw::store_state(states + (int64_t)e * hw::WORDS, li, L, t, si);
        if (li == 0) {
            reward[e] = r;
            flags[e] = (term ? 1 : 0) | (trunc ? 2 : 0);
            if (avail) avail[e] = hw::avail_mask(ego_y, si);
        }
    }
}

// Exhaustive check of hw::div_const against the IEEE division for the two constant divisors of the spec:
// every fp32 mantissa, both signs, exponents -60 .. +60 (quotients stay normal); and of hw::div_fast against the
// `/` operator on 2^33 operand pairs (every numerator mantissa x 1024 hashed divisors of either sign, both
// magnitudes in 2^-40 .. 2^40), and of hw::div_nz on the same pairs and on zero numerators of either sign; and of
// hw::sqrt_fast against sqrtf on every value of [2^-3, 2); and of hw::lane_of against clip(rint(y / 4), 0, 3) on every
// fp32 bit pattern.  Counts mismatching bit patterns.
__global__ void const_division_selftest_kernel(unsigned long long* mismatches) {
    const unsigned m = blockIdx.x * blockDim.x + threadIdx.x;       // mantissa, 2^23 threads
    unsigned long long bad = 0;
    for (int e = 127 - 60; e <= 127 + 60; e += 3) {
        for (unsigned sgn = 0; sgn < 2; ++sgn) {
            const float x = __uint_as_float((sgn << 31) | ((unsigned)e << 23) | m);
            const float a = x / hw::TWO_SQRT_AB, b = hw::div_const(x, hw::TWO_SQRT_AB, hw::RCP_TWO_SQRT_AB);
            const float c = x / hw::HALF_LENGTH, d = hw::div_const(x, hw::HALF_LENGTH, hw::RCP_HALF_LENGTH);
            bad += (__float_as_uint(a) != __float_as_uint(b)) + (__float_as_uint(c) != __float_as_uint(d));
        }
    }
    for (unsigned e = 124; e <= 127; ++e) {      // hw::sqrt_fast on every fp32 value of [2^-3, 2)
        float x = __uint_as_float((e << 23) | m);
        asm volatile("" : "+f"(x));
        bad += __float_as_uint(sqrtf(x)) != __float_as_uint(hw::sqrt_fast(x));
    }
    for (unsigned hi = 0; hi < 512; ++hi) {      // hw::lane_of on all 2^32 bit patterns (NaN and +-inf included)
        float y = __uint_as_float((hi << 23) | m);
        asm volatile("" : "+f"(y));
        bad += (int)fminf(fmaxf(rintf(y / hw::LANE_W), 0.0f), 3.0f) != hw::lane_of(y);
    }
    unsigned long long h = 0x9e3779b97f4a7c15ull * (m + 1);
    for (int it = 0; it < 1024; ++it) {
        h ^= h >> 30; h *= 0xbf58476d1ce4e5b9ull; h ^= h >> 27; h *= 0x94d049bb133111ebull; h ^= h >> 31;
        const unsigned ea = 127 - 40 + (unsigned)(h >> 56) % 81u, eb = 127 - 40 + (unsigned)((h >> 48) & 0xff) % 81u;
        const float x = __uint_as_float((((unsigned)(h >> 47) & 1u) << 31) | (ea << 23) | m);
        float y = __uint_as_float((((unsigned)(h >> 46) & 1u) << 31) | (eb << 23) | ((unsigned)h & 0x7fffffu));
        asm volatile("" : "+f"(y));      // opaque: the reference quotient below is the compiler's own division
        const float q = x / y, f = hw::div_fast(x, y);
        bad += __float_as_uint(q) != __float_as_uint(f);
        bad += __float_as_uint(q) != __float_as_uint(hw::div_nz(x, y));
        const float z = __uint_as_float(((unsigned)(h >> 45) & 1u) << 31);     // +0 or -0
        bad += __float_as_uint(z / y) != __float_as_uint(hw::div_nz(z, y));
    }
    if (bad) atomicAdd(mismatches, bad);
}

// Test entry of hw::step in the per-group mode of the one-tree-per-group planners (mcts.cu, olop.cu, ...): scene s on
// its own 16-lane group through HighwayEnv::step with that group's gmask, n_steps[s] decisions each, so the two groups
// of a warp step different numbers of times.  Decision k of scene s reads actions[s * max_steps + k] and writes the new
// state to trace[(s * max_steps + k) * 136 ..] and reward / flags (bit0 terminated, bit1 truncated, avail mask << 2)
// to out[s * max_steps + k].
__global__ void __launch_bounds__(64) highway_step_groups_kernel(const int32_t* states, const int32_t* actions,
                                                                const int32_t* n_steps, int32_t* trace, float* reward,
                                                                int32_t* flags, int n_scenes, int max_steps) {
    const int lane = threadIdx.x & 31, li = lane & 15;
    const int s = (blockIdx.x * 64 + threadIdx.x) >> 4;
    if (s >= n_scenes) return;       // a whole group leaves: the other group of the warp works alone
    const unsigned gmask = 0xFFFFu << (lane & 16);
    HighwayEnv env;
    env.load_root(states, s, li);
    for (int k = 0; k < n_steps[s]; ++k) {
        const int64_t o = (int64_t)s * max_steps + k;
        bool term, trunc;
        double r;
        int bad_row;
        env.step(LaneModel{}, actions[o], li, gmask, true, term, trunc, r, bad_row);
        const int avail = env.avail(hw::A_SLOWER + 1, gmask);
        hw::store_state(trace + o * hw::WORDS, li, env.L, env.t, env.si);
        if (li == 0) {
            reward[o] = (float)r;
            flags[o] = (term ? 1 : 0) | (trunc ? 2 : 0) | (avail << 2);
        }
    }
}

static int make_layout(const b2_opd_config* cfg, LevelLayout* lay, int smem_budget_doubles) {
    int n = cfg->node_capacity, l = 0;
    lay->n_levels = 0;
    while (true) {
        if (l >= MAX_LEVELS) return -1;
        lay->size[l] = n;
        ++l;
        if (n <= 32) break;
        n = (n + 31) / 32;
    }
    lay->n_levels = l;
    // upper levels are the hottest: place from the top down while they fit
    int64_t smem_used = 0, ws_used = 0;
    for (int k = l - 1; k >= 0; --k) {
        const int64_t sz = (lay->size[k] + 1) & ~1;
        const bool want = (k > 0) || cfg->keys_in_smem;
        if (want && smem_used + sz <= smem_budget_doubles) {
            lay->in_smem[k] = 1;
            lay->offset[k] = smem_used;
            smem_used += sz;
        } else {
            lay->in_smem[k] = 0;
            lay->offset[k] = ws_used;
            ws_used += sz;
        }
    }
    lay->smem_doubles = (int)smem_used;
    lay->ws_doubles = ws_used;
    int64_t bytes = ws_used * 8 + (int64_t)cfg->n_expansions * 4;
    lay->ws_bytes_per_tree = (bytes + 127) & ~(int64_t)127;
    return 0;
}

}  // namespace b2

using namespace b2;

static const int kSmemBudgetDoubles = (96 * 1024) / 8;

extern "C" int64_t b2_opd_workspace_bytes(const b2_opd_config* cfg) {
    LevelLayout lay;
    if (!cfg || make_layout(cfg, &lay, kSmemBudgetDoubles)) return -1;
    return lay.ws_bytes_per_tree * (int64_t)cfg->n_trees;
}

extern "C" int b2_opd_plan(const b2_opd_config* cfg, const int32_t* root_states, const b2_opd_tree* tree,
                           void* workspace, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_states && tree && workspace && plan && result, "null pointer");
    B2_REQUIRE(cfg->reserved == 0, "b2_opd_config.reserved must be 0");
    B2_REQUIRE(cfg->n_trees > 0 && cfg->n_expansions >= 0, "bad batch / budget");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions <= MAX_BRANCH, "n_actions must be in 1..8");
    B2_REQUIRE((int64_t)cfg->node_capacity >= 1 + (int64_t)cfg->n_expansions * cfg->n_actions, "node_capacity too small");
    B2_REQUIRE(cfg->plan_capacity >= cfg->n_expansions + 1, "plan_capacity too small");
    B2_REQUIRE(cfg->gamma_pow && cfg->gamma_pow_div && cfg->terminal_bonus, "gamma tables missing");
    cudaStream_t stream = (cudaStream_t)stream_;
    OpdArgs a;
    a.cfg = *cfg; a.tree = *tree; a.root_states = root_states; a.workspace = (char*)workspace;
    a.plan = plan; a.result = result;
    if (make_layout(cfg, &a.lay, kSmemBudgetDoubles)) {
        set_error("node_capacity %d exceeds 32^%d", cfg->node_capacity, MAX_LEVELS);
        return B2_ERR_UNSUPPORTED;
    }
    const size_t smem = (size_t)a.lay.smem_doubles * 8;
    if (cfg->env_kind == B2_ENV_FINITE) {
        B2_REQUIRE(cfg->mdp.transition && cfg->mdp.reward && cfg->mdp.terminal, "finite MDP tables missing");
        B2_REQUIRE(cfg->mdp.n_actions == cfg->n_actions, "mdp.n_actions != n_actions");
        B2_CUDA_CHECK(cudaFuncSetAttribute(opd_finite_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        opd_finite_kernel<<<cfg->n_trees, 32, smem, stream>>>(a);
    } else if (cfg->env_kind == B2_ENV_HIGHWAY) {
        B2_REQUIRE(cfg->n_actions == B2_HW_ACTIONS, "HighwayLite has 5 actions");
        const size_t smem_multi = smem * MT_TREES;
        if (cfg->n_trees >= 2 * MT_TREES && smem_multi <= 64 * 1024) {
            // batch mode: 8 trees per CTA, children packed densely on the simulation slots
            B2_CUDA_CHECK(cudaFuncSetAttribute(opd_highway_multi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)smem_multi));
            opd_highway_multi_kernel<<<(cfg->n_trees + MT_TREES - 1) / MT_TREES, MT_THREADS, smem_multi, stream>>>(a);
        } else {
            // latency mode: one tree per CTA
            B2_CUDA_CHECK(cudaFuncSetAttribute(opd_highway_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            opd_highway_kernel<<<cfg->n_trees, HW_THREADS, smem, stream>>>(a);
        }
    } else {
        set_error("unknown env_kind %d", cfg->env_kind);
        return B2_ERR_INVALID;
    }
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_selftest_const_division(unsigned long long* mismatches_dev, void* stream) {
    B2_REQUIRE(mismatches_dev, "null pointer");
    B2_CUDA_CHECK(cudaMemsetAsync(mismatches_dev, 0, 8, (cudaStream_t)stream));
    const_division_selftest_kernel<<<(1u << 23) / 256, 256, 0, (cudaStream_t)stream>>>(mismatches_dev);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_selftest_highway_step_groups(const int32_t* states, const int32_t* actions, const int32_t* n_steps,
                                               int32_t* trace, float* reward, int32_t* flags, int32_t n_scenes,
                                               int32_t max_steps, void* stream) {
    B2_REQUIRE(states && actions && n_steps && trace && reward && flags && n_scenes > 0 && max_steps > 0,
               "null pointer / empty batch");
    highway_step_groups_kernel<<<(n_scenes + 3) / 4, 64, 0, (cudaStream_t)stream>>>(states, actions, n_steps, trace,
                                                                                    reward, flags, n_scenes, max_steps);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_highway_step(int32_t* states, const int32_t* actions, float* reward, int32_t* flags,
                               int32_t* avail_mask, int32_t n_envs, void* stream) {
    B2_REQUIRE(states && actions && reward && flags && n_envs > 0, "null pointer / empty batch");
    const int groups_per_block = 128 / 16;
    const int grid = (n_envs + groups_per_block - 1) / groups_per_block;
    highway_step_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(states, actions, reward, flags, avail_mask, n_envs);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
