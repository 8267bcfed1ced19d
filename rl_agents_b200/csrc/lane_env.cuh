// Device env models of the one-tree-per-lane-group planners (mcts.cu, olop.cu, mdp_gape.cu, brue.cu, mcts_dpw.cu): one
// tree per lane on a finite MDP, one tree per 16-lane group on HighwayLite and IntersectionLite (lane = vehicle slot, the
// scene in registers, so the reference's deep copy of the env is a register copy).  B2_LANE_MAP places a thread in
// its group; each model reads only what it needs: the launch's LaneModel, the root states and the action count.
//
// Every model has the same step(); it reports truncation separately; MCTS reads it, the other planners ignore it (the
// reference's 4-tuple step drops truncation).  seed() and load_rng() set the env generator of SampledFiniteEnv and do
// nothing on the deterministic models.
//
// A b2_finite_mdp_sampled row is sampled with sampled_next().  The planners that keep one env generator per episode
// (mcts.cu, olop.cu, mdp_gape.cu, mcts_dpw.cu) step SampledFiniteEnv with its step(); PlaTyPOOS (platypoos.cu) and
// sparse sampling (sparse_sampling.cu) seed a fresh generator per child or sample and check row_ok in their own loops.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "highway_lite.cuh"
#include "intersection_lite.cuh"
#include "pcg64.cuh"

namespace b2 {

// The lane mapping of a lane-group kernel of 128-thread blocks, declared as the kernel's locals: tree = thread /
// Env::GROUP and li = its lane in the group; writer: lane 0 of the group; gmask: the group's lanes in the warp (one
// lane on a finite MDP, a half warp on HighwayLite and IntersectionLite).  B2_LANE_MAP keeps the threads of a group
// past n_trees (live false): they shadow the last tree and never store.  B2_LANE_MAP_LIVE returns from them.
// Macros, not a value type or helper function: inlining one, even with the same statements in the same order, changes
// how ptxas assigns the registers of mcts_kernel<HighwayEnv>, and moving the early return after the shadowing form
// changes the code of the four kernels that return.
#define B2_LANE_GTID(Env)                                                         \
    constexpr int G = Env::GROUP;                                                 \
    const int gtid = blockIdx.x * 128 + threadIdx.x
#define B2_LANE_GMASK                                                             \
    const int lane = threadIdx.x & 31;                                            \
    const unsigned gmask = G == 1 ? (1u << lane) : (0xFFFFu << (lane & 16))
#define B2_LANE_MAP(Env, n_trees)                                                 \
    B2_LANE_GTID(Env);                                                            \
    const int tree_raw = gtid / G, li = gtid % G;                                 \
    const bool live = tree_raw < (n_trees);                                       \
    const int tree = live ? tree_raw : (n_trees) - 1;                             \
    const bool writer = live && li == 0;                                          \
    B2_LANE_GMASK
#define B2_LANE_MAP_LIVE(Env, n_trees)                                            \
    B2_LANE_GTID(Env);                                                            \
    const int tree = gtid / G, li = gtid % G;                                     \
    if (tree >= (n_trees)) return;                                                \
    const bool writer = li == 0;                                                  \
    B2_LANE_GMASK

// The finite model of one launch, as every lane env's step() reads it: the deterministic tables (FiniteEnv), or the
// sampled tables, terminal and whether a step draws from the env generator (SampledFiniteEnv).  HighwayLite and
// IntersectionLite read none of it.
struct LaneModel {
    b2_finite_mdp mdp;
    b2_finite_mdp_sampled smdp;
    const uint8_t* terminal;
    int32_t draws;
};

// searchsorted(cdf, u, side="right") on a non-decreasing row: the number of entries <= u
__device__ __forceinline__ int searchsorted_right(const double* cdf, int n, double u) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cdf[mid] <= u) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// The next state of FiniteMDPEnv.step on row s * n_actions + a: next[row, k] with k = Generator.choice(p.size, p=p)
// of the env's generator `env_rng`, i.e. searchsorted(cdf[row], random(), "right"); draw = false (a deterministic
// table) takes k = 0 and leaves env_rng alone.  The caller checks row_ok first.
__device__ __forceinline__ int sampled_next(const b2_finite_mdp_sampled& m, int64_t row, bool draw, Pcg64& env_rng) {
    const int B = m.n_next;
    const int k = draw ? searchsorted_right(m.cdf + row * B, B, env_rng.random()) : 0;
    return m.next[row * B + k];
}

// The env generator of a deterministic model: there is none to seed or load.
struct NoEnvRng {
    __device__ __forceinline__ void seed(const LaneModel& m, uint32_t seed) {}
    __device__ __forceinline__ void load_rng(const uint64_t* words) {}
};

struct FiniteEnv : NoEnvRng {
    static constexpr int GROUP = 1;
    int s;
    __device__ __forceinline__ void load_root(const int32_t* root_states, int tree, int li) { s = root_states[tree]; }
    __device__ __forceinline__ int avail(int n_actions, unsigned gmask) const { return (1 << n_actions) - 1; }
    __device__ __forceinline__ static int nth(int mask, int n) { return n; }
    // position of `action` among the available actions in the env's order, or -1
    __device__ __forceinline__ static int rank_of(int mask, int action) { return (action >= 0 && (mask >> action) & 1) ? action : -1; }
    // Steps every lane, whatever `taken` says; never fails.
    __device__ __forceinline__ bool step(const LaneModel& m, int action, int li, unsigned gmask, bool taken,
                                         bool& term, bool& trunc, double& r, int& bad_row) {
        r = m.mdp.reward[(int64_t)s * m.mdp.n_actions + action];
        term = m.mdp.terminal[s] != 0;    // finite_mdp's MDP.step: done = terminal[state BEFORE the transition]
        s = m.mdp.transition[(int64_t)s * m.mdp.n_actions + action];
        trunc = false;
        return true;
    }
};

// A finite MDP in any mode, stepped as FiniteMDPEnv.step with the episode's env generator env_rng.  kSampled<Env>
// selects what only the planners' sampled instantiations do.
struct SampledFiniteEnv : FiniteEnv {
    Pcg64 env_rng;
    // the env copy's state.seed(seed): default_rng(seed) when the steps draw
    __device__ __forceinline__ void seed(const LaneModel& m, uint32_t seed) { if (m.draws) env_rng.seed_from(seed); }
    __device__ __forceinline__ void load_rng(const uint64_t* words) { env_rng.load(words); }
    // FiniteMDPEnv.step on row s * n_actions + action, for a step the reference takes; any other step leaves s and
    // env_rng alone.  When the steps draw, a row Generator.choice rejects (its ValueError) returns false with
    // bad_row = the row and s unchanged.  Otherwise term = terminal[state BEFORE the transition], r = reward[row], and
    // sampled_next() moves s.
    __device__ __forceinline__ bool step(const LaneModel& m, int action, int li, unsigned gmask, bool taken,
                                         bool& term, bool& trunc, double& r, int& bad_row) {
        const bool draw = m.draws != 0;
        term = false;
        trunc = false;
        r = 0.0;
        if (!taken) return true;
        const int64_t row = (int64_t)s * m.smdp.n_actions + action;
        if (draw && !m.smdp.row_ok[row]) { bad_row = (int)row; return false; }
        term = m.terminal[s] != 0;
        r = m.smdp.reward[row];
        s = sampled_next(m.smdp, row, draw, env_rng);
        return true;
    }
};

template <class Env>
constexpr bool kSampled = std::is_same<Env, SampledFiniteEnv>::value;

struct HighwayEnv : NoEnvRng {
    static constexpr int GROUP = 16;
    hw::Lane L;
    int t, si;
    __device__ __forceinline__ void load_root(const int32_t* root_states, int tree, int li) {
        hw::load_state(root_states + (int64_t)tree * hw::WORDS, li, L, t, si);
    }
    __device__ __forceinline__ int avail(int n_actions, unsigned gmask) const {
        const float ego_y = __shfl_sync(gmask, L.y, 0, 16);
        return hw::avail_mask(ego_y, si);
    }
    __device__ __forceinline__ static int nth(int mask, int n) { return hw::nth_action(mask, n); }
    __device__ __forceinline__ static int rank_of(int mask, int action) {
        if (action < 0 || !((mask >> action) & 1)) return -1;
        const int order[5] = {hw::A_IDLE, hw::A_LEFT, hw::A_RIGHT, hw::A_FASTER, hw::A_SLOWER};
        int k = 0;
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            if (order[i] == action) return k;
            k += (mask >> order[i]) & 1;
        }
        return -1;
    }
    __device__ __forceinline__ bool step(const LaneModel& m, int action, int li, unsigned gmask, bool taken,
                                         bool& term, bool& trunc, double& r, int& bad_row) {
        r = (double)hw::step(L, li, t, si, action, term, trunc, gmask);
        return true;
    }
};

// IntersectionLite (mcts.cu and olop.cu only): the same 16-lane group and 136-word slot as HighwayLite; three actions
// offered in the env's order IDLE, FASTER, SLOWER, which is not ascending action id.
struct IntersectionEnv : NoEnvRng {
    static constexpr int GROUP = 16;
    il::Lane L;
    il::Globals g;
    __device__ __forceinline__ void load_root(const int32_t* root_states, int tree, int li) {
        il::load_state<false>(root_states + (int64_t)tree * il::WORDS, li, L, g);
    }
    __device__ __forceinline__ int avail(int n_actions, unsigned gmask) const { return il::avail_mask(g.si); }
    __device__ __forceinline__ static int nth(int mask, int n) { return il::nth_action(mask, n); }
    __device__ __forceinline__ static int rank_of(int mask, int action) {
        if (action < 0 || !((mask >> action) & 1)) return -1;
        const int order[3] = {il::A_IDLE, il::A_FASTER, il::A_SLOWER};
        int k = 0;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            if (order[i] == action) return k;
            k += (mask >> order[i]) & 1;
        }
        return -1;
    }
    __device__ __forceinline__ bool step(const LaneModel& m, int action, int li, unsigned gmask, bool taken,
                                         bool& term, bool& trunc, double& r, int& bad_row) {
        r = (double)il::step(L, li, g, action, term, trunc, gmask);
        return true;
    }
};

}  // namespace b2
