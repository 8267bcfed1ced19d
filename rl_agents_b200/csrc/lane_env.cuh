// Device env models of the one-tree-per-lane-group planners (mcts.cu, olop.cu, mdp_gape.cu, brue.cu, mcts_dpw.cu): one
// tree per lane on a finite MDP, one tree per 16-lane group on HighwayLite and IntersectionLite (lane = vehicle slot, the
// scene in registers, so the reference's deep copy of the env is a register copy).  Each model reads only what it
// needs: the finite tables, the root states and the action count.
//
// step() reports truncation separately; MCTS reads it, the other planners pass a dummy (the reference's 4-tuple step
// drops truncation).
//
// A b2_finite_mdp_sampled row is sampled with sampled_next().  The planners that keep one env generator per episode
// (olop.cu, mdp_gape.cu, mcts_dpw.cu) step SampledFiniteEnv with its step(); PlaTyPOOS (platypoos.cu) and sparse
// sampling (sparse_sampling.cu) seed a fresh generator per child or sample and check row_ok in their own loops.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "highway_lite.cuh"
#include "intersection_lite.cuh"
#include "pcg64.cuh"

namespace b2 {

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

struct FiniteEnv {
    static constexpr int GROUP = 1;
    int s;
    __device__ __forceinline__ void load_root(const int32_t* root_states, int tree, int li) { s = root_states[tree]; }
    __device__ __forceinline__ int avail(int n_actions, unsigned gmask) const { return (1 << n_actions) - 1; }
    __device__ __forceinline__ static int nth(int mask, int n) { return n; }
    // position of `action` among the available actions in the env's order, or -1
    __device__ __forceinline__ static int rank_of(int mask, int action) { return (action >= 0 && (mask >> action) & 1) ? action : -1; }
    __device__ __forceinline__ double step(const b2_finite_mdp& m, int action, int li, unsigned gmask,
                                           bool& term, bool& trunc) {
        const double r = m.reward[(int64_t)s * m.n_actions + action];
        term = m.terminal[s] != 0;        // finite_mdp's MDP.step: done = terminal[state BEFORE the transition]
        s = m.transition[(int64_t)s * m.n_actions + action];
        trunc = false;
        return r;
    }
};

// A finite MDP in any mode, stepped as FiniteMDPEnv.step with the episode's env generator (env_rng; seeded by the
// planner only when draw is set).  kSampled<Env> selects the code that calls this step().
struct SampledFiniteEnv : FiniteEnv {
    Pcg64 env_rng;
    // FiniteMDPEnv.step on row s * n_actions + action.  With draw set, a row Generator.choice rejects (its ValueError)
    // returns false with bad_row = the row and s unchanged.  Otherwise term = terminal[state BEFORE the transition],
    // r = reward[row], and sampled_next() moves s.
    __device__ __forceinline__ bool step(const b2_finite_mdp_sampled& m, const uint8_t* terminal, bool draw, int action,
                                         bool& term, double& r, int& bad_row) {
        const int64_t row = (int64_t)s * m.n_actions + action;
        if (draw && !m.row_ok[row]) { bad_row = (int)row; return false; }
        term = terminal[s] != 0;
        r = m.reward[row];
        s = sampled_next(m, row, draw, env_rng);
        return true;
    }
};

template <class Env>
constexpr bool kSampled = std::is_same<Env, SampledFiniteEnv>::value;

struct HighwayEnv {
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
    __device__ __forceinline__ double step(const b2_finite_mdp& m, int action, int li, unsigned gmask,
                                           bool& term, bool& trunc) {
        return (double)hw::step(L, li, t, si, action, term, trunc, gmask);
    }
};

// IntersectionLite (mcts.cu and olop.cu only): the same 16-lane group and 136-word slot as HighwayLite; three actions
// offered in the env's order IDLE, FASTER, SLOWER, which is not ascending action id.
struct IntersectionEnv {
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
    __device__ __forceinline__ double step(const b2_finite_mdp& m, int action, int li, unsigned gmask,
                                           bool& term, bool& trunc) {
        return (double)il::step(L, li, g, action, term, trunc, gmask);
    }
};

}  // namespace b2
