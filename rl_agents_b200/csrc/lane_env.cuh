// Device env models of the one-tree-per-lane-group planners (mcts.cu, olop.cu, mdp_gape.cu, brue.cu): one tree per
// lane on a finite MDP, one tree per 16-lane group on HighwayLite (lane = vehicle slot, the scene in registers, so
// the reference's deep copy of the env is a register copy).  Each model reads only what it needs: the finite tables,
// the root states and the action count.
//
// step() reports truncation separately; MCTS reads it, the other planners pass a dummy (the reference's 4-tuple step
// drops truncation).
#pragma once
#include "common.cuh"
#include "highway_lite.cuh"

namespace b2 {

struct FiniteEnv {
    static constexpr int GROUP = 1;
    int s;
    __device__ __forceinline__ void load_root(const int32_t* root_states, int tree, int li) { s = root_states[tree]; }
    __device__ __forceinline__ int avail(int n_actions, unsigned gmask) const { return (1 << n_actions) - 1; }
    __device__ __forceinline__ static int nth(int mask, int n) { return n; }
    // position of `action` among the available actions in the env's order, or -1
    __device__ __forceinline__ static int rank_of(int mask, int action) { return (action >= 0 && (mask >> action) & 1) ? action : -1; }
    __device__ __forceinline__ double step(const b2_finite_mdp& m, int action, int li, unsigned gmask, float* gs,
                                           bool& term, bool& trunc) {
        const double r = m.reward[(int64_t)s * m.n_actions + action];
        term = m.terminal[s] != 0;        // finite_mdp's MDP.step: done = terminal[state BEFORE the transition]
        s = m.transition[(int64_t)s * m.n_actions + action];
        trunc = false;
        return r;
    }
};

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
    __device__ __forceinline__ double step(const b2_finite_mdp& m, int action, int li, unsigned gmask, float* gs,
                                           bool& term, bool& trunc) {
        return (double)hw::step(L, li, t, si, action, term, trunc, gmask, gs);
    }
};

}  // namespace b2
