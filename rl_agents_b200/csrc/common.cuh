// Shared host/device helpers of libb2planner (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/b2_planner.h"

namespace b2 {

void set_error(const char* fmt, ...);

#define B2_CUDA_CHECK(expr)                                                              \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            b2::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return B2_ERR_CUDA;                                                          \
        }                                                                                \
    } while (0)

#define B2_REQUIRE(cond, msg)                            \
    do {                                                 \
        if (!(cond)) {                                   \
            b2::set_error("invalid argument: %s", msg);  \
            return B2_ERR_INVALID;                       \
        }                                                \
    } while (0)

int sm_count();

// Launch checks of the planners that run one tree per lane group.  Both return B2_OK, or B2_ERR_INVALID with the
// error set.  check_env_kind: a known env_kind, and HighwayLite's 5 actions; check_lane_env also requires the
// finite tables and their action count.  check_lane_env_il (MCTS and OLOP, the planners with an IntersectionLite
// model) also accepts IntersectionLite with its 3 actions; the other planners keep refusing it.
int check_env_kind(int env_kind, int n_actions);
int check_lane_env(int env_kind, int n_actions, const b2_finite_mdp& mdp);
int check_lane_env_il(int env_kind, int n_actions, const b2_finite_mdp& mdp);
// Launch check of a finite MDP stepped as FiniteMDPEnv.step (OLOP, MDP-GapE, MCTS-DPW, PlaTyPOOS, sparse sampling):
// B2_OK, or B2_ERR_INVALID with the error set.  Its tables, and terminal when the planner reads it (needs_terminal),
// then its shape against the planner's n_actions.
int check_sampled_mdp(const b2_finite_mdp_sampled& mdp, int n_actions, const uint8_t* terminal, bool needs_terminal);
// The launch check the *_sampled entry points (MCTS per tree and wavefront, OLOP, MDP-GapE) share after their own
// config checks: B2_OK, or B2_ERR_INVALID with the error set.  A finite env_kind, check_sampled_mdp with terminal,
// and env_draws 0 or 1.
int check_sampled_entry(int env_kind, const b2_finite_mdp_sampled& mdp, int n_actions, const uint8_t* terminal,
                        int32_t env_draws);

// Blocks of 128 threads for n_trees trees of Env::GROUP lanes each.
template <class Env>
inline int lane_grid(int n_trees) { return (n_trees * Env::GROUP + 127) / 128; }

// Grid-wide barrier of a cooperative launch (all CTAs co-resident), keyed on two control words of `ctl` that the launch
// wrapper zeroes: the arrival count `bar_count` and the generation `bar_gen`.  Data written before it by any CTA is
// visible to every CTA after it.
template <class Control>
__device__ __forceinline__ void grid_barrier(Control* ctl, unsigned n_ctas) {
    __syncthreads();
    if (threadIdx.x == 0) {
        volatile unsigned* gen_p = &ctl->bar_gen;
        const unsigned gen = *gen_p;
        __threadfence();
        if (atomicAdd(&ctl->bar_count, 1u) == n_ctas - 1) {
            ctl->bar_count = 0;
            __threadfence();
            atomicAdd(&ctl->bar_gen, 1u);
        } else {
            while (*gen_p == gen) {}
        }
        __threadfence();
    }
    __syncthreads();
}

__device__ __forceinline__ double warp_max_f64(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        double w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w > v ? w : v;
    }
    return v;
}

// One step of numpy's max / min reduction (ndarray.max, np.min): a NaN operand wins, so a NaN anywhere in the reduced
// axis makes the result NaN, whatever its position.  On other operands these are `x > m ? x : m` / `x < m ? x : m`.
__device__ __forceinline__ double np_max(double m, double x) { return (x > m || isnan(x)) ? x : m; }
__device__ __forceinline__ double np_min(double m, double x) { return (x < m || isnan(x)) ? x : m; }

// numpy.isclose(a, b, rtol, atol) as numpy >= 2 states it: (|a - b| <= atol + rtol * |b| and b finite) or a == b.  Equal
// infinities are close, NaN is close to nothing, and so are equal finite values even when atol + rtol * |b| < 0 (the
// value-iteration sweeps' "early exit off" setting rtol = 0, atol = -1 still stops at an exact fixed point).
__device__ __forceinline__ bool np_isclose(double a, double b, double rtol, double atol) {
    return (fabs(a - b) <= atol + rtol * fabs(b) && isfinite(b)) || a == b;
}

}  // namespace b2
