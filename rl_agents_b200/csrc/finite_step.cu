// Batched FiniteMDPEnv.step (b2_finite_step): one thread per episode, each stepping its episode's state with
// lane_env.cuh's SampledFiniteEnv::step -- the transition, row check and env-generator draw the sampling planners run
// inside their searches.  The closed-loop evaluation (evaluation.py, env "finite") advances every live episode with one
// launch per decision step.
#include "common.cuh"
#include "lane_env.cuh"

namespace b2 {
namespace {

constexpr int kThreads = 128;
constexpr int kMaxDevices = 64;

// The first live episode whose state or action is outside the MDP, as 2 * episode + (1: the action), or left at
// INT32_MAX.  Nothing is stepped before every live episode has passed.
__global__ void finite_step_check_kernel(int32_t n_states, int32_t n_actions, const int32_t* states,
                                         const int32_t* actions, const uint8_t* alive, int32_t n, int32_t* first_bad) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n || !alive[i]) return;
    const int s = states[i], a = actions[i];
    if (s < 0 || s >= n_states) atomicMin(first_bad, 2 * i);
    else if (a < 0 || a >= n_actions) atomicMin(first_bad, 2 * i + 1);
}

__global__ void finite_step_kernel(LaneModel m, int32_t* states, const int32_t* actions, const uint8_t* alive,
                                   uint64_t* env_rng, double* reward, int32_t* flags, int32_t* bad_row, int32_t n) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n || !alive[i]) return;
    SampledFiniteEnv env;
    env.s = states[i];
    if (m.draws) env.load_rng(env_rng + (int64_t)i * B2_PCG64_STATE_WORDS);
    bool term, trunc;
    double r;
    int bad = -1;
    if (env.step(m, actions[i], 0, 1u, true, term, trunc, r, bad)) {
        states[i] = env.s;
        if (m.draws) env.env_rng.store(env_rng + (int64_t)i * B2_PCG64_STATE_WORDS);
    }
    reward[i] = r;
    flags[i] = term ? 1 : 0;
    bad_row[i] = bad;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" int b2_finite_step(const b2_finite_mdp_sampled* mdp, const uint8_t* terminal, int32_t env_draws,
                              int32_t* states, const int32_t* actions, const uint8_t* alive, uint64_t* env_rng,
                              double* reward, int32_t* flags, int32_t* bad_row, int32_t n, void* stream) {
    B2_REQUIRE(mdp && states && actions && alive && reward && flags && bad_row, "null pointer");
    B2_REQUIRE(n >= 1, "n must be >= 1");
    if (check_sampled_mdp(*mdp, mdp->n_actions, terminal, true) != B2_OK) return B2_ERR_INVALID;
    B2_REQUIRE(env_draws == 0 || env_draws == 1, "env_draws must be 0 or 1");
    B2_REQUIRE(env_rng || !env_draws, "null pointer: env_rng is needed when the steps draw");
    const cudaStream_t s = (cudaStream_t)stream;
    const int blocks = (n + kThreads - 1) / kThreads;
    // The check's result word: one per host thread and device, allocated on first use and kept.  A call reads it back
    // before it returns, so the calls of one thread never share it in flight, whatever their streams.
    static thread_local int32_t* first_bad[kMaxDevices] = {};
    int dev = 0;
    B2_CUDA_CHECK(cudaGetDevice(&dev));
    B2_REQUIRE(dev < kMaxDevices, "device ordinal too large");
    if (!first_bad[dev]) B2_CUDA_CHECK(cudaMalloc((void**)&first_bad[dev], sizeof(int32_t)));
    int32_t bad = INT32_MAX;
    B2_CUDA_CHECK(cudaMemcpyAsync(first_bad[dev], &bad, sizeof(int32_t), cudaMemcpyHostToDevice, s));
    finite_step_check_kernel<<<blocks, kThreads, 0, s>>>(mdp->n_states, mdp->n_actions, states, actions, alive, n,
                                                         first_bad[dev]);
    B2_CUDA_CHECK(cudaGetLastError());
    B2_CUDA_CHECK(cudaMemcpyAsync(&bad, first_bad[dev], sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    B2_CUDA_CHECK(cudaStreamSynchronize(s));
    if (bad != INT32_MAX) {
        set_error("invalid argument: episode %d: %s outside [0, %d)", bad / 2, bad & 1 ? "action" : "state",
                  bad & 1 ? mdp->n_actions : mdp->n_states);
        return B2_ERR_INVALID;
    }
    LaneModel m{};
    m.smdp = *mdp;
    m.terminal = terminal;
    m.draws = env_draws;
    finite_step_kernel<<<blocks, kThreads, 0, s>>>(m, states, actions, alive, env_rng, reward, flags, bad_row, n);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
