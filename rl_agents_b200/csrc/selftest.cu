// Test entry points of the device primitives the planners share (tests/test_gpu_device_primitives.py): numpy's PCG64
// (pcg64.cuh), the Bernoulli KL bounds (kl_bound.cuh) and the sampled finite-MDP step (lane_env.cuh).  Each kernel
// calls the same inline functions the planners call, one thread per stream or case.
#include "common.cuh"
#include "kl_bound.cuh"
#include "lane_env.cuh"
#include "pcg64.cuh"

namespace b2 {
namespace {

constexpr int PCG_NEXT64 = 0, PCG_NEXT32 = 1, PCG_RANDOM = 2, PCG_INTEGERS = 3, PCG_SKIP32 = 4, PCG_SEED_FROM = 5;

__global__ void pcg64_selftest_kernel(const uint64_t* words, const int32_t* ops, const uint64_t* args, uint64_t* out,
                                      uint64_t* words_out, int n_streams, int n_ops) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_streams) return;
    Pcg64 g;
    g.load(words + (int64_t)s * 6);
    for (int i = 0; i < n_ops; ++i) {
        const int64_t at = (int64_t)s * n_ops + i;
        const uint64_t a = args[at];
        uint64_t r = 0;
        switch (ops[at]) {
            case PCG_NEXT64: r = g.next64(); break;
            case PCG_NEXT32: r = g.next32(); break;
            case PCG_RANDOM: r = (uint64_t)__double_as_longlong(g.random()); break;
            case PCG_INTEGERS: r = g.integers((uint32_t)a); break;
            case PCG_SKIP32: g.skip32(a); r = (uint64_t)g.state; break;
            case PCG_SEED_FROM: g.seed_from((uint32_t)a); r = (uint64_t)g.state; break;
            default: continue;
        }
        out[at] = r;
    }
    g.store(words_out + (int64_t)s * 6);
}

__global__ void kl_selftest_kernel(const double* p, const double* q, int n_kl, double* kl, const double* sum,
                                   const int32_t* count, const double* threshold, const int32_t* lower, int n_bound,
                                   double* bound) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_kl) kl[i] = bernoulli_kl(p[i], q[i]);
    if (i < n_bound) bound[i] = kl_bound(sum[i], count[i], threshold[i], lower[i] != 0);
}

__global__ void sampled_next_selftest_kernel(const double* cdf, int B, const double* u, const int32_t* u_row, int n_u,
                                             int32_t* k, b2_finite_mdp_sampled m, const int64_t* rows,
                                             const int32_t* draw, const uint64_t* words, int n_steps, int32_t* next,
                                             uint64_t* words_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_u) k[i] = searchsorted_right(cdf + (int64_t)u_row[i] * B, B, u[i]);
    if (i < n_steps) {
        Pcg64 g;
        g.load(words + (int64_t)i * 6);
        next[i] = sampled_next(m, rows[i], draw[i] != 0, g);
        g.store(words_out + (int64_t)i * 6);
    }
}

inline int blocks(int n) { return (n + 127) / 128; }

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" int b2_selftest_pcg64(const uint64_t* words, const int32_t* ops, const uint64_t* args, uint64_t* out,
                                 uint64_t* words_out, int32_t n_streams, int32_t n_ops, void* stream) {
    B2_REQUIRE(words && words_out && n_streams > 0 && n_ops >= 0 && (n_ops == 0 || (ops && args && out)),
               "null pointer / empty batch");
    pcg64_selftest_kernel<<<blocks(n_streams), 128, 0, (cudaStream_t)stream>>>(words, ops, args, out, words_out,
                                                                               n_streams, n_ops);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_selftest_kl(const double* p, const double* q, int32_t n_kl, double* kl, const double* sum,
                              const int32_t* count, const double* threshold, const int32_t* lower, int32_t n_bound,
                              double* bound, void* stream) {
    B2_REQUIRE(n_kl >= 0 && n_bound >= 0 && n_kl + n_bound > 0, "empty batch");
    B2_REQUIRE(n_kl == 0 || (p && q && kl), "null pointer");
    B2_REQUIRE(n_bound == 0 || (sum && count && threshold && lower && bound), "null pointer");
    const int n = n_kl > n_bound ? n_kl : n_bound;
    kl_selftest_kernel<<<blocks(n), 128, 0, (cudaStream_t)stream>>>(p, q, n_kl, kl, sum, count, threshold, lower,
                                                                    n_bound, bound);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_selftest_sampled_next(const double* cdf, int32_t n_next, const double* u, const int32_t* u_row,
                                        int32_t n_u, int32_t* k, const b2_finite_mdp_sampled* mdp, const int64_t* rows,
                                        const int32_t* draw, const uint64_t* words, int32_t n_steps, int32_t* next,
                                        uint64_t* words_out, void* stream) {
    B2_REQUIRE(n_u >= 0 && n_steps >= 0 && n_u + n_steps > 0, "empty batch");
    B2_REQUIRE(n_u == 0 || (cdf && u && u_row && k && n_next >= 1), "null pointer / bad n_next");
    B2_REQUIRE(n_steps == 0 || (mdp && rows && draw && words && next && words_out), "null pointer");
    b2_finite_mdp_sampled m{};
    if (n_steps > 0) {
        if (check_sampled_mdp(*mdp, mdp->n_actions, nullptr, false) != B2_OK) return B2_ERR_INVALID;
        m = *mdp;
    }
    const int n = n_u > n_steps ? n_u : n_steps;
    sampled_next_selftest_kernel<<<blocks(n), 128, 0, (cudaStream_t)stream>>>(cdf, n_next, u, u_row, n_u, k, m, rows,
                                                                              draw, words, n_steps, next, words_out);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
