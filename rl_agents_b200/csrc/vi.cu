// Value-iteration Bellman sweep (value_iteration.py:51-73 of the reference).
//
// One launch = one application of  Q' = R + gamma * E[V(s')]  over a slab of
// states, fused with V' = max_a Q' (best_action_value, :47-49) and with the
// element-wise np.allclose(Q, Q') test of fixed_point_iteration (:70).
//
// HBM-bound (SURVEY 8d): per (s,a,b) the kernel streams 8 B of P and 4 B of N
// once, gathers 8 B of V (L2 resident: 8 MB at S=1e6), and per (s,a) streams
// R, Q_old in and Q' out.  Summation order over the successor axis is numpy's
// pairwise_sum so that results are bit-identical with the reference's
// `(P * take(V, N)).sum(axis=-1)`.
#include "common.cuh"

namespace b2 {

// numpy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src):
// < 8 sequential; <= 128 eight strided accumulators; else split in halves (n2 = n/2 rounded down to a multiple
// of 8) and add the two halves' sums.  The recursion is unrolled on an explicit stack (device recursion would
// need a per-thread stack the compiler cannot bound): leaf(lo, n) sums one block of n <= 128 elements.
template <typename Leaf>
__device__ __forceinline__ double np_pairwise_tree(Leaf leaf, int lo0, int n0) {
    int lo_s[26], n_s[26];
    double left_s[26];
    unsigned char st_s[26];
    int sp = 0;
    lo_s[0] = lo0; n_s[0] = n0; st_s[0] = 0;
    double ret = 0.0;
    while (sp >= 0) {
        const int lo = lo_s[sp], n = n_s[sp];
        if (n <= 128) { ret = leaf(lo, n); --sp; continue; }
        int n2 = n / 2;
        n2 -= n2 % 8;
        if (st_s[sp] == 0) { st_s[sp] = 1; ++sp; lo_s[sp] = lo; n_s[sp] = n2; st_s[sp] = 0; }
        else if (st_s[sp] == 1) { left_s[sp] = ret; st_s[sp] = 2; ++sp; lo_s[sp] = lo + n2; n_s[sp] = n - n2; st_s[sp] = 0; }
        else { ret = left_s[sp] + ret; --sp; }
    }
    return ret;
}

template <typename Load>
__device__ __forceinline__ double np_pairwise_leaf(Load a, int lo, int n) {   // 8 <= n <= 128
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a(lo + j);
    int i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] += a(lo + i + j);
    }
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a(lo + i);
    return res;
}

template <typename Load>
__device__ __noinline__ double np_pairwise_sum_big(Load a, int lo, int n) {
    return np_pairwise_tree([&](int l, int m) { return np_pairwise_leaf(a, l, m); }, lo, n);
}

template <typename Load>
__device__ __forceinline__ double np_pairwise_sum(Load a, int lo, int n) {
    if (n < 8) {   // the common sparse case (B = 2..4): stays inline, no call
        double res = 0.;
        for (int i = 0; i < n; ++i) res += a(lo + i);
        return res;
    }
    return np_pairwise_sum_big(a, lo, n);
}

struct SweepArgs {
    const double* P;       // sparse/stochastic probabilities (slab-local)
    const int32_t* N;      // sparse successors or deterministic transition
    const double* R;
    const uint8_t* term;
    const double* v_in;
    const double* q_old;
    double* q_new;
    double* v_out;
    int32_t* viol;
    int32_t sweep;
    int64_t rows;          // states in the slab
    int64_t row_begin;
    int A, B;
    int tile_states;
    double gamma, rtol, atol;
};

// Sparse (B successors) and deterministic (B = 1, P == nullptr) modes.
// CTA = tile of `tile_states` states; dynamic smem: prod[tile*A*B] + q[tile*A].
__global__ void __launch_bounds__(256, 4) vi_sweep_gather_kernel(SweepArgs g) {
    if (g.sweep > 0 && g.viol[g.sweep - 1] == 0) return;   // already converged
    extern __shared__ double smem[];
    const int E = g.A * g.B;
    double* prod = smem;
    double* qs = smem + (size_t)g.tile_states * E;
    const int tid = threadIdx.x;
    const int64_t n_tiles = (g.rows + g.tile_states - 1) / g.tile_states;
    int bad = 0;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t s0 = tile * g.tile_states;
        const int ns = (int)min((int64_t)g.tile_states, g.rows - s0);
        const int ne = ns * E;
        const int64_t base = s0 * E;
        // phase 1: stream P/N coalesced, gather V, stage products
        if (g.P) {
            constexpr int U = 4;
            for (int i0 = tid; i0 < ne; i0 += 256 * U) {
                double p[U];
                int32_t n[U];
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    int i = i0 + u * 256;
                    if (i < ne) {
                        p[u] = __ldcs(g.P + base + i);
                        n[u] = __ldcs(g.N + base + i);
                    }
                }
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    int i = i0 + u * 256;
                    if (i < ne) prod[i] = p[u] * __ldg(g.v_in + n[u]);
                }
            }
        } else {
            for (int i = tid; i < ne; i += 256) prod[i] = __ldg(g.v_in + __ldcs(g.N + base + i));
        }
        __syncthreads();
        // phase 2: one thread per (s,a): successor sum in numpy order, Bellman, allclose
        const int nsa = ns * g.A;
        for (int r = tid; r < nsa; r += 256) {
            double nv = np_pairwise_sum([&](int i) { return prod[i]; }, r * g.B, g.B);
            const int s = r / g.A;
            if (g.term[s0 + s]) nv = 0.0;
            const int64_t qi = s0 * g.A + r;
            const double q = __ldcs(g.R + qi) + g.gamma * nv;
            const double qo = __ldcs(g.q_old + qi);
            if (!np_isclose(qo, q, g.rtol, g.atol)) bad++;
            __stcs(g.q_new + qi, q);
            qs[r] = q;
        }
        __syncthreads();
        // phase 3: V' = max_a Q'
        for (int s = tid; s < ns; s += 256) {
            double m = qs[s * g.A];
            for (int a = 1; a < g.A; ++a) m = np_max(m, qs[s * g.A + a]);
            g.v_out[g.row_begin + s0 + s] = m;
        }
        __syncthreads();
    }
    bad = __reduce_add_sync(0xffffffffu, bad);
    if ((tid & 31) == 0 && bad) atomicAdd(g.viol + g.sweep, bad);
}

// ---------------------------------------------------------------------------
// Register variant for the common small shapes (B in {1,2,4,8}, A a power of two
// <= 32): one thread per (s,a) row keeps its B probabilities, successors and
// gathered values in registers (16-byte vector loads, all B gathers in flight),
// sums them in numpy's order, and the max over the A actions of a state is a
// segmented warp-shuffle reduction -- no shared memory, no block barrier.
// ---------------------------------------------------------------------------
template <int B, bool HAS_P>
__global__ void __launch_bounds__(256) vi_sweep_row_kernel(SweepArgs g) {
    if (g.sweep > 0 && g.viol[g.sweep - 1] == 0) return;
    const int64_t n_sa = g.rows * g.A;
    const int A = g.A;
    int bad = 0;
    for (int64_t qi = (int64_t)blockIdx.x * 256 + threadIdx.x; qi - threadIdx.x % 32 < n_sa;
         qi += (int64_t)gridDim.x * 256) {
        const bool live = qi < n_sa;
        double q = -INFINITY;
        if (live) {
            int32_t n[B];
            double p[B], v[B];
            const int32_t* np = g.N + qi * B;
            if constexpr (B % 4 == 0) {
#pragma unroll
                for (int b = 0; b < B; b += 4) {
                    const int4 t = __ldcs(reinterpret_cast<const int4*>(np + b));
                    n[b] = t.x; n[b + 1] = t.y; n[b + 2] = t.z; n[b + 3] = t.w;
                }
            } else if constexpr (B == 2) {
                const int2 t = __ldcs(reinterpret_cast<const int2*>(np));
                n[0] = t.x; n[1] = t.y;
            } else {
#pragma unroll
                for (int b = 0; b < B; ++b) n[b] = __ldcs(np + b);
            }
#pragma unroll
            for (int b = 0; b < B; ++b) v[b] = __ldcg(g.v_in + n[b]);   // L2 only: V never hits in L1 anyway
            if constexpr (HAS_P) {
                const double* pp = g.P + qi * B;
                if constexpr (B % 2 == 0) {
#pragma unroll
                    for (int b = 0; b < B; b += 2) {
                        const double2 t = __ldcs(reinterpret_cast<const double2*>(pp + b));
                        p[b] = t.x; p[b + 1] = t.y;
                    }
                } else {
#pragma unroll
                    for (int b = 0; b < B; ++b) p[b] = __ldcs(pp + b);
                }
#pragma unroll
                for (int b = 0; b < B; ++b) v[b] = p[b] * v[b];
            }
            double nv;
            if constexpr (B < 8) {          // numpy pairwise_sum, n < 8: sequential from 0.
                nv = 0.;
#pragma unroll
                for (int b = 0; b < B; ++b) nv += v[b];
            } else {                         // n == 8: eight accumulators, fixed combination tree
                nv = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
            }
            const int64_t srow = qi / A;
            if (g.term[srow]) nv = 0.0;
            q = __ldcs(g.R + qi) + g.gamma * nv;
            if (!np_isclose(__ldcs(g.q_old + qi), q, g.rtol, g.atol)) bad++;
            __stcs(g.q_new + qi, q);
        }
        // V' = max_a Q': the A actions of a state sit in A consecutive lanes
        double m = q;
        for (int o = 1; o < A; o <<= 1) m = np_max(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (live && (qi % A) == 0) g.v_out[g.row_begin + qi / A] = m;
    }
    bad = __reduce_add_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && bad) atomicAdd(g.viol + g.sweep, bad);
}

// Dense stochastic mode, cooperative: an 8-lane group per (s,a) row.  numpy's pairwise sum keeps eight strided
// accumulators r[j] += a[i + j] over a block of <= 128 elements and combines them as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)): lane j of the group IS accumulator j, so the row of P is read in
// coalesced 64-byte pieces (one thread per row would read with a stride of S doubles), and the fixed
// combination tree is an xor-butterfly (fp addition commutes, so every lane ends with the same bits).
// Blocks longer than 128 split in halves exactly as numpy does (n2 = n/2 rounded down to a multiple of 8).
template <typename Load>
__device__ __noinline__ double np_pairwise_sum_group(Load a, int lo, int n, int lane8, unsigned gmask) {
    if (n < 8) {
        double res = 0.;
        for (int i = 0; i < n; ++i) res += a(lo + i);
        return res;
    }
    return np_pairwise_tree([&](int l, int m) {
        double r = a(l + lane8);
        const int body = m - (m % 8);
        for (int i = 8; i < body; i += 8) r += a(l + i + lane8);
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) r = r + __shfl_xor_sync(gmask, r, o);
        for (int i = body; i < m; ++i) r += a(l + i);
        return r;
    }, lo, n);
}

__global__ void __launch_bounds__(256) vi_sweep_dense_group_kernel(SweepArgs g) {
    if (g.sweep > 0 && g.viol[g.sweep - 1] == 0) return;
    const int tid = threadIdx.x, lane8 = tid & 7;
    const unsigned gmask = 0xffu << (tid & 24);
    const int64_t n_rows = g.rows * g.A;
    const int64_t row_raw = (int64_t)blockIdx.x * 32 + (tid >> 3);
    const bool live = row_raw < n_rows;
    const int64_t row = live ? row_raw : n_rows - 1;       // idle groups shadow the last row, never store
    const double* p = g.P + row * (int64_t)g.B;
    double nv = np_pairwise_sum_group([&](int i) { return p[i] * g.v_in[i]; }, 0, g.B, lane8, gmask);
    int bad = 0;
    if (live && lane8 == 0) {
        if (g.term[row / g.A]) nv = 0.0;
        const double q = g.R[row] + g.gamma * nv;
        if (!np_isclose(g.q_old[row], q, g.rtol, g.atol)) bad = 1;
        g.q_new[row] = q;
    }
    bad = __reduce_add_sync(0xffffffffu, bad);
    if ((tid & 31) == 0 && bad) atomicAdd(g.viol + g.sweep, bad);
}

// V' = max_a Q' for the dense mode (rows may straddle CTAs there)
__global__ void vi_rowmax_kernel(SweepArgs g) {
    if (g.sweep > 0 && g.viol[g.sweep - 1] == 0) return;
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= g.rows) return;
    const double* q = g.q_new + s * g.A;
    double m = q[0];
    for (int a = 1; a < g.A; ++a) m = np_max(m, q[a]);
    g.v_out[g.row_begin + s] = m;
}

// ---------------------------------------------------------------------------
// Robust value iteration (robust_value_iteration.py:39-58): Q' = min over the M
// models of R_m + gamma * E_m[V(s')]; no terminal handling.  One thread per (s,a)
// loops over the models (deterministic: one gather each; stochastic: a dense
// row in numpy's summation order); V' = max_a Q' by vi_rowmax_kernel.
// ---------------------------------------------------------------------------
struct RobustArgs {
    const void* transition;   // int32 [M, S, A]  |  double [M, S, A, S]
    const double* reward;     // [M, S, A]
    int n_models, dense;
};

__global__ void __launch_bounds__(128) vi_robust_kernel(SweepArgs g, RobustArgs ra) {
    if (g.sweep > 0 && g.viol[g.sweep - 1] == 0) return;
    const int64_t n_rows = g.rows * g.A;
    const int64_t row = (int64_t)blockIdx.x * 128 + threadIdx.x;
    int bad = 0;
    if (row < n_rows) {
        double q = INFINITY;
        for (int m = 0; m < ra.n_models; ++m) {
            double nv;
            if (ra.dense) {
                const double* p = (const double*)ra.transition + ((int64_t)m * n_rows + row) * g.rows;
                nv = np_pairwise_sum([&](int i) { return p[i] * g.v_in[i]; }, 0, (int)g.rows);
            } else {
                nv = g.v_in[((const int32_t*)ra.transition)[(int64_t)m * n_rows + row]];
            }
            const double qm = ra.reward[(int64_t)m * n_rows + row] + g.gamma * nv;
            q = np_min(q, qm);                         // np.min over the model axis
        }
        if (!np_isclose(g.q_old[row], q, g.rtol, g.atol)) bad = 1;
        g.q_new[row] = q;
    }
    bad = __reduce_add_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31) == 0 && bad) atomicAdd(g.viol + g.sweep, bad);
}

}  // namespace b2

using namespace b2;

extern "C" int b2_vi_sweep(const b2_vi_problem* p, const double* v_in, const double* q_old, double* q_new,
                           double* v_out, int32_t* viol, int32_t sweep_index, void* stream_) {
    B2_REQUIRE(p && v_in && q_old && q_new && v_out && viol, "null pointer");
    B2_REQUIRE(p->reward && p->transition && p->terminal, "MDP tables (reward / transition / terminal) missing");
    B2_REQUIRE(p->n_actions > 0 && p->row_end >= p->row_begin && p->row_end <= p->n_states, "bad shape");
    B2_REQUIRE(sweep_index >= 0, "sweep_index < 0");
    B2_REQUIRE(p->reserved == 0, "b2_vi_problem.reserved must be 0");
    cudaStream_t stream = (cudaStream_t)stream_;
    SweepArgs g;
    g.R = p->reward; g.term = p->terminal; g.v_in = v_in; g.q_old = q_old; g.q_new = q_new; g.v_out = v_out;
    g.viol = viol; g.sweep = sweep_index; g.rows = p->row_end - p->row_begin; g.row_begin = p->row_begin;
    g.A = p->n_actions; g.gamma = p->gamma; g.rtol = p->rtol; g.atol = p->atol;
    if (g.rows == 0) return B2_OK;
    if (p->mode == B2_VI_STOCHASTIC) {
        B2_REQUIRE(p->n_next == p->n_states, "stochastic mode: n_next must equal n_states");
        g.P = (const double*)p->transition; g.N = nullptr; g.B = (int)p->n_states; g.tile_states = 0;
        const int64_t n_rows = g.rows * g.A;
        vi_sweep_dense_group_kernel<<<(unsigned)((n_rows + 31) / 32), 256, 0, stream>>>(g);
        vi_rowmax_kernel<<<(unsigned)((g.rows + 255) / 256), 256, 0, stream>>>(g);
        B2_CUDA_CHECK(cudaGetLastError());
        return B2_OK;
    }
    if (p->mode == B2_VI_SPARSE) {
        B2_REQUIRE(p->n_next > 0 && p->next, "sparse mode needs next[] and n_next");
        g.P = (const double*)p->transition; g.N = p->next; g.B = p->n_next;
    } else if (p->mode == B2_VI_DETERMINISTIC) {
        g.P = nullptr; g.N = (const int32_t*)p->transition; g.B = 1;
    } else {
        set_error("unknown VI mode %d", p->mode);
        return B2_ERR_INVALID;
    }
    const int E = g.A * g.B;
    B2_REQUIRE(E <= 8192, "n_actions * n_next > 8192 not supported by the tiled kernel");
    // register kernel: B in {1,2,4,8}, A a power of two <= 32, vector-load alignment
    if ((g.A & (g.A - 1)) == 0 && g.A <= 32 && (g.B == 1 || g.B == 2 || g.B == 4 || g.B == 8) &&
        (uintptr_t)g.N % 16 == 0 && (!g.P || (uintptr_t)g.P % 16 == 0)) {
        const int64_t n_sa = g.rows * g.A;
        const int64_t blocks = (n_sa + 255) / 256;
        const int64_t cap = (int64_t)sm_count() * 64;
        const unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
#define B2_ROW(BB)                                                                            \
    if (g.P) vi_sweep_row_kernel<BB, true><<<grid, 256, 0, stream>>>(g);                      \
    else vi_sweep_row_kernel<BB, false><<<grid, 256, 0, stream>>>(g)
        if (g.B == 1) { B2_ROW(1); } else if (g.B == 2) { B2_ROW(2); } else if (g.B == 4) { B2_ROW(4); } else { B2_ROW(8); }
#undef B2_ROW
        B2_CUDA_CHECK(cudaGetLastError());
        return B2_OK;
    }
    int tile = 4096 / E;
    if (tile < 1) tile = 1;
    if (tile * g.A > 2048) tile = 2048 / g.A;
    if (tile < 1) tile = 1;
    g.tile_states = tile;
    const size_t smem = ((size_t)tile * E + (size_t)tile * g.A) * sizeof(double);
    // at most (8192 + 8192) doubles = 128 KB: tile * E <= max(4096, E) and tile * A <= max(2048, A), E <= 8192
    // (one state of A = 8192, B = 1).  Per device and cheap: set on every call (a process may drive several devices)
    B2_CUDA_CHECK(cudaFuncSetAttribute(vi_sweep_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       2 * 8192 * (int)sizeof(double)));
    const int64_t n_tiles = (g.rows + tile - 1) / tile;
    const int64_t max_grid = (int64_t)sm_count() * 8;
    const unsigned grid = (unsigned)(n_tiles < max_grid ? n_tiles : max_grid);
    vi_sweep_gather_kernel<<<grid, 256, smem, stream>>>(g);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_vi_solve(const b2_vi_problem* p, double* q0, double* q1, double* v0, double* v1,
                           int32_t* viol, int32_t iterations, void* stream) {
    B2_REQUIRE(p && p->row_begin == 0 && p->row_end == p->n_states, "b2_vi_solve needs the full state range");
    double* q[2] = {q0, q1};
    double* v[2] = {v0, v1};
    for (int k = 0; k < iterations; ++k) {
        int rc = b2_vi_sweep(p, v[k & 1], q[k & 1], q[(k + 1) & 1], v[(k + 1) & 1], viol, k, stream);
        if (rc) return rc;
    }
    return B2_OK;
}

extern "C" int b2_vi_robust_sweep(const b2_vi_problem* p, int32_t n_models, const double* v_in, const double* q_old,
                                  double* q_new, double* v_out, int32_t* viol, int32_t sweep_index, void* stream_) {
    B2_REQUIRE(p && v_in && q_old && q_new && v_out && viol && p->transition && p->reward, "null pointer");
    B2_REQUIRE(n_models > 0 && p->n_actions > 0 && p->row_begin == 0 && p->row_end == p->n_states, "bad shape");
    B2_REQUIRE(p->mode == B2_VI_DETERMINISTIC || p->mode == B2_VI_STOCHASTIC, "robust VI: deterministic or stochastic mode");
    cudaStream_t stream = (cudaStream_t)stream_;
    SweepArgs g;
    memset(&g, 0, sizeof(g));
    g.v_in = v_in; g.q_old = q_old; g.q_new = q_new; g.v_out = v_out; g.viol = viol; g.sweep = sweep_index;
    g.rows = p->n_states; g.row_begin = 0; g.A = p->n_actions; g.gamma = p->gamma; g.rtol = p->rtol; g.atol = p->atol;
    RobustArgs ra;
    ra.transition = p->transition; ra.reward = p->reward; ra.n_models = n_models; ra.dense = p->mode == B2_VI_STOCHASTIC;
    const int64_t n_rows = g.rows * g.A;
    vi_robust_kernel<<<(unsigned)((n_rows + 127) / 128), 128, 0, stream>>>(g, ra);
    vi_rowmax_kernel<<<(unsigned)((g.rows + 255) / 256), 256, 0, stream>>>(g);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
