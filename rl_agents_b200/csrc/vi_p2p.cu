// Slab-sharded value iteration with the exchange step FUSED into the sweep kernel over NVLink peer memory.
//
// value_iteration.py:42-73 sharded over G GPUs (SURVEY 8e): rank g owns the rows [g*S/G, (g+1)*S/G) of
// P / N / R / Q and needs the whole V for its gathers.  Instead of "sweep kernel, then ncclAllGather(V), then
// ncclAllReduce(violations)" (two collective launches per sweep, as long as the sweep itself at S/8 rows),
// every rank holds the V ping-pong buffers in IPC-shared device memory and the sweep kernel
//   * stores V'[s] = max_a Q'[s, a] straight into EVERY rank's copy of V (peer stores over NVLink, issued
//     while the kernel is still streaming P / N -- the transfer overlaps the compute tile by tile),
//   * when its last CTA retires, publishes the slab's allclose violation count and an arrival flag into every
//     peer (system-scope release),
// and the next sweep starts by acquiring all G flags (which is also the write-after-read guard on the buffer it
// is about to overwrite) and summing the G violation counts: zero -> the fixed point was reached one sweep
// earlier and the launch only passes the flag on (the reference's "return the OLD iterate", :70-72).
// No NCCL call, no host round trip inside the fixed-point loop.
#include "common.cuh"

namespace b2 {

__device__ __forceinline__ int ld_acquire_sys(const int32_t* p) {
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(int32_t* p, int v) {
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

struct P2PSweep {
    const double* P;
    const int32_t* N;
    const double* R;
    const uint8_t* term;
    const double* q_old;
    double* q_new;
    int64_t rows, row_begin;
    int A;
    int sweep;
    double gamma, rtol, atol;
    b2_vi_p2p x;
};

template <int B, bool HAS_P>
__global__ void __launch_bounds__(256) vi_sweep_row_p2p_kernel(P2PSweep g) {
    __shared__ int s_conv, s_last;
    const int world = g.x.world, rank = g.x.rank, k = g.sweep;
    const int tid = threadIdx.x;
    // ---- acquire: every peer has finished sweep k-1 (its V' is in my memory; it no longer reads the
    //      buffer this sweep overwrites) ----
    if (tid == 0) s_conv = 0;
    if (k > 0) {
        if (tid < world) {
            // bounded: a peer that never arrives (crashed rank, mismatched launch) must not hang the GPU
            const int32_t* f = g.x.flags[rank] + tid;
            const long long t0 = clock64();
            while (ld_acquire_sys(f) < k) {
                if (*(volatile int32_t*)g.x.status != 0) break;            // a wait already timed out: do not wait again
                if (clock64() - t0 > 2000000000ll) { atomicExch(g.x.status, 1); break; }
            }
        }
        __syncthreads();
        if (tid == 0) {
            int total = 0;
            for (int r = 0; r < world; ++r) total += __ldcg(g.x.parts[rank] + (int64_t)(k - 1) * world + r);
            s_conv = total == 0;
        }
    }
    __syncthreads();
    const bool converged = s_conv != 0;
    int bad = 0;
    if (!converged) {
        const double* v_in = g.x.v[k & 1][rank];
        const int out_i = (k + 1) & 1;
        const int64_t n_sa = g.rows * g.A;
        const int A = g.A;
        for (int64_t qi = (int64_t)blockIdx.x * 256 + tid; qi - tid % 32 < n_sa; qi += (int64_t)gridDim.x * 256) {
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
                for (int b = 0; b < B; ++b) v[b] = __ldcg(v_in + n[b]);   // L2: the point of coherence for peer stores
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
                } else {
                    nv = ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
                }
                if (g.term[qi / A]) nv = 0.0;
                q = __ldcs(g.R + qi) + g.gamma * nv;
                if (!np_isclose(__ldcs(g.q_old + qi), q, g.rtol, g.atol)) bad++;
                __stcs(g.q_new + qi, q);
            }
            double m = q;
            for (int o = 1; o < A; o <<= 1) m = np_max(m, __shfl_xor_sync(0xffffffffu, m, o));
            // the exchange step: V'[s] into every rank's copy (own copy first)
            if (live && (qi % A) == 0) {
                const int64_t s = g.row_begin + qi / A;
                for (int r = 0; r < world; ++r) g.x.v[out_i][(rank + r) % world][s] = m;
            }
        }
        bad = __reduce_add_sync(0xffffffffu, bad);
        if ((tid & 31) == 0 && bad) atomicAdd(g.x.viol_local + k, bad);
    }
    // ---- release: the last CTA to retire publishes this rank's violation count and its arrival flag ----
    __syncthreads();
    if (tid == 0) {
        __threadfence_system();
        s_last = atomicAdd(g.x.done + k, 1u) == gridDim.x - 1;
        __threadfence();
    }
    __syncthreads();
    if (s_last && tid < world) {
        const int mine = converged ? 0 : __ldcg(g.x.viol_local + k);
        g.x.parts[tid][(int64_t)k * world + rank] = mine;
        __threadfence_system();
        st_release_sys(g.x.flags[tid] + rank, k + 1);
    }
}

}  // namespace b2

using namespace b2;

extern "C" int b2_p2p_alloc(int64_t bytes, void** ptr) {
    B2_REQUIRE(ptr && bytes > 0, "bad size");
    B2_CUDA_CHECK(cudaMalloc(ptr, (size_t)bytes));
    B2_CUDA_CHECK(cudaMemset(*ptr, 0, (size_t)bytes));
    return B2_OK;
}
extern "C" int b2_p2p_free(void* ptr) {
    if (ptr) B2_CUDA_CHECK(cudaFree(ptr));
    return B2_OK;
}
extern "C" int b2_p2p_export(void* ptr, unsigned char* handle64) {
    B2_REQUIRE(ptr && handle64, "null pointer");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    B2_CUDA_CHECK(cudaIpcGetMemHandle(&h, ptr));
    memcpy(handle64, &h, 64);
    return B2_OK;
}
extern "C" int b2_p2p_import(const unsigned char* handle64, void** peer_ptr) {
    B2_REQUIRE(handle64 && peer_ptr, "null pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    B2_CUDA_CHECK(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return B2_OK;
}
extern "C" int b2_p2p_close(void* peer_ptr) {
    if (peer_ptr) B2_CUDA_CHECK(cudaIpcCloseMemHandle(peer_ptr));
    return B2_OK;
}
extern "C" int b2_p2p_memset(void* ptr, int32_t value, int64_t bytes, void* stream) {
    B2_REQUIRE(ptr && bytes >= 0, "bad argument");
    B2_CUDA_CHECK(cudaMemsetAsync(ptr, value, (size_t)bytes, (cudaStream_t)stream));
    return B2_OK;
}
extern "C" int b2_p2p_read(void* dst_host, const void* src_dev, int64_t bytes, void* stream) {
    B2_REQUIRE(dst_host && src_dev && bytes >= 0, "bad argument");
    B2_CUDA_CHECK(cudaMemcpyAsync(dst_host, src_dev, (size_t)bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    B2_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
    return B2_OK;
}

extern "C" int b2_vi_sweep_p2p(const b2_vi_problem* p, const b2_vi_p2p* x, const double* q_old, double* q_new,
                               int32_t sweep_index, void* stream_) {
    B2_REQUIRE(p && x && q_old && q_new, "null pointer");
    B2_REQUIRE(x->world >= 1 && x->world <= B2_MAX_PEERS && x->rank >= 0 && x->rank < x->world, "bad world / rank");
    B2_REQUIRE(p->mode == B2_VI_SPARSE || p->mode == B2_VI_DETERMINISTIC, "p2p sweep: sparse or deterministic mode");
    B2_REQUIRE(p->reward && p->transition && p->terminal, "tables missing");
    B2_REQUIRE(sweep_index >= 0 && p->row_end > p->row_begin && p->row_end <= p->n_states, "bad shape");
    for (int r = 0; r < x->world; ++r)
        B2_REQUIRE(x->v[0][r] && x->v[1][r] && x->flags[r] && x->parts[r], "peer pointer missing");
    B2_REQUIRE(x->viol_local && x->done && x->status, "scratch missing");
    P2PSweep g;
    g.R = p->reward; g.term = p->terminal; g.q_old = q_old; g.q_new = q_new;
    g.rows = p->row_end - p->row_begin; g.row_begin = p->row_begin; g.A = p->n_actions; g.sweep = sweep_index;
    g.gamma = p->gamma; g.rtol = p->rtol; g.atol = p->atol; g.x = *x;
    int B;
    if (p->mode == B2_VI_SPARSE) {
        B2_REQUIRE(p->next && p->n_next > 0, "sparse mode needs next[]");
        g.P = (const double*)p->transition; g.N = p->next; B = p->n_next;
    } else {
        g.P = nullptr; g.N = (const int32_t*)p->transition; B = 1;
    }
    if (!((g.A & (g.A - 1)) == 0 && g.A <= 32 && (B == 1 || B == 2 || B == 4 || B == 8) && (uintptr_t)g.N % 16 == 0 &&
          (!g.P || (uintptr_t)g.P % 16 == 0))) {
        set_error("p2p sweep supports A a power of two <= 32 and B in {1,2,4,8} (got A=%d B=%d)", g.A, B);
        return B2_ERR_UNSUPPORTED;
    }
    const int64_t n_sa = g.rows * g.A;
    const int64_t blocks = (n_sa + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;       // all CTAs resident: they start by spinning on the flags
    const unsigned grid = (unsigned)(blocks < cap ? blocks : cap);
    cudaStream_t stream = (cudaStream_t)stream_;
#define B2_ROW(BB)                                                                    \
    if (g.P) vi_sweep_row_p2p_kernel<BB, true><<<grid, 256, 0, stream>>>(g);          \
    else vi_sweep_row_p2p_kernel<BB, false><<<grid, 256, 0, stream>>>(g)
    if (B == 1) { B2_ROW(1); } else if (B == 2) { B2_ROW(2); } else if (B == 4) { B2_ROW(4); } else { B2_ROW(8); }
#undef B2_ROW
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
