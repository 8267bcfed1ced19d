// Wavefront OPD: ONE decision searched by the whole GPU (b2_opd_plan_wave).
//
// The reference's OptimisticDeterministicPlanner.run (deterministic.py:106-114) expands one leaf per
// iteration -- a chain of `budget / n_actions` dependent env transitions.
// The wavefront expands, per wave, the k = min(width, expansions left, frontier size) best
// leaves in the reference's own arg-max order (value_upper descending, node id ascending, :110), in
// increasing node-id order, and simulates all their children at once on every SM.  width = 1 is the
// reference's algorithm; the specification for any width is oracle/planners.py::opd_plan_wavefront, and the
// kernel is bit-identical with it (node ids, counts, fp64 bounds).
//
// One cooperative launch, one CTA per SM, waves separated by two grid barriers:
//   select (CTA 0)  the k-th largest frontier key by bisection over the order-preserving 64-bit image of
//                   the fp64 keys staged in shared memory (early exit as soon as a threshold isolates
//                   exactly k keys), ties at the threshold by lowest node id, ordered compaction, child
//                   ids by prefix sum of the leaves' available-action counts -> work list
//   simulate (all)  one 16-lane group per child: parent scene -> hw::step -> child scene, node record and
//                   frontier key (value_upper) written in place; finite MDPs: one thread per child
// then CTA 0 runs the bottom-up pass (counts :64-65, backup_to_root :74-79) wave by wave in reverse and the
// greedy plan walk (abstract.py:143-156).
#include <cooperative_groups.h>

#include "common.cuh"
#include "highway_lite.cuh"
#include "intersection_lite.cuh"

namespace b2 {
namespace wave {

#ifndef B2_WAVE_THREADS
#define B2_WAVE_THREADS 256
#endif
constexpr int THREADS = B2_WAVE_THREADS;
constexpr int WARPS = THREADS / 32;
constexpr int STAGE_CAP = 24576;            // fp64 keys staged in shared memory per tile (192 KB)
constexpr int MAX_BRANCH = 8;

struct Control {                            // head of the workspace; zeroed by the launch wrapper
    unsigned bar_count, bar_gen;
    int n_nodes, n_expanded, wave_children, wave_base, n_waves, stop;
    int error, max_depth, term_exp, pad;
    long long prof[8];   // CTA 0 clock64 totals: 0 stage, 1 range+bisection, 2 compaction+layout, 3 barrier after select,
                         // 4 simulate (CTA 0's share), 5 barrier after simulate, 6 bottom-up + plan, 7 bisection steps
};

constexpr int MAX_STEPS = 80;
struct DistScratch {                        // cross-CTA reductions of the distributed selection, by wave parity
    unsigned long long gmin[2], gmax[2];
    unsigned gt[2], pad[2];
    unsigned counts[2][MAX_STEPS][4];
};

struct Args {
    b2_opd_wave_config cfg;
    b2_opd_tree tree;
    const int32_t* root_state;
    Control* ctl;
    double* keys;          // [node_capacity] value_upper of frontier leaves, -inf otherwise
    int32_t* exp_order;    // [n_expansions] expanded leaves, wave-major, id order inside a wave
    int32_t* wave_start;   // [n_expansions + 1]
    int32_t* work;         // [width * n_actions] leaf | action << 28 for every child of the current wave
    double* lowerv;        // joint (robust) mode: [node_capacity, n_models] per-model value_lower along the node's path
    double* wave_up;       // joint mode: [width * n_actions, n_models] per-model value_upper of the wave's children
    int32_t* wave_flags;   // joint mode: done | avail << 8 | reward-out-of-range << 16, per (child, model)
    DistScratch* dscr;     // distributed selection (trees larger than one shared-memory tile)
    int2* cta_cnt;         // [grid] per-CTA (taken-by-threshold, equal-to-threshold) counts
    // speculative strict search (opd_spec_kernel)
    int32_t* work_slot;    // [width * n_actions] arena slot of every transition of the current wave
    int32_t* cand;         // [width] the wave's candidate leaves, id order
    int32_t* spec_base;    // [node_capacity] first arena slot of a leaf's cached children, -1: not simulated yet
    int32_t* state_slot;   // [node_capacity] arena slot holding the node's own state
    double* spec_reward;   // [arena slots] reward of the cached transition
    int32_t* spec_flags;   // [arena slots] action | done << 16 | reward-out-of-range << 17 | avail << 24
    int8_t* plan;
    int32_t* result;
};

__device__ __forceinline__ unsigned long long sortable(double x) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(x);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
constexpr unsigned long long ABSENT = 0x000fffffffffffffull;   // image of -inf: not a frontier leaf

__device__ __forceinline__ int ld_cg(const int32_t* p) { return __ldcg(p); }
__device__ __forceinline__ double ld_cg(const double* p) { return __ldcg(p); }

// Data written before a grid barrier (common.cuh) by any CTA is read after it with ld.global.cg (L2) by the others.

__device__ __forceinline__ int block_sum(int v, int* red, int slot) {   // red: [2][WARPS]; slot alternates
    const int w = __reduce_add_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0) red[slot * WARPS + (threadIdx.x >> 5)] = w;
    __syncthreads();
    int s = 0;
#pragma unroll
    for (int i = 0; i < WARPS; ++i) s += red[slot * WARPS + i];
    return s;
}

struct SelShared {
    int red[4 * WARPS];        // two slots x two packed words
    int scan_a[THREADS], scan_b[THREADS];
    unsigned long long theta;
    int k, need_eq, total_children;
};

// exclusive prefix sums of (a, b) over the block; returns totals through ta/tb
__device__ __forceinline__ void block_scan2(int a, int b, SelShared& sh, int& ea, int& eb, int& ta, int& tb) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int ia = a, ib = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int xa = __shfl_up_sync(0xffffffffu, ia, o), xb = __shfl_up_sync(0xffffffffu, ib, o);
        if (lane >= o) { ia += xa; ib += xb; }
    }
    if (lane == 31) { sh.scan_a[warp] = ia; sh.scan_b[warp] = ib; }
    __syncthreads();
    int wa = 0, wb = 0;
    ta = 0; tb = 0;
#pragma unroll
    for (int i = 0; i < WARPS; ++i) {
        const int va = sh.scan_a[i], vb = sh.scan_b[i];
        if (i < warp) { wa += va; wb += vb; }
        ta += va; tb += vb;
    }
    ea = wa + ia - a;
    eb = wb + ib - b;
    __syncthreads();
}

// CTA 0: lay out the children of the k chosen leaves (exp_order[n_expanded .. n_expanded + k), id order):
// child ids by prefix sum of the available-action counts, parent records, work list.
// JOINT_IL: IntersectionLite with n_models > 0 (see opd_wave_kernel).
template <bool JOINT_IL>
__device__ int layout_wave(const Args& a, SelShared& sh, unsigned long long* skeys, bool resident, int n_nodes,
                           int n_expanded, int k, int slot, long long* prof) {
    const int tid = threadIdx.x;
    long long t0 = clock64();
    const int32_t* sel = a.exp_order + n_expanded;
    // ---- children layout: ids by prefix sum of the available-action counts, in leaf-id order ----
    int run = 0, term = 0;
    for (int j0 = 0; j0 < k; j0 += THREADS) {
        const int j = j0 + tid;
        int leaf = 0, mask = 0, n = 0, meta = 0;
        if (j < k) {
            leaf = __ldcg(sel + j);
            meta = __ldcg(a.tree.meta + leaf);
            mask = a.cfg.env_kind != B2_ENV_FINITE ? (meta >> 24) & 0x1f : (1 << a.cfg.n_actions) - 1;
            n = __popc(mask);
            term += (meta >> 16) & 1;
        }
        int en, e2, tn, t2;
        block_scan2(n, 0, sh, en, e2, tn, t2);
        if (j < k) {
            const int c0 = n_nodes + run + en;
            a.tree.first_child[leaf] = c0;
            a.tree.meta[leaf] = meta | (n << 8);
            a.keys[leaf] = -INFINITY;
            if (resident) skeys[leaf] = ABSENT;
            int q = 0;
            for (int act_i = 0; act_i < MAX_BRANCH; ++act_i) {
                int act;
                if (a.cfg.env_kind == B2_ENV_HIGHWAY && a.cfg.n_models == 0) {
                    if (act_i >= 5) break;
                    const int order[5] = {hw::A_IDLE, hw::A_LEFT, hw::A_RIGHT, hw::A_FASTER, hw::A_SLOWER};
                    act = order[act_i];
                } else if (a.cfg.env_kind == B2_ENV_INTERSECTION && !JOINT_IL) {
                    if (act_i >= 3) break;
                    const int order[3] = {il::A_IDLE, il::A_FASTER, il::A_SLOWER};
                    act = order[act_i];
                } else {     // finite MDPs, and JointEnv.get_available_actions (robust.py:22-26): ascending ids
                    if (act_i >= a.cfg.n_actions) break;
                    act = act_i;
                }
                if (mask & (1 << act)) {
                    a.work[run + en + q] = leaf | (act << 28);
                    ++q;
                }
            }
        }
        run += tn;
    }
    term = block_sum(term, sh.red, slot);
    if (tid == 0) {
        Control* c = a.ctl;
        c->term_exp += term;
        a.wave_start[c->n_waves] = n_expanded;
        c->n_waves += 1;
        a.wave_start[c->n_waves] = n_expanded + k;
        c->wave_base = n_nodes;
        c->wave_children = run;
        c->n_nodes = n_nodes + run;
        c->n_expanded = n_expanded + k;
        prof[2] += clock64() - t0;
    }
    return run;
}

// ALL CTAs (trees that do not fit one shared-memory tile): the same selection with the key array split in
// contiguous id slices, one per CTA; every reduction of the search (range, threshold counts, tie count,
// compaction offsets) goes through global atomics + a grid barrier, so all CTAs take identical decisions.
// Leaves the wave's k leaves in exp_order[n_expanded ..) in id order and returns k (0: search finished).
__device__ int select_dist(const Args& a, SelShared& sh, unsigned long long* skeys, int n_nodes, int n_expanded,
                           int wave, unsigned n_ctas) {
    const int tid = threadIdx.x, bid = blockIdx.x;
    const int remaining = a.cfg.n_expansions - n_expanded;
    const int frontier = n_nodes - n_expanded;
    const int k = min(min(a.cfg.width, remaining), frontier);
    if (k <= 0) return 0;
    const int par = wave & 1;
    DistScratch* d = a.dscr;
    volatile DistScratch* vd = a.dscr;
    const int L = (n_nodes + (int)n_ctas - 1) / (int)n_ctas;
    const int sb = min(bid * L, n_nodes), se = min(sb + L, n_nodes), len = se - sb;
    const int n_tiles = (len + STAGE_CAP - 1) / STAGE_CAP;
    auto stage = [&](int tile) {
        const int base = sb + tile * STAGE_CAP, n = min(STAGE_CAP, se - base);
        __syncthreads();
#pragma unroll 8
        for (int i = tid; i < n; i += THREADS) skeys[i] = sortable(__ldcg(a.keys + base + i));
        __syncthreads();
        return n;
    };
    auto chunk_of = [&](int n, int& lo, int& hi) {
        const int c = ((n + THREADS - 1) / THREADS) | 1;
        lo = min(tid * c, n);
        hi = min(lo + c, n);
    };
    // the other parity's scratch is idle: reset it for the next wave
    if (bid == 0) {
        if (tid == 0) { d->gmin[par ^ 1] = ~0ull; d->gmax[par ^ 1] = 0ull; d->gt[par ^ 1] = 0u; }
        for (int i = tid; i < MAX_STEPS * 4; i += THREADS) (&d->counts[par ^ 1][0][0])[i] = 0u;
    }
    int n0 = n_tiles > 0 ? stage(0) : 0;
    int slot = 0;
    // ---- range of the frontier keys ----
    {
        unsigned long long mx = 0, mn = ~0ull;
        for (int t = 0; t < n_tiles; ++t) {
            const int n = t == 0 ? n0 : stage(t);
            int b, e;
            chunk_of(n, b, e);
#pragma unroll 8
            for (int i = b; i < e; ++i) {
                const unsigned long long u = skeys[i];
                if (u > ABSENT) { mx = max(mx, u); mn = min(mn, u); }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        }
        if ((tid & 31) == 0 && mx > ABSENT) { atomicMax(&d->gmax[par], mx); atomicMin(&d->gmin[par], mn); }
    }
    grid_barrier(a.ctl, n_ctas);
    unsigned long long lo = vd->gmin[par], hi = vd->gmax[par], theta = 0;
    bool exact = false;
    if (k == frontier) { theta = lo; exact = true; }
    int step = 0;
    while (!exact) {
        if (lo == hi) { theta = lo; break; }
        const unsigned long long range = hi - lo, fifth = range / 5;
        unsigned long long m[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) m[j] = range >= 5 ? lo + fifth * (j + 1) : min(lo + (unsigned long long)(j + 1), hi);
        int c[4] = {0, 0, 0, 0};
        for (int t = 0; t < n_tiles; ++t) {
            const int n = n_tiles == 1 ? n0 : stage(t);
            int b, e;
            chunk_of(n, b, e);
            int c01 = 0, c23 = 0;
#pragma unroll 8
            for (int i = b; i < e; ++i) {
                const unsigned long long u = skeys[i];
                c01 += (u >= m[0] ? 1 : 0) + (u >= m[1] ? 0x10000 : 0);
                c23 += (u >= m[2] ? 1 : 0) + (u >= m[3] ? 0x10000 : 0);
            }
            const int w01 = __reduce_add_sync(0xffffffffu, c01), w23 = __reduce_add_sync(0xffffffffu, c23);
            if ((tid & 31) == 0) { sh.red[slot * 2 * WARPS + (tid >> 5)] = w01; sh.red[slot * 2 * WARPS + WARPS + (tid >> 5)] = w23; }
            __syncthreads();
            int s01 = 0, s23 = 0;
#pragma unroll
            for (int i = 0; i < WARPS; ++i) { s01 += sh.red[slot * 2 * WARPS + i]; s23 += sh.red[slot * 2 * WARPS + WARPS + i]; }
            slot ^= 1;
            c[0] += s01 & 0xffff; c[1] += (unsigned)s01 >> 16; c[2] += s23 & 0xffff; c[3] += (unsigned)s23 >> 16;
        }
        if (tid < 4 && c[tid] != 0) atomicAdd(&d->counts[par][step][tid], (unsigned)c[tid]);
        grid_barrier(a.ctl, n_ctas);
        int j_gt = -1;
        bool hit = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int cj = (int)vd->counts[par][step][j];
            if (cj == k && !hit) { theta = m[j]; hit = true; }
            if (cj > k) j_gt = j;
        }
        ++step;
        if (hit) { exact = true; break; }
        const unsigned long long new_hi = j_gt < 3 ? m[j_gt + 1] - 1 : hi;
        if (j_gt >= 0) lo = m[j_gt];
        hi = new_hi;
    }
    int need_eq = 0;
    if (!exact) {
        int c = 0;
        for (int t = 0; t < n_tiles; ++t) {
            const int n = n_tiles == 1 ? n0 : stage(t);
            int b, e;
            chunk_of(n, b, e);
#pragma unroll 8
            for (int i = b; i < e; ++i) c += skeys[i] > theta ? 1 : 0;
        }
        c = block_sum(c, sh.red, slot);
        slot ^= 1;
        if (tid == 0 && c) atomicAdd(&d->gt[par], (unsigned)c);
        grid_barrier(a.ctl, n_ctas);
        need_eq = k - (int)vd->gt[par];
    }
    // ---- compaction, pass 1: this CTA's totals ----
    {
        int cg = 0, ce = 0;
        for (int t = 0; t < n_tiles; ++t) {
            const int n = n_tiles == 1 ? n0 : stage(t);
            int b, e;
            chunk_of(n, b, e);
#pragma unroll 8
            for (int i = b; i < e; ++i) {
                const unsigned long long u = skeys[i];
                if (exact) cg += u >= theta ? 1 : 0;
                else { cg += u > theta ? 1 : 0; ce += u == theta ? 1 : 0; }
            }
        }
        int eg, ee, tg, te;
        block_scan2(cg, ce, sh, eg, ee, tg, te);
        if (tid == 0) a.cta_cnt[bid] = make_int2(tg, te);
    }
    grid_barrier(a.ctl, n_ctas);
    // ---- pass 2: offsets of the CTAs before this one, then ordered writes ----
    int gt_before, eq_before;
    {
        int pg = 0, pe = 0;
        if (tid < bid) {
            const int2 v = __ldcg(a.cta_cnt + tid);
            pg = v.x; pe = v.y;
        }
        int eg, ee;
        block_scan2(pg, pe, sh, eg, ee, gt_before, eq_before);
    }
    int32_t* sel = a.exp_order + n_expanded;
    int run_sel = gt_before + min(eq_before, need_eq), run_eq = eq_before;
    for (int t = 0; t < n_tiles; ++t) {
        const int n = n_tiles == 1 ? n0 : stage(t);
        const int base = sb + t * STAGE_CAP;
        int b, e;
        chunk_of(n, b, e);
        int cg = 0, ce = 0;
#pragma unroll 8
        for (int i = b; i < e; ++i) {
            const unsigned long long u = skeys[i];
            if (exact) cg += u >= theta ? 1 : 0;
            else { cg += u > theta ? 1 : 0; ce += u == theta ? 1 : 0; }
        }
        int eg, ee, tg, te;
        block_scan2(cg, ce, sh, eg, ee, tg, te);
        int eq_seen = run_eq + ee;
        int pos = run_sel + eg + min(eq_seen, need_eq) - min(run_eq, need_eq);
        for (int i = b; i < e; ++i) {
            const unsigned long long u = skeys[i];
            bool take;
            if (exact) take = u >= theta;
            else if (u > theta) take = true;
            else if (u == theta) { take = eq_seen < need_eq; ++eq_seen; }
            else take = false;
            if (take) sel[pos++] = base + i;
        }
        run_sel += tg + min(run_eq + te, need_eq) - min(run_eq, need_eq);
        run_eq += te;
    }
    grid_barrier(a.ctl, n_ctas);
    return k;
}

// CTA 0: choose this wave's leaves and lay out their children.  Returns the number of children (0: done).
// `sel_out` / `do_layout`: the speculative kernel takes the chosen leaves (id order) in its own array and lays the
// wave out itself; it then returns k.
template <bool JOINT_IL = false>
__device__ int select_wave(const Args& a, SelShared& sh, unsigned long long* skeys, int n_nodes, int n_expanded,
                           int staged_nodes, long long* prof, int32_t* sel_out = nullptr, bool do_layout = true) {
    const int tid = threadIdx.x;
    long long t0 = clock64();
    const int remaining = a.cfg.n_expansions - n_expanded;
    const int frontier = n_nodes - n_expanded;
    const int k = min(min(a.cfg.width, remaining), frontier);
    if (k <= 0) return 0;
    // a tree that fits one tile keeps its keys resident in shared memory: only the children of the previous
    // wave (ids >= staged_nodes) are fetched; larger trees are streamed tile by tile on every pass
    const bool resident = a.cfg.node_capacity <= STAGE_CAP;
    const int n_tiles = resident ? 1 : (n_nodes + STAGE_CAP - 1) / STAGE_CAP;
    auto stage = [&](int tile) {
        const int base = tile * STAGE_CAP, n = min(STAGE_CAP, n_nodes - base);
        __syncthreads();
#pragma unroll 8
        for (int i = tid; i < n; i += THREADS) skeys[i] = sortable(__ldcg(a.keys + base + i));
        __syncthreads();
        return n;
    };
    // blocked partition of a tile with an odd chunk (conflict-free 8-byte shared loads)
    auto chunk_of = [&](int n, int& lo, int& hi) {
        const int c = ((n + THREADS - 1) / THREADS) | 1;
        lo = min(tid * c, n);
        hi = min(lo + c, n);
    };
    int n0;
    if (resident) {
        for (int i = staged_nodes + tid; i < n_nodes; i += THREADS) skeys[i] = sortable(__ldcg(a.keys + i));
        __syncthreads();
        n0 = n_nodes;
    } else {
        n0 = stage(0);
    }
    if (tid == 0) { const long long t1 = clock64(); prof[0] += t1 - t0; t0 = t1; }
    // ---- bisection on the 64-bit images: largest theta with count(u >= theta) >= k ----
    unsigned long long lo = ABSENT + 1, hi = ~0ull;    // invariant: count(u >= lo) >= k
    unsigned long long theta = 0;
    bool exact = false;                                 // count(u >= theta) == k: no tie handling needed
    int slot = 0;
    {
        // tighten [lo, hi] to the frontier's own range first (two reductions instead of ~12 bisection steps)
        unsigned long long mx = 0, mn = ~0ull;
        for (int t = 0; t < n_tiles; ++t) {
            const int n = t == 0 ? n0 : stage(t);
            int b, e;
            chunk_of(n, b, e);
#pragma unroll 8
            for (int i = b; i < e; ++i) {
                const unsigned long long u = skeys[i];
                if (u > ABSENT) { mx = max(mx, u); mn = min(mn, u); }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        }
        unsigned long long* r64 = reinterpret_cast<unsigned long long*>(sh.scan_a);
        __syncthreads();
        if ((tid & 31) == 0) { r64[tid >> 5] = mx; r64[WARPS + (tid >> 5)] = mn; }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < WARPS; ++i) { mx = max(mx, r64[i]); mn = min(mn, r64[WARPS + i]); }
        __syncthreads();
        lo = mn; hi = mx;
    }
    if (k == frontier) { theta = lo; exact = true; }
    int steps = 0;
    while (!exact) {
        ++steps;
        if (lo == hi) { theta = lo; break; }
        // five-way split: four thresholds lo < m1 <= m2 <= m3 <= m4 <= hi per pass over the keys
        const unsigned long long range = hi - lo, fifth = range / 5;
        unsigned long long m[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) m[j] = range >= 5 ? lo + fifth * (j + 1) : min(lo + (unsigned long long)(j + 1), hi);
        int c01 = 0, c23 = 0;                       // two 16-bit counters per word (a tile holds < 2^15 keys)
        int c[4] = {0, 0, 0, 0};
        for (int t = 0; t < n_tiles; ++t) {
            const int n = n_tiles == 1 ? n0 : stage(t);
            int b, e;
            chunk_of(n, b, e);
            c01 = 0; c23 = 0;
#pragma unroll 8
            for (int i = b; i < e; ++i) {
                const unsigned long long u = skeys[i];
                c01 += (u >= m[0] ? 1 : 0) + (u >= m[1] ? 0x10000 : 0);
                c23 += (u >= m[2] ? 1 : 0) + (u >= m[3] ? 0x10000 : 0);
            }
            // block totals of both packed words in one barrier
            const int w01 = __reduce_add_sync(0xffffffffu, c01), w23 = __reduce_add_sync(0xffffffffu, c23);
            if ((tid & 31) == 0) { sh.red[slot * 2 * WARPS + (tid >> 5)] = w01; sh.red[slot * 2 * WARPS + WARPS + (tid >> 5)] = w23; }
            __syncthreads();
            int s01 = 0, s23 = 0;
#pragma unroll
            for (int i = 0; i < WARPS; ++i) { s01 += sh.red[slot * 2 * WARPS + i]; s23 += sh.red[slot * 2 * WARPS + WARPS + i]; }
            slot ^= 1;
            c[0] += s01 & 0xffff; c[1] += (unsigned)s01 >> 16; c[2] += s23 & 0xffff; c[3] += (unsigned)s23 >> 16;
        }
        int j_gt = -1;                               // largest j with count(u >= m[j]) > k
        bool hit = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (c[j] == k && !hit) { theta = m[j]; hit = true; }
            if (c[j] > k) j_gt = j;
        }
        if (hit) { exact = true; break; }
        const unsigned long long new_hi = j_gt < 3 ? m[j_gt + 1] - 1 : hi;
        if (j_gt >= 0) lo = m[j_gt];
        hi = new_hi;
    }
    if (tid == 0) { const long long t1 = clock64(); prof[1] += t1 - t0; t0 = t1; prof[7] += steps; }
    // ---- ordered compaction: keys > theta, then the lowest ids among keys == theta ----
    int need_eq = 0;
    if (!exact) {
        int c = 0;
        for (int t = 0; t < n_tiles; ++t) {
            const int n = n_tiles == 1 ? n0 : stage(t);
            int b, e;
            chunk_of(n, b, e);
#pragma unroll 8
            for (int i = b; i < e; ++i) c += skeys[i] > theta ? 1 : 0;
        }
        c = block_sum(c, sh.red, slot);
        slot ^= 1;
        need_eq = k - c;
    }
    int32_t* sel = sel_out ? sel_out : a.exp_order + n_expanded;     // the wave's leaves, id order (doubles as the expansion record)
    int run_sel = 0, run_eq = 0;
    for (int t = 0; t < n_tiles; ++t) {
        const int n = n_tiles == 1 ? n0 : stage(t);
        const int base = t * STAGE_CAP;
        int b, e;
        chunk_of(n, b, e);
        int cg = 0, ce = 0;
#pragma unroll 8
        for (int i = b; i < e; ++i) {
            const unsigned long long u = skeys[i];
            if (exact) cg += u >= theta ? 1 : 0;
            else { cg += u > theta ? 1 : 0; ce += u == theta ? 1 : 0; }
        }
        int eg, ee, tg, te;
        block_scan2(cg, ce, sh, eg, ee, tg, te);
        int eq_seen = run_eq + ee;
        int pos = run_sel + eg + min(eq_seen, need_eq) - min(run_eq, need_eq);
        for (int i = b; i < e; ++i) {
            const unsigned long long u = skeys[i];
            bool take;
            if (exact) take = u >= theta;
            else if (u > theta) take = true;
            else if (u == theta) { take = eq_seen < need_eq; ++eq_seen; }
            else take = false;
            if (take) sel[pos++] = base + i;
        }
        run_sel += tg + min(run_eq + te, need_eq) - min(run_eq, need_eq);
        run_eq += te;
    }
    __syncthreads();
    if (tid == 0) prof[2] += clock64() - t0;
    if (!do_layout) return k;
    return layout_wave<JOINT_IL>(a, sh, skeys, resident, n_nodes, n_expanded, k, slot, prof);
}

// node record of a new child: DeterministicNode.__init__ / update (deterministic.py:10-19, 45-63)
__device__ __forceinline__ void write_child(const Args& a, int c, int leaf, int action, double r, bool done, int avail) {
    const b2_opd_tree& tr = a.tree;
    const int d = ld_cg(tr.depth + leaf) + 1;
    double lo = ld_cg(tr.lower + leaf) + a.cfg.gamma_pow[d - 1] * r;
    double up = lo + a.cfg.gamma_pow_div[d];
    if (done) {
        lo = lo + a.cfg.terminal_bonus[d];
        up = lo;
    }
    tr.parent[c] = leaf;
    tr.first_child[c] = -1;
    tr.depth[c] = d;
    tr.count[c] = 2;
    tr.meta[c] = action | (done ? 1 << 16 : 0) | (avail << 24);
    tr.reward[c] = r;
    tr.lower[c] = lo;
    tr.upper[c] = up;
    a.keys[c] = up;
    if (!(r >= 0.0 && r <= 1.0)) a.ctl->error = 1;     // :46-47
    atomicMax(&a.ctl->max_depth, d);
}

__device__ __forceinline__ void load_state_cg(const int32_t* w, int li, hw::Lane& L, int& t, int& si) {
    L.x = __int_as_float(__ldcg(w + 0 * hw::V + li));
    L.y = __int_as_float(__ldcg(w + 1 * hw::V + li));
    L.h = __int_as_float(__ldcg(w + 2 * hw::V + li));
    L.v = __int_as_float(__ldcg(w + 3 * hw::V + li));
    L.ts = __int_as_float(__ldcg(w + 4 * hw::V + li));
    L.timer = __int_as_float(__ldcg(w + 5 * hw::V + li));
    L.tgt = __ldcg(w + 6 * hw::V + li);
    L.flags = __ldcg(w + 7 * hw::V + li);
    t = __ldcg(w + 8 * hw::V + 0);
    si = __ldcg(w + 8 * hw::V + 1);
}

// Joint (robust) mode, per (child, model): the model's own path bounds (deterministic.py:52-59 with vector
// rewards / terminals); the node's bounds are their minima over the models (robust.py:40-47), taken by
// finalize_joint_children once every model of the wave has been simulated.
__device__ __forceinline__ void write_model_bounds(const Args& a, int task, int c, int leaf, int m, double r, bool done,
                                                   int avail) {
    const int M = a.cfg.n_models;
    const int d = ld_cg(a.tree.depth + leaf) + 1;
    double lo = ld_cg(a.lowerv + (int64_t)leaf * M + m) + a.cfg.gamma_pow[d - 1] * r;
    double up = lo + a.cfg.gamma_pow_div[d];
    if (done) {
        lo = lo + a.cfg.terminal_bonus[d];
        up = lo;
    }
    a.lowerv[(int64_t)c * M + m] = lo;
    a.wave_up[task] = up;
    a.wave_flags[task] = (done ? 1 : 0) | (avail << 8) | ((r >= 0.0 && r <= 1.0) ? 0 : 1 << 16);
}

__device__ __forceinline__ void finalize_joint_children(const Args& a, int total, int base, unsigned n_ctas) {
    const int M = a.cfg.n_models;
    const b2_opd_tree& tr = a.tree;
    for (int w = blockIdx.x * THREADS + threadIdx.x; w < total; w += THREADS * (int)n_ctas) {
        const int item = __ldcg(a.work + w);
        const int leaf = item & 0x0fffffff, action = (item >> 28) & 7;
        const int c = base + w;
        const int d = ld_cg(tr.depth + leaf) + 1;
        double lo = INFINITY, up = INFINITY;
        int done_all = 1, avail = 0, bad = 0;
        for (int m = 0; m < M; ++m) {
            const double l2 = __ldcg(a.lowerv + (int64_t)c * M + m), u2 = __ldcg(a.wave_up + (int64_t)w * M + m);
            const int f = __ldcg(a.wave_flags + (int64_t)w * M + m);
            lo = l2 < lo ? l2 : lo;          // np.min over the models (robust.py:41-44)
            up = u2 < up ? u2 : up;
            done_all &= f & 1;
            avail |= (f >> 8) & 0xff;
            bad |= f >> 16;
        }
        tr.parent[c] = leaf;
        tr.first_child[c] = -1;
        tr.depth[c] = d;
        tr.count[c] = 2;
        tr.meta[c] = action | (done_all ? 1 << 16 : 0) | (avail << 24);
        tr.reward[c] = 0.0;
        tr.lower[c] = lo;
        tr.upper[c] = up;
        a.keys[c] = up;
        if (bad) a.ctl->error = 1;
        atomicMax(&a.ctl->max_depth, d);
    }
}

// CTA 0, once the search is over: counts and bounds bottom-up, wave by wave in reverse, then the greedy plan.
__device__ void finish_tree(const Args& a, long long tp) {
    const int tid = threadIdx.x, lane = tid & 31;
    Control* ctl = a.ctl;
    const b2_opd_tree& tr = a.tree;
    // ------------------------------------------------------------------ bottom-up pass, reverse wave order
    const volatile Control* vc = ctl;
    const int n_waves = vc->n_waves, n_exp = vc->n_expanded, n_nodes = vc->n_nodes;
    for (int w = n_waves - 1; w >= 0; --w) {
        const int b = a.wave_start[w], e = a.wave_start[w + 1];
        for (int j = b + tid; j < e; j += THREADS) {
            const int p = a.exp_order[j];
            const int fc = tr.first_child[p];
            const int n = (tr.meta[p] >> 8) & 0xff;
            double lo = -INFINITY, up = -INFINITY;
            int desc = 0;
            for (int q = 0; q < n; ++q) {
                const double l2 = ld_cg(tr.lower + fc + q), u2 = ld_cg(tr.upper + fc + q);
                lo = l2 > lo ? l2 : lo;
                up = u2 > up ? u2 : up;
                desc += ld_cg(tr.count + fc + q) - 1;
            }
            tr.lower[p] = lo;                       // backup_to_root (:74-79)
            tr.upper[p] = up;
            tr.count[p] = (p == 0 ? 1 : 2) + desc;  // :64-65
        }
        __threadfence();
        __syncthreads();
    }
    if (tid >= 32) return;
    // get_plan (abstract.py:143-156) on value_lower; a tie is broken on the host with the planner RNG
    int node = 0, len = 0, tie_node = -1;
    while (true) {
        const int fc = ld_cg(tr.first_child + node);
        if (fc < 0) break;
        const int n = (ld_cg(tr.meta + node) >> 8) & 0xff;
        const double lo = lane < n ? ld_cg(tr.lower + fc + lane) : -INFINITY;
        const double m = warp_max_f64(lo);
        const unsigned eq = __ballot_sync(0xffffffffu, lane < n && lo == m);
        if (__popc(eq) > 1) { tie_node = node; break; }
        const int c = fc + __ffs(eq) - 1;
        if (lane == 0 && len < a.cfg.plan_capacity) a.plan[len] = (int8_t)(ld_cg(tr.meta + c) & 0xff);
        ++len;
        node = c;
    }
    if (lane == 0) {
        int32_t* res = a.result;
        res[0] = n_nodes;
        res[1] = n_nodes - n_exp;
        res[2] = vc->max_depth;
        res[3] = vc->term_exp;
        res[4] = vc->error;
        res[5] = len;
        res[6] = tie_node;
        res[7] = n_waves;
        ctl->prof[6] += clock64() - tp;
        for (int i = 0; i < 8; ++i) res[8 + i] = (int32_t)(i == 7 ? ctl->prof[i] : ctl->prof[i] >> 8);   // 256-cycle units
    }
}

// JOINT_IL: DROP on IntersectionLite (env_kind INTERSECTION, n_models > 0), an instantiation of its own so that every
// other configuration, plain IntersectionLite included, runs the same code as without it.
template <bool JOINT_IL>
__global__ void __launch_bounds__(THREADS, 1) opd_wave_kernel(Args a) {
    extern __shared__ unsigned long long skeys[];
    __shared__ SelShared sh;
    __shared__ int s_nodes, s_expanded, s_staged;
    const int tid = threadIdx.x, lane = tid & 31, li = tid & 15;
    const unsigned n_ctas = gridDim.x;
    Control* ctl = a.ctl;
    const b2_opd_tree& tr = a.tree;
    const bool hwy = a.cfg.env_kind == B2_ENV_HIGHWAY;
    if (blockIdx.x == 0) {
        // root: DeterministicNode.__init__ (:10-19)
        int avail = 0;
        const int Mx = a.cfg.n_models > 0 ? a.cfg.n_models : 1;
        if (JOINT_IL) {
            for (int i = tid; i < Mx * il::WORDS; i += THREADS) tr.state[i] = a.root_state[i];
            for (int m = 0; m < Mx; ++m)      // JointEnv.get_available_actions: the union over the models
                avail |= il::avail_mask(a.root_state[m * il::WORDS + 129]);
        } else if (a.cfg.env_kind == B2_ENV_INTERSECTION) {
            for (int i = tid; i < il::WORDS; i += THREADS) tr.state[i] = a.root_state[i];
            avail = il::avail_mask(a.root_state[129]);
        } else if (hwy) {
            for (int i = tid; i < Mx * hw::WORDS; i += THREADS) tr.state[i] = a.root_state[i];
            for (int m = 0; m < Mx; ++m)      // JointEnv.get_available_actions: the union over the models
                avail |= hw::avail_mask(__int_as_float(a.root_state[m * hw::WORDS + hw::V]),
                                        a.root_state[m * hw::WORDS + 8 * hw::V + 1]);
        } else if (tid < Mx) {
            tr.state[tid] = a.root_state[tid];
        }
        if (a.cfg.n_models > 0 && tid < a.cfg.n_models) a.lowerv[tid] = 0.0;
        if (tid == 0) {
            tr.parent[0] = -1; tr.first_child[0] = -1; tr.depth[0] = 0; tr.count[0] = 1;
            tr.meta[0] = 0xff | (avail << 24);
            tr.reward[0] = 0.0; tr.lower[0] = 0.0; tr.upper[0] = 0.0;
            a.keys[0] = 0.0;
            s_nodes = 1; s_expanded = 0; s_staged = 0;
        }
        __syncthreads();
    }
    const bool dist_mode = a.cfg.node_capacity > STAGE_CAP;
    if (dist_mode) {
        if (blockIdx.x == 0 && tid == 0) {
            a.dscr->gmin[0] = a.dscr->gmin[1] = ~0ull;
            ctl->n_nodes = 1;
        }
        grid_barrier(ctl, n_ctas);
    }
    int wave = 0;
    long long tp = clock64();
    auto lap = [&](int slot) {
        if (blockIdx.x == 0 && tid == 0) { const long long t1 = clock64(); ctl->prof[slot] += t1 - tp; tp = t1; }
    };
    // ------------------------------------------------------------------ waves
    while (true) {
        if (dist_mode) {
            const int nn = *(volatile int*)&ctl->n_nodes, ne = *(volatile int*)&ctl->n_expanded;
            const int k = select_dist(a, sh, skeys, nn, ne, wave, n_ctas);
            lap(1);
            if (blockIdx.x == 0) {
                int children = 0;
                if (k > 0) children = layout_wave<JOINT_IL>(a, sh, skeys, false, nn, ne, k, 0, ctl->prof);
                if (tid == 0) {
                    if (children == 0) ctl->stop = 1;
                    tp = clock64();
                }
            }
            ++wave;
        } else if (blockIdx.x == 0) {
            const int nn = s_nodes, ne = s_expanded, ns = s_staged;
            __syncthreads();
            const int children = select_wave<JOINT_IL>(a, sh, skeys, nn, ne, ns, ctl->prof);
            if (tid == 0) {
                if (children == 0) ctl->stop = 1;
                else { s_staged = nn; s_nodes = ctl->n_nodes; s_expanded = ctl->n_expanded; }
                tp = clock64();
            }
        }
        grid_barrier(ctl, n_ctas);
        lap(3);
        if (*(volatile int*)&ctl->stop) break;
        const int total = *(volatile int*)&ctl->wave_children;
        const int base = *(volatile int*)&ctl->wave_base;
        const int M = a.cfg.n_models, Mx = M > 0 ? M : 1;
        if (hwy) {
            // one (child, model) per 16-lane group; consecutive tasks go to different SMs first: a small wave
            // runs one warp per SM
            const int warp_global = (tid >> 5) * (int)n_ctas + (int)blockIdx.x;
            const int n_warps = WARPS * (int)n_ctas;
            const int n_tasks = total * Mx;
            for (int w0 = 2 * warp_global; w0 < n_tasks; w0 += 2 * n_warps) {
                const int task_raw = w0 + ((tid >> 4) & 1);
                const bool real = task_raw < n_tasks;
                const int task = real ? task_raw : w0;
                const int w = task / Mx, m = task - w * Mx;
                const int item = __ldcg(a.work + w);
                const int leaf = item & 0x0fffffff, action = real ? (item >> 28) & 7 : hw::A_IDLE;
                hw::Lane L;
                int t, si;
                load_state_cg(tr.state + ((int64_t)leaf * Mx + m) * hw::WORDS, li, L, t, si);
                bool term, trunc;
                const float r = hw::step(L, li, t, si, action, term, trunc, 0xffffffffu);
                const float ego_y = __shfl_sync(0xffffffffu, L.y, 0, 16);
                if (real) {
                    const int c = base + w;
                    hw::store_state(tr.state + ((int64_t)c * Mx + m) * hw::WORDS, li, L, t, si);
                    if (li == 0) {
                        if (M == 0) write_child(a, c, leaf, action, (double)r, term, hw::avail_mask(ego_y, si));
                        else write_model_bounds(a, task, c, leaf, m, (double)r, term, hw::avail_mask(ego_y, si));
                    }
                }
            }
        } else if (a.cfg.env_kind == B2_ENV_INTERSECTION && !JOINT_IL) {
            const int warp_global = (tid >> 5) * (int)n_ctas + (int)blockIdx.x;
            const int n_warps = WARPS * (int)n_ctas;
            for (int w0 = 2 * warp_global; w0 < total; w0 += 2 * n_warps) {
                const int w_raw = w0 + ((tid >> 4) & 1);
                const bool real = w_raw < total;
                const int w = real ? w_raw : w0;
                const int item = __ldcg(a.work + w);
                const int leaf = item & 0x0fffffff, action = real ? (item >> 28) & 7 : il::A_IDLE;
                il::Lane L;
                il::Globals g;
                il::load_state<true>(tr.state + (int64_t)leaf * il::WORDS, li, L, g);
                bool term, trunc;
                const float r = il::step(L, li, g, action, term, trunc, 0xffffffffu);
                if (real) {
                    const int c = base + w;
                    il::store_state(tr.state + (int64_t)c * il::WORDS, li, L, g);
                    if (li == 0) write_child(a, c, leaf, action, (double)r, term, il::avail_mask(g.si));
                }
            }
        } else if (JOINT_IL) {
            // joint mode: one (child, model) per 16-lane group, the model's scene at (node * M + m) * WORDS
            const int warp_global = (tid >> 5) * (int)n_ctas + (int)blockIdx.x;
            const int n_warps = WARPS * (int)n_ctas;
            const int n_tasks = total * M;
            for (int w0 = 2 * warp_global; w0 < n_tasks; w0 += 2 * n_warps) {
                const int task_raw = w0 + ((tid >> 4) & 1);
                const bool real = task_raw < n_tasks;
                const int task = real ? task_raw : w0;
                const int w = task / M, m = task - w * M;
                const int item = __ldcg(a.work + w);
                const int leaf = item & 0x0fffffff, action = real ? (item >> 28) & 7 : il::A_IDLE;
                il::Lane L;
                il::Globals g;
                il::load_state<true>(tr.state + ((int64_t)leaf * M + m) * il::WORDS, li, L, g);
                bool term, trunc;
                const float r = il::step(L, li, g, action, term, trunc, 0xffffffffu);
                if (real) {
                    const int c = base + w;
                    il::store_state(tr.state + ((int64_t)c * M + m) * il::WORDS, li, L, g);
                    if (li == 0) write_model_bounds(a, task, c, leaf, m, (double)r, term, il::avail_mask(g.si));
                }
            }
        } else if (M > 0) {
            for (int task = blockIdx.x * THREADS + tid; task < total * M; task += THREADS * (int)n_ctas) {
                const int w = task / M, m = task - w * M;
                const b2_finite_mdp& mm = a.cfg.model_mdps[m];
                const int item = __ldcg(a.work + w);
                const int leaf = item & 0x0fffffff, action = (item >> 28) & 7;
                const int s = ld_cg(tr.state + (int64_t)leaf * M + m);
                const int c = base + w;
                tr.state[(int64_t)c * M + m] = mm.transition[(int64_t)s * mm.n_actions + action];
                write_model_bounds(a, task, c, leaf, m, mm.reward[(int64_t)s * mm.n_actions + action],
                                   mm.terminal[s] != 0, 0);
            }
        } else {
            const b2_finite_mdp& m = a.cfg.mdp;
            for (int w = blockIdx.x * THREADS + tid; w < total; w += THREADS * (int)n_ctas) {
                const int item = __ldcg(a.work + w);
                const int leaf = item & 0x0fffffff, action = (item >> 28) & 7;
                const int s = ld_cg(tr.state + leaf);
                const int s2 = m.transition[(int64_t)s * m.n_actions + action];
                const int c = base + w;
                tr.state[c] = s2;
                write_child(a, c, leaf, action, m.reward[(int64_t)s * m.n_actions + action], m.terminal[s] != 0, 0);
            }
        }
        lap(4);
        if (M > 0) {        // the children's robust bounds need every model's result
            grid_barrier(ctl, n_ctas);
            finalize_joint_children(a, total, base, n_ctas);
        }
        grid_barrier(ctl, n_ctas);
        lap(5);
        if (*(volatile int*)&ctl->error) break;
    }
    if (blockIdx.x != 0) return;
    finish_tree(a, tp);
}

// ---------------------------------------------------------------------------
// Speculative strict search (b2_opd_plan_spec): the reference's one-leaf-per-iteration order
// (deterministic.py:106-114), bit for bit, without paying one dependent env transition per expansion.
//
// Per wave CTA 0 takes the K best frontier leaves in the reference's arg-max order (value_upper descending, node
// id ascending); every SM simulates the children of those that have not been simulated yet into an arena
// (a leaf is simulated at most once: the results stay cached until the leaf is expanded).  The strict search
// would expand candidate j next iff no child created by candidates 0..j-1 has a larger value_upper than j (a
// child that ties loses: it has the larger id), so CTA 0 commits the longest such prefix -- children get their
// final ids by a prefix sum, in the strict order -- and the rest stays speculative.  Candidate 0 always
// commits, so the search advances every wave; gamma < 1 makes children's bounds tighter than their parents'
// and the prefix long.
// ---------------------------------------------------------------------------
__device__ __forceinline__ int ordered_actions(const Args& a, int mask, int* acts) {
    int q = 0;
    for (int i = 0; i < MAX_BRANCH; ++i) {
        int act;
        if (a.cfg.env_kind == B2_ENV_HIGHWAY) {
            if (i >= 5) break;
            const int order[5] = {hw::A_IDLE, hw::A_LEFT, hw::A_RIGHT, hw::A_FASTER, hw::A_SLOWER};
            act = order[i];
        } else if (a.cfg.env_kind == B2_ENV_INTERSECTION) {
            if (i >= 3) break;
            const int order[3] = {il::A_IDLE, il::A_FASTER, il::A_SLOWER};
            act = order[i];
        } else {
            if (i >= a.cfg.n_actions) break;
            act = i;
        }
        if (mask & (1 << act)) acts[q++] = act;
    }
    return q;
}

struct SpecShared {
    unsigned long long key[THREADS];    // candidates in strict order
    int leaf[THREADS];
    unsigned long long wmax[WARPS];
    int first_fail;
};

__global__ void __launch_bounds__(THREADS, 1) opd_spec_kernel(Args a) {
    extern __shared__ unsigned long long skeys[];
    __shared__ SelShared sh;
    __shared__ SpecShared sp;
    __shared__ int s_nodes, s_expanded, s_slots;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, li = tid & 15;
    const unsigned n_ctas = gridDim.x;
    Control* ctl = a.ctl;
    const b2_opd_tree& tr = a.tree;
    const int kind = a.cfg.env_kind;
    static_assert(hw::WORDS == il::WORDS, "one arena stride for both scene kinds");
    const int words = kind == B2_ENV_FINITE ? 1 : hw::WORDS;
    for (int i = blockIdx.x * THREADS + tid; i < a.cfg.node_capacity; i += THREADS * (int)n_ctas) a.spec_base[i] = -1;
    if (blockIdx.x == 0) {
        int avail = 0;
        if (kind == B2_ENV_INTERSECTION) avail = il::avail_mask(a.root_state[129]);
        else if (kind == B2_ENV_HIGHWAY) avail = hw::avail_mask(__int_as_float(a.root_state[hw::V]), a.root_state[8 * hw::V + 1]);
        else avail = (1 << a.cfg.n_actions) - 1;
        for (int i = tid; i < words; i += THREADS) tr.state[i] = a.root_state[i];       // arena slot 0
        if (tid == 0) {
            tr.parent[0] = -1; tr.first_child[0] = -1; tr.depth[0] = 0; tr.count[0] = 1;
            tr.meta[0] = 0xff | (avail << 24);
            tr.reward[0] = 0.0; tr.lower[0] = 0.0; tr.upper[0] = 0.0;
            a.state_slot[0] = 0;
            skeys[0] = sortable(0.0);
            s_nodes = 1; s_expanded = 0; s_slots = 1;
        }
    }
    grid_barrier(ctl, n_ctas);
    long long tp = clock64();
    auto lap = [&](int slot) {
        if (blockIdx.x == 0 && tid == 0) { const long long t1 = clock64(); ctl->prof[slot] += t1 - tp; tp = t1; }
    };
    int k = 0;
    while (true) {
        // ---------------------------------------------------------------- candidates + transitions to simulate
        if (blockIdx.x == 0) {
            const int nn = s_nodes, ne = s_expanded, slots0 = s_slots;
            __syncthreads();
            k = select_wave(a, sh, skeys, nn, ne, nn, ctl->prof, a.cand, false);
            if (k > 0) {
                // strict order: key descending, id ascending (the candidates arrive in id order)
                long long t0 = clock64();
                int my_leaf = 0;
                unsigned long long my_key = 0;
                if (tid < k) { my_leaf = a.cand[tid]; my_key = skeys[my_leaf]; sp.key[tid] = my_key; }
                __syncthreads();
                int rank = 0;
                if (tid < k) {
                    for (int i = 0; i < k; ++i) {
                        const unsigned long long ki = sp.key[i];
                        rank += (ki > my_key || (ki == my_key && i < tid)) ? 1 : 0;
                    }
                }
                __syncthreads();
                if (tid < k) { sp.key[rank] = my_key; sp.leaf[rank] = my_leaf; }
                __syncthreads();
                int leaf = 0, n = 0, need = 0, acts[MAX_BRANCH];
                if (tid < k) {
                    leaf = sp.leaf[tid];
                    const int meta = tr.meta[leaf];
                    const int mask = kind != B2_ENV_FINITE ? (meta >> 24) & 0x1f : (1 << a.cfg.n_actions) - 1;
                    n = ordered_actions(a, mask, acts);
                    need = a.spec_base[leaf] < 0 ? n : 0;
                }
                int e1, e2, total, t2;
                block_scan2(need, 0, sh, e1, e2, total, t2);
                if (need > 0) {
                    a.spec_base[leaf] = slots0 + e1;
                    for (int q = 0; q < n; ++q) {
                        a.work[e1 + q] = leaf | (acts[q] << 28);
                        a.work_slot[e1 + q] = slots0 + e1 + q;
                    }
                }
                if (tid == 0) {
                    ctl->wave_children = total;
                    s_slots = slots0 + total;
                    ctl->prof[2] += clock64() - t0;
                }
            } else if (tid == 0) {
                ctl->stop = 1;
            }
            if (tid == 0) tp = clock64();
        }
        grid_barrier(ctl, n_ctas);
        lap(3);
        if (*(volatile int*)&ctl->stop) break;
        // ---------------------------------------------------------------- simulate (all CTAs)
        const int total = *(volatile int*)&ctl->wave_children;
        if (kind == B2_ENV_FINITE) {
            const b2_finite_mdp& m = a.cfg.mdp;
            for (int w = blockIdx.x * THREADS + tid; w < total; w += THREADS * (int)n_ctas) {
                const int item = __ldcg(a.work + w), slot = __ldcg(a.work_slot + w);
                const int leaf = item & 0x0fffffff, action = (item >> 28) & 7;
                const int s = ld_cg(tr.state + __ldcg(a.state_slot + leaf));
                const double r = m.reward[(int64_t)s * m.n_actions + action];
                tr.state[slot] = m.transition[(int64_t)s * m.n_actions + action];
                a.spec_reward[slot] = r;
                a.spec_flags[slot] = action | (m.terminal[s] != 0 ? 1 << 16 : 0) | ((r >= 0.0 && r <= 1.0) ? 0 : 1 << 17);
            }
        } else {
            const int warp_global = warp * (int)n_ctas + (int)blockIdx.x;
            const int n_warps = WARPS * (int)n_ctas;
            for (int w0 = 2 * warp_global; w0 < total; w0 += 2 * n_warps) {
                const int w_raw = w0 + ((tid >> 4) & 1);
                const bool real = w_raw < total;
                const int w = real ? w_raw : w0;
                const int item = __ldcg(a.work + w), slot = __ldcg(a.work_slot + w);
                const int leaf = item & 0x0fffffff;
                const int32_t* src = tr.state + (int64_t)__ldcg(a.state_slot + leaf) * hw::WORDS;
                int32_t* dst = tr.state + (int64_t)slot * hw::WORDS;
                bool term, trunc;
                float r;
                int avail, action;
                if (kind == B2_ENV_HIGHWAY) {
                    action = real ? (item >> 28) & 7 : hw::A_IDLE;
                    hw::Lane L;
                    int t, si;
                    load_state_cg(src, li, L, t, si);
                    r = hw::step(L, li, t, si, action, term, trunc, 0xffffffffu);
                    const float ego_y = __shfl_sync(0xffffffffu, L.y, 0, 16);
                    avail = hw::avail_mask(ego_y, si);
                    if (real) hw::store_state(dst, li, L, t, si);
                } else {
                    action = real ? (item >> 28) & 7 : il::A_IDLE;
                    il::Lane L;
                    il::Globals g;
                    il::load_state<true>(src, li, L, g);
                    r = il::step(L, li, g, action, term, trunc, 0xffffffffu);
                    avail = il::avail_mask(g.si);
                    if (real) il::store_state(dst, li, L, g);
                }
                if (real && li == 0) {
                    const double rd = (double)r;
                    a.spec_reward[slot] = rd;
                    a.spec_flags[slot] = action | (term ? 1 << 16 : 0) | ((rd >= 0.0 && rd <= 1.0) ? 0 : 1 << 17) | (avail << 24);
                }
            }
        }
        lap(4);
        grid_barrier(ctl, n_ctas);
        lap(5);
        // ---------------------------------------------------------------- commit the strict prefix (CTA 0)
        if (blockIdx.x == 0) {
            const int nn = s_nodes, ne = s_expanded;
            const int remaining = a.cfg.n_expansions - ne;
            int leaf = 0, n = 0, base = 0, d = 0, flags[MAX_BRANCH];
            double rew[MAX_BRANCH], lo[MAX_BRANCH], up[MAX_BRANCH];
            unsigned long long m = 0;                         // largest child key of this candidate
            if (tid < k) {
                leaf = sp.leaf[tid];
                base = a.spec_base[leaf];
                const int meta = tr.meta[leaf];
                n = __popc(kind != B2_ENV_FINITE ? (meta >> 24) & 0x1f : (1 << a.cfg.n_actions) - 1);
                d = tr.depth[leaf] + 1;
                const double lowl = tr.lower[leaf], gp = a.cfg.gamma_pow[d - 1], gpd = a.cfg.gamma_pow_div[d],
                             tb = a.cfg.terminal_bonus[d];
                for (int q = 0; q < MAX_BRANCH; ++q) {
                    if (q >= n) break;
                    rew[q] = __ldcg(a.spec_reward + base + q);
                    flags[q] = __ldcg(a.spec_flags + base + q);
                    double l2 = lowl + gp * rew[q];           // DeterministicNode.update (:52-63)
                    double u2 = l2 + gpd;
                    if (flags[q] & (1 << 16)) { l2 = l2 + tb; u2 = l2; }
                    lo[q] = l2; up[q] = u2;
                    const unsigned long long uk = sortable(u2);
                    m = uk > m ? uk : m;
                }
            }
            // exclusive prefix maximum of m over the strict order
            unsigned long long inc = m;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long x = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc = x > inc ? x : inc;
            }
            unsigned long long exc = __shfl_up_sync(0xffffffffu, inc, 1);
            if (lane == 0) exc = 0;
            if (lane == 31) sp.wmax[warp] = inc;
            if (tid == 0) sp.first_fail = k;
            __syncthreads();
            for (int i = 0; i < warp; ++i) exc = sp.wmax[i] > exc ? sp.wmax[i] : exc;
            if (tid < k && exc > sp.key[tid]) atomicMin(&sp.first_fail, tid);
            __syncthreads();
            const int n_commit = min(sp.first_fail, remaining);
            const bool mine = tid < n_commit;
            int ec, e2, total_c, t2;
            block_scan2(mine ? n : 0, 0, sh, ec, e2, total_c, t2);
            int term = 0;
            if (mine) {
                const int c0 = nn + ec;
                const int meta = tr.meta[leaf];
                tr.first_child[leaf] = c0;
                tr.meta[leaf] = meta | (n << 8);
                skeys[leaf] = ABSENT;
                a.exp_order[ne + tid] = leaf;
                term = (meta >> 16) & 1;
                for (int q = 0; q < MAX_BRANCH; ++q) {
                    if (q >= n) break;
                    const int c = c0 + q;
                    tr.parent[c] = leaf;
                    tr.first_child[c] = -1;
                    tr.depth[c] = d;
                    tr.count[c] = 2;
                    tr.meta[c] = flags[q] & ~(1 << 17);
                    tr.reward[c] = rew[q];
                    tr.lower[c] = lo[q];
                    tr.upper[c] = up[q];
                    a.state_slot[c] = base + q;
                    skeys[c] = sortable(up[q]);
                    if (flags[q] & (1 << 17)) ctl->error = 1;          // :46-47
                }
                atomicMax(&ctl->max_depth, d);
            }
            term = block_sum(term, sh.red, 0);
            if (tid == 0) {
                ctl->term_exp += term;
                a.wave_start[ctl->n_waves] = ne;
                ctl->n_waves += 1;
                a.wave_start[ctl->n_waves] = ne + n_commit;
                ctl->n_nodes = nn + total_c;
                ctl->n_expanded = ne + n_commit;
                s_nodes = nn + total_c;
                s_expanded = ne + n_commit;
            }
            __syncthreads();
            lap(0);
            if (ctl->error) {
                if (tid == 0) ctl->stop = 1;
            }
        }
    }
    if (blockIdx.x != 0) return;
    finish_tree(a, tp);
}


static int64_t align_up(int64_t x) { return (x + 255) & ~(int64_t)255; }

struct Layout {
    int64_t ctl, keys, exp_order, wave_start, work, lowerv, wave_up, wave_flags, dscr, cta_cnt, total;
};

struct SpecLayout {
    int64_t ctl, exp_order, wave_start, work, work_slot, cand, spec_base, state_slot, spec_reward, spec_flags, total;
};

static int64_t spec_arena_slots(const b2_opd_wave_config* c) { return 1 + (int64_t)c->node_capacity * c->n_actions; }

static SpecLayout make_spec_layout(const b2_opd_wave_config* c) {
    SpecLayout l;
    const int64_t wa = (int64_t)c->width * c->n_actions, slots = spec_arena_slots(c);
    l.ctl = 0;
    l.exp_order = align_up(sizeof(Control));
    l.wave_start = l.exp_order + align_up((int64_t)c->n_expansions * 4 + 4);
    l.work = l.wave_start + align_up(((int64_t)c->n_expansions + 2) * 4);
    l.work_slot = l.work + align_up(wa * 4 + 4);
    l.cand = l.work_slot + align_up(wa * 4 + 4);
    l.spec_base = l.cand + align_up((int64_t)c->width * 4 + 4);
    l.state_slot = l.spec_base + align_up((int64_t)c->node_capacity * 4);
    l.spec_reward = l.state_slot + align_up((int64_t)c->node_capacity * 4);
    l.spec_flags = l.spec_reward + align_up(slots * 8);
    l.total = l.spec_flags + align_up(slots * 4);
    return l;
}

static Layout make_layout(const b2_opd_wave_config* c) {
    Layout l;
    l.ctl = 0;
    l.keys = align_up(sizeof(Control));
    l.exp_order = l.keys + align_up((int64_t)c->node_capacity * 8);
    l.wave_start = l.exp_order + align_up((int64_t)c->n_expansions * 4 + 4);
    l.work = l.wave_start + align_up(((int64_t)c->n_expansions + 2) * 4);
    const int64_t M = c->n_models > 0 ? c->n_models : 0;
    l.lowerv = l.work + align_up((int64_t)c->width * c->n_actions * 4 + 4);
    l.wave_up = l.lowerv + align_up((int64_t)c->node_capacity * M * 8);
    l.wave_flags = l.wave_up + align_up((int64_t)c->width * c->n_actions * M * 8);
    l.dscr = l.wave_flags + align_up((int64_t)c->width * c->n_actions * M * 4);
    l.cta_cnt = l.dscr + align_up(sizeof(DistScratch));
    l.total = l.cta_cnt + align_up(1024 * sizeof(int2));
    return l;
}

}  // namespace wave
}  // namespace b2

using namespace b2;

extern "C" int64_t b2_opd_wave_workspace_bytes(const b2_opd_wave_config* cfg) {
    if (!cfg || cfg->n_expansions < 0 || cfg->width <= 0 || cfg->n_actions <= 0) return -1;
    return wave::make_layout(cfg).total;
}

extern "C" int b2_opd_plan_wave(const b2_opd_wave_config* cfg, const int32_t* root_state, const b2_opd_tree* tree,
                                void* workspace, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_state && tree && workspace && plan && result, "null pointer");
    B2_REQUIRE(cfg->n_expansions >= 0 && cfg->width > 0, "bad budget / wave width");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions <= wave::MAX_BRANCH, "n_actions must be in 1..8");
    B2_REQUIRE((int64_t)cfg->node_capacity >= 1 + (int64_t)cfg->n_expansions * cfg->n_actions, "node_capacity too small");
    B2_REQUIRE(cfg->node_capacity < (1 << 28), "node_capacity must be < 2^28");
    B2_REQUIRE(cfg->plan_capacity >= 1, "plan_capacity too small");
    B2_REQUIRE(cfg->gamma_pow && cfg->gamma_pow_div && cfg->terminal_bonus, "gamma tables missing");
    B2_REQUIRE(cfg->n_models >= 0 && cfg->n_models <= B2_MAX_MODELS, "n_models must be in 0..8");
    if (cfg->env_kind == B2_ENV_FINITE && cfg->n_models > 0) {
        for (int m = 0; m < cfg->n_models; ++m) {
            const b2_finite_mdp& mm = cfg->model_mdps[m];
            B2_REQUIRE(mm.transition && mm.reward && mm.terminal && mm.n_actions == cfg->n_actions, "model MDP tables missing");
        }
    } else if (cfg->env_kind == B2_ENV_FINITE) {
        B2_REQUIRE(cfg->mdp.transition && cfg->mdp.reward && cfg->mdp.terminal, "finite MDP tables missing");
        B2_REQUIRE(cfg->mdp.n_actions == cfg->n_actions, "mdp.n_actions != n_actions");
    } else if (cfg->env_kind == B2_ENV_HIGHWAY) {
        B2_REQUIRE(cfg->n_actions == B2_HW_ACTIONS, "HighwayLite has 5 actions");
    } else if (cfg->env_kind == B2_ENV_INTERSECTION) {
        B2_REQUIRE(cfg->n_actions == B2_IL_ACTIONS, "IntersectionLite has 3 actions");
    } else {
        set_error("unknown env_kind %d", cfg->env_kind);
        return B2_ERR_INVALID;
    }
    cudaStream_t stream = (cudaStream_t)stream_;
    const wave::Layout l = wave::make_layout(cfg);
    char* ws = (char*)workspace;
    wave::Args a;
    a.cfg = *cfg; a.tree = *tree; a.root_state = root_state;
    a.ctl = (wave::Control*)(ws + l.ctl);
    a.keys = (double*)(ws + l.keys);
    a.exp_order = (int32_t*)(ws + l.exp_order);
    a.wave_start = (int32_t*)(ws + l.wave_start);
    a.work = (int32_t*)(ws + l.work);
    a.lowerv = (double*)(ws + l.lowerv);
    a.wave_up = (double*)(ws + l.wave_up);
    a.wave_flags = (int32_t*)(ws + l.wave_flags);
    a.dscr = (wave::DistScratch*)(ws + l.dscr);
    a.cta_cnt = (int2*)(ws + l.cta_cnt);
    a.plan = plan; a.result = result;
    B2_CUDA_CHECK(cudaMemsetAsync(a.ctl, 0, sizeof(wave::Control), stream));
    B2_CUDA_CHECK(cudaMemsetAsync(a.dscr, 0, sizeof(wave::DistScratch), stream));
    const int stage = cfg->node_capacity < wave::STAGE_CAP ? cfg->node_capacity : wave::STAGE_CAP;
    const size_t smem = (size_t)stage * 8;
    const void* kernel = cfg->env_kind == B2_ENV_INTERSECTION && cfg->n_models > 0 ? (const void*)wave::opd_wave_kernel<true>
                                                                                    : (const void*)wave::opd_wave_kernel<false>;
    B2_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B2_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, wave::THREADS, smem));
    B2_REQUIRE(per_sm >= 1, "wave kernel does not fit on an SM");
    // one CTA per SM; a wave of w children keeps ceil(w / 16) CTAs busy, the others only pass the barriers
    int grid = sm_count();
    if (cfg->max_ctas > 0 && cfg->max_ctas < grid) grid = cfg->max_ctas;
    if (grid > wave::THREADS) grid = wave::THREADS;      // the distributed selection scans the CTA table with one block
    void* params[] = {&a};
    B2_CUDA_CHECK(cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(wave::THREADS), params,
                                              smem, stream));
    return B2_OK;
}

static bool spec_config_ok(const b2_opd_wave_config* cfg) {
    return cfg && cfg->n_expansions >= 0 && cfg->width > 0 && cfg->width <= wave::THREADS && cfg->n_actions > 0 &&
           cfg->n_actions <= wave::MAX_BRANCH && cfg->n_models == 0 && cfg->node_capacity <= wave::STAGE_CAP &&
           (int64_t)cfg->node_capacity >= 1 + (int64_t)cfg->n_expansions * cfg->n_actions;
}

extern "C" int64_t b2_opd_spec_workspace_bytes(const b2_opd_wave_config* cfg) {
    if (!spec_config_ok(cfg)) return -1;
    return wave::make_spec_layout(cfg).total;
}

extern "C" int64_t b2_opd_spec_arena_slots(const b2_opd_wave_config* cfg) {
    if (!spec_config_ok(cfg)) return -1;
    return wave::spec_arena_slots(cfg);
}

extern "C" int b2_opd_plan_spec(const b2_opd_wave_config* cfg, const int32_t* root_state, const b2_opd_tree* tree,
                                void* workspace, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_state && tree && workspace && plan && result, "null pointer");
    B2_REQUIRE(spec_config_ok(cfg),
               "speculative search: width in 1..256, n_actions in 1..8, n_models = 0, node_capacity in "
               "[1 + n_expansions * n_actions, 24576]");
    B2_REQUIRE(cfg->plan_capacity >= 1, "plan_capacity too small");
    B2_REQUIRE(cfg->gamma_pow && cfg->gamma_pow_div && cfg->terminal_bonus, "gamma tables missing");
    if (cfg->env_kind == B2_ENV_FINITE) {
        B2_REQUIRE(cfg->mdp.transition && cfg->mdp.reward && cfg->mdp.terminal, "finite MDP tables missing");
        B2_REQUIRE(cfg->mdp.n_actions == cfg->n_actions, "mdp.n_actions != n_actions");
    } else if (cfg->env_kind == B2_ENV_HIGHWAY) {
        B2_REQUIRE(cfg->n_actions == B2_HW_ACTIONS, "HighwayLite has 5 actions");
    } else if (cfg->env_kind == B2_ENV_INTERSECTION) {
        B2_REQUIRE(cfg->n_actions == B2_IL_ACTIONS, "IntersectionLite has 3 actions");
    } else {
        set_error("unknown env_kind %d", cfg->env_kind);
        return B2_ERR_INVALID;
    }
    cudaStream_t stream = (cudaStream_t)stream_;
    const wave::SpecLayout l = wave::make_spec_layout(cfg);
    char* ws = (char*)workspace;
    wave::Args a;
    memset(&a, 0, sizeof(a));
    a.cfg = *cfg; a.tree = *tree; a.root_state = root_state;
    a.ctl = (wave::Control*)(ws + l.ctl);
    a.exp_order = (int32_t*)(ws + l.exp_order);
    a.wave_start = (int32_t*)(ws + l.wave_start);
    a.work = (int32_t*)(ws + l.work);
    a.work_slot = (int32_t*)(ws + l.work_slot);
    a.cand = (int32_t*)(ws + l.cand);
    a.spec_base = (int32_t*)(ws + l.spec_base);
    a.state_slot = (int32_t*)(ws + l.state_slot);
    a.spec_reward = (double*)(ws + l.spec_reward);
    a.spec_flags = (int32_t*)(ws + l.spec_flags);
    a.plan = plan; a.result = result;
    B2_CUDA_CHECK(cudaMemsetAsync(a.ctl, 0, sizeof(wave::Control), stream));
    const size_t smem = (size_t)cfg->node_capacity * 8;
    B2_CUDA_CHECK(cudaFuncSetAttribute(wave::opd_spec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    B2_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wave::opd_spec_kernel, wave::THREADS, smem));
    B2_REQUIRE(per_sm >= 1, "speculative kernel does not fit on an SM");
    int grid = sm_count();
    if (cfg->max_ctas > 0 && cfg->max_ctas < grid) grid = cfg->max_ctas;
    void* params[] = {&a};
    B2_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)wave::opd_spec_kernel, dim3(grid), dim3(wave::THREADS), params,
                                              smem, stream));
    return B2_OK;
}

// ---------------------------------------------------------------------------
// batched IntersectionLite transition (b2_intersection_step): one scene per 16-lane group
// ---------------------------------------------------------------------------
namespace b2 {
__global__ void __launch_bounds__(128) intersection_step_kernel(int32_t* states, const int32_t* actions, float* reward,
                                                                int32_t* flags, int32_t* avail, int n_envs) {
    const int gidx = (blockIdx.x * 128 + threadIdx.x) >> 4, li = threadIdx.x & 15;
    const bool live = gidx < n_envs;
    const int e = live ? gidx : n_envs - 1;
    il::Lane L;
    il::Globals g;
    il::load_state<false>(states + (int64_t)e * il::WORDS, li, L, g);
    bool term, trunc;
    const float r = il::step(L, li, g, actions[e], term, trunc, 0xffffffffu);
    if (live) {
        il::store_state(states + (int64_t)e * il::WORDS, li, L, g);
        if (li == 0) {
            reward[e] = r;
            flags[e] = (term ? 1 : 0) | (trunc ? 2 : 0);
            if (avail) avail[e] = il::avail_mask(g.si);
        }
    }
}
}  // namespace b2

extern "C" int b2_intersection_step(int32_t* states, const int32_t* actions, float* reward, int32_t* flags,
                                    int32_t* avail_mask, int32_t n_envs, void* stream) {
    B2_REQUIRE(states && actions && reward && flags && n_envs > 0, "null pointer / empty batch");
    const int grid = (n_envs + 7) / 8;
    b2::intersection_step_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(states, actions, reward, flags, avail_mask, n_envs);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
