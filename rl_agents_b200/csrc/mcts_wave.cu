// Wavefront MCTS: ONE decision searched by the whole GPU (b2_mcts_plan_wave).
//
// The reference's MCTS.plan (mcts.py:179-184) runs its episodes one after the other on one sequential RNG
// stream: 4096 episodes x horizon 20 is a chain of 81 920 dependent env transitions.  The
// wavefront keeps the reference's episode -- selection (:141-149), expansion (:151-154), rollout (:160-177),
// backup (:257-265), recommendation (:212-218) -- and runs the episodes in waves of `width`:
//   select (CTA 0)   all selections of the wave, level by level.  A node's arrivals are a contiguous, episode-
//                    ordered segment; one thread per segment walks its arrivals in order, scoring the children
//                    with value + T*n*prior/(count + virtual + 1) where `virtual` counts the wave's earlier
//                    arrivals routed to that child, so the wave spreads over the tree; the children's segments
//                    are the stable partition of the parent's segment.  A childless node is expanded by the
//                    first episode that reached it; ties are broken by a counter-based generator.
//   simulate (all)   one 16-lane group per episode: root scene -> selected path -> (expansion) -> random
//                    rollout to the horizon; then count += 1, value_sum += return along the path with integer
//                    atomics on a 2^-40 fixed-point sum (order independent, exact).
// Specification: oracle/planners.py::mcts_plan_wavefront (bit-identical: node ids, counts, value sums).
//
// b2_mcts_plan_wave_sampled runs a finite MDP in any mode (mcts_wave_kernel<true>).  Every episode's env is a deep
// copy of the same live env, generator included, so step h of every episode draws the same double u[h] of that
// generator's stream: each CTA computes the horizon's doubles once and a step is searchsorted(cdf[row], u[h]).  The
// lowest episode that reaches a row Generator.choice rejects is reported (that episode backs nothing up), and the
// search stops after its wave.
#include "common.cuh"
#include "highway_lite.cuh"
#include "lane_env.cuh"
#include "pcg64.cuh"

namespace b2 {
namespace mwave {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int MAX_WIDTH = 1024;
constexpr int MAX_A = 8;
constexpr int MAX_H = 64;
constexpr double FIX_SCALE = 1099511627776.0;   // 2^40

struct Control {
    unsigned bar_count, bar_gen;
    int env_steps, pad;
    long long prof[4];       // CTA 0 clock64 totals: 0 select, 1 barrier, 2 simulate, 3 barrier
    unsigned long long rejected;   // sampled: max of ~(episode << 32 | row) over the rejected rows reached; 0 none
};

struct Args {
    b2_mcts_wave_config cfg;
    b2_mcts_wave_tree tree;
    const int32_t* root_state;
    Control* ctl;
    int32_t* paths;          // [width, horizon] node reached at depth h+1
    int32_t* plen;           // [width] selection depth
    int32_t* expands;        // [width] 1: this episode creates the children of its leaf
    double* recip;           // [episodes + width + 2] 1.0 / k (filled at kernel start)
    int8_t* plan;
    int32_t* result;
    // mcts_wave_kernel<true> only
    b2_finite_mdp_sampled smdp;
    const uint8_t* terminal;
    int32_t env_draws;
    const uint64_t* env_rng;
    int32_t* rejected;       // [2] episode, row
};

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
    unsigned long long z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ int wave_random(unsigned long long seed, int episode, int step, int stream, int n) {
    const unsigned long long key = seed + (unsigned long long)episode * 0x9E3779B97F4A7C15ull +
                                   (unsigned long long)(step + 1) * 0xD1B54A32D192ED03ull +
                                   (unsigned long long)stream * 0x8CB92BA72F3D8DD7ull;
    return (int)((unsigned)(splitmix64(key) >> 33) % (unsigned)n);    // 31-bit value: a 32-bit modulo gives the same result
}

// order-preserving image of a finite double as a signed 64-bit integer (+0 and -0 coincide)
__device__ __forceinline__ long long score_key(double x) {
    const long long b = __double_as_longlong(x + 0.0);
    return b >= 0 ? b : (long long)(0x8000000000000000ull - (unsigned long long)b);
}

constexpr int BIG_MIN = 16;                 // arrivals from which a segment gets a precomputed score table
constexpr int MAX_BIG = MAX_WIDTH / BIG_MIN;
constexpr int TABLE_KEYS = 6144;            // 48 KB of dynamic shared memory

struct SelShared {
    unsigned short order[2][MAX_WIDTH];
    unsigned char pick[MAX_WIDTH];
    int seg_node[2][MAX_WIDTH];
    unsigned short seg_start[2][MAX_WIDTH], seg_len[2][MAX_WIDTH];
    int nseg[2];
    int n_big, tab_used;
    int big_seg[MAX_BIG], big_off[MAX_BIG], big_fc[MAX_BIG];
    unsigned char big_n[MAX_BIG];
    double big_val[MAX_BIG][MAX_A];
    int big_cnt[MAX_BIG][MAX_A];
};

// One segment's arrivals, in episode order: pick the best child by (score, counter-based tie-break), bump its
// virtual count, record the path; then split the segment into the children's segments (stable partition).
// `key_of(c, k)` is the order-preserving image of child c's score after k virtual visits.
template <bool RUNS, typename KeyOf>
__device__ __forceinline__ void route_segment(const Args& a, SelShared& sh, int cur, int nxt, int w0, int d, int start,
                                              int m, int fc, int n, KeyOf key_of) {
    const int H = a.cfg.horizon;
    long long key[MAX_A];
    int vc[MAX_A];
#pragma unroll
    for (int c = 0; c < MAX_A; ++c) {
        vc[c] = 0;
        key[c] = c < n ? key_of(c, 0) : (long long)0x8000000000000000ull;      // below every real score
    }
    for (int i = 0; i < m;) {
        long long best = key[0];
#pragma unroll
        for (int c = 1; c < MAX_A; ++c) best = key[c] > best ? key[c] : best;
        int ties = 0;
        long long second = (long long)0x8000000000000000ull;                    // best key among the others
#pragma unroll
        for (int c = 0; c < MAX_A; ++c) {
            ties += key[c] == best ? 1 : 0;
            second = (key[c] != best && key[c] > second) ? key[c] : second;
        }
        int sel = 0, run = 1;
        if (ties > 1) {
            int pick = wave_random(a.cfg.seed, w0 + sh.order[cur][start + i], d, 0, ties);
#pragma unroll
            for (int c = 0; c < MAX_A; ++c) {
                if (key[c] == best) {
                    if (pick == 0) sel = c;
                    --pick;
                }
            }
        } else {
#pragma unroll
            for (int c = 0; c < MAX_A; ++c) sel = key[c] == best ? c : sel;
            if (RUNS) {
                // a child's score only falls as its virtual count grows: the unique best child keeps winning
                // until its score reaches the runner-up's -- binary search for that point in its score row
                int base = 0;
#pragma unroll
                for (int c = 0; c < MAX_A; ++c) base = c == sel ? vc[c] : base;
                int lo = 1, hi = m - i;                     // the run is in [lo, hi]
                while (lo < hi) {
                    const int mid = (lo + hi + 1) >> 1;     // can the run be `mid` long?  (pick mid-1 still wins)
                    if (key_of(sel, base + mid - 1) > second) lo = mid; else hi = mid - 1;
                }
                run = lo;
            }
        }
        for (int q = 0; q < run; ++q) {
            const int j = sh.order[cur][start + i + q];
            sh.pick[start + i + q] = (unsigned char)sel;
            a.paths[(int64_t)j * H + d] = fc + sel;
        }
#pragma unroll
        for (int c = 0; c < MAX_A; ++c) {
            if (c == sel) {
                vc[c] += run;
                key[c] = key_of(c, vc[c]);
            }
        }
        i += run;
    }
    int cstart[MAX_A];
    int run = start;
#pragma unroll
    for (int c = 0; c < MAX_A; ++c) {
        cstart[c] = run;
        if (c < n && vc[c] > 0) {
            const int q = atomicAdd(&sh.nseg[nxt], 1);
            sh.seg_node[nxt][q] = fc + c;
            sh.seg_start[nxt][q] = (unsigned short)run;
            sh.seg_len[nxt][q] = (unsigned short)vc[c];
        }
        run += c < n ? vc[c] : 0;
    }
    for (int i = 0; i < m; ++i) {
        const int sel = sh.pick[start + i];
#pragma unroll
        for (int c = 0; c < MAX_A; ++c)
            if (c == sel) sh.order[nxt][cstart[c]++] = sh.order[cur][start + i];
    }
}

// CTA 0: the selections of the episodes [w0, w0 + nw) -> paths / plen / expands
__device__ void select_wave(const Args& a, SelShared& sh, long long* table, int w0, int nw) {
    const int tid = threadIdx.x;
    const b2_mcts_wave_tree& tr = a.tree;
    const int H = a.cfg.horizon;
    const double T = a.cfg.temperature;
    for (int j = tid; j < nw; j += THREADS) sh.order[0][j] = (unsigned short)j;
    if (tid == 0) {
        sh.seg_node[0][0] = 0; sh.seg_start[0][0] = 0; sh.seg_len[0][0] = (unsigned short)nw;
        sh.nseg[0] = 1; sh.nseg[1] = 0;
        sh.n_big = 0; sh.tab_used = 0;
    }
    __syncthreads();
    int cur = 0;
    for (int d = 0; d <= H; ++d) {
        const int nseg = sh.nseg[cur];
        if (nseg == 0) break;
        const int nxt = cur ^ 1;
#ifdef B2_MWAVE_DEBUG
        const long long dbg_t0 = clock64();
#endif
        // ---- A: one thread per segment.  Small segments are routed right here (scores computed on the fly);
        //         segments with many arrivals register for a precomputed score table ----
        for (int s = tid; s < nseg; s += THREADS) {
            const int node = sh.seg_node[cur][s], start = sh.seg_start[cur][s], m = sh.seg_len[cur][s];
            const int fc = d < H ? __ldcg(tr.first_child + node) : -1;
            if (fc < 0) {
                // the wave's arrivals stop here: the first one expands the node (if below the horizon)
                for (int i = 0; i < m; ++i) {
                    const int j = sh.order[cur][start + i];
                    a.plen[j] = d;
                    a.expands[j] = (i == 0 && d < H) ? 1 : 0;
                }
                continue;
            }
            const int n = (__ldcg(tr.meta + node) >> 8) & 0xff;
            double val[MAX_A];
            int cnt[MAX_A];
#pragma unroll
            for (int c = 0; c < MAX_A; ++c) {
                val[c] = 0.0; cnt[c] = 0;
                if (c < n) {
                    cnt[c] = __ldcg(tr.count + fc + c);
                    const long long vs = __ldcg(tr.vsum + fc + c);
                    val[c] = cnt[c] > 0 ? ((double)vs / FIX_SCALE) / (double)cnt[c] : 0.0;
                }
            }
            int b = -1, off = 0;
            if (m >= BIG_MIN) {
                off = atomicAdd(&sh.tab_used, n * (m + 1));
                if (off + n * (m + 1) <= TABLE_KEYS) b = atomicAdd(&sh.n_big, 1);
            }
            if (b >= 0) {
                sh.big_seg[b] = s; sh.big_off[b] = off; sh.big_fc[b] = fc; sh.big_n[b] = (unsigned char)n;
#pragma unroll
                for (int c = 0; c < MAX_A; ++c) { sh.big_val[b][c] = val[c]; sh.big_cnt[b][c] = cnt[c]; }
                continue;
            }
            const double tnp = T * (double)n * (1.0 / (double)n);
            route_segment<false>(a, sh, cur, nxt, w0, d, start, m, fc, n, [&](int c, int k) {
                double v = 0.0;
                int base = 0;
#pragma unroll
                for (int q = 0; q < MAX_A; ++q)
                    if (q == c) { v = val[q]; base = cnt[q]; }
                return score_key(v + tnp * a.recip[base + k + 1]);
            });
        }
        __syncthreads();
        // ---- B: the score tables of the big segments, filled by the whole CTA: child c after k virtual visits ----
        const int n_big = sh.n_big;
        for (int b = 0; b < n_big; ++b) {
            const int s = sh.big_seg[b], m = sh.seg_len[cur][s], n = sh.big_n[b], off = sh.big_off[b];
            const double tnp = T * (double)n * (1.0 / (double)n);
            for (int idx = tid; idx < n * (m + 1); idx += THREADS) {
                const int c = idx / (m + 1), k = idx - c * (m + 1);
                table[off + idx] = score_key(sh.big_val[b][c] + tnp * a.recip[sh.big_cnt[b][c] + k + 1]);
            }
        }
        __syncthreads();
        // ---- C: one thread per big segment walks its arrivals with table look-ups only ----
        if (tid < n_big) {
            const int s = sh.big_seg[tid], start = sh.seg_start[cur][s], m = sh.seg_len[cur][s];
            const long long* tab = table + sh.big_off[tid];
            route_segment<true>(a, sh, cur, nxt, w0, d, start, m, sh.big_fc[tid], sh.big_n[tid],
                          [&](int c, int k) { return tab[c * (m + 1) + k]; });
        }
        __syncthreads();
#ifdef B2_MWAVE_DEBUG
        if (tid == 0 && w0 == 8 * a.cfg.width) printf("level %d nseg %d big %d cycles %lld\n", d, nseg, n_big, clock64() - dbg_t0);
#endif
        if (tid == 0) { sh.nseg[cur] = 0; sh.n_big = 0; sh.tab_used = 0; }
        cur = nxt;
        __syncthreads();
    }
}

__device__ __forceinline__ void backup(const Args& a, int j, int reached, double total, int li, int lanes, unsigned gmask) {
    const b2_mcts_wave_tree& tr = a.tree;
    const long long fixed = __double2ll_rn(total * FIX_SCALE);
    for (int q = li; q <= reached; q += lanes) {
        const int node = q == 0 ? 0 : a.paths[(int64_t)j * a.cfg.horizon + q - 1];
        atomicAdd(tr.count + node, 1);
        atomicAdd(reinterpret_cast<unsigned long long*>(tr.vsum + node), (unsigned long long)fixed);
    }
}

// FiniteMDPEnv.step of a sampled table at step h of an episode (u: the env stream's doubles); false with `row` set
// when the row is one Generator.choice rejects
__device__ __forceinline__ bool sampled_step(const Args& a, const double* u, int h, int& s, int action, double& r,
                                             bool& term, int& row) {
    const b2_finite_mdp_sampled& m = a.smdp;
    const int64_t rw = (int64_t)s * m.n_actions + action;
    if (a.env_draws && !m.row_ok[rw]) { row = (int)rw; return false; }
    term = a.terminal[s] != 0;
    r = m.reward[rw];
    const int B = m.n_next;
    const int k = a.env_draws ? searchsorted_right(m.cdf + rw * B, B, u[h]) : 0;
    s = m.next[rw * B + k];
    return true;
}

template <bool SAMPLED>
__global__ void __launch_bounds__(THREADS, 1) mcts_wave_kernel(Args a) {
    extern __shared__ long long score_table[];
    __shared__ SelShared sh;
    const int tid = threadIdx.x, lane = tid & 31, li = tid & 15;
    const unsigned n_ctas = gridDim.x;
    Control* ctl = a.ctl;
    const b2_mcts_wave_tree& tr = a.tree;
    const bool hwy = !SAMPLED && a.cfg.env_kind == B2_ENV_HIGHWAY;
    const double* env_u = nullptr;
    if constexpr (SAMPLED) {
        // the env copies' common stream: step h of every episode draws env_u[h]
        __shared__ double u_sh[MAX_H];
        if (tid == 0 && a.env_draws) {
            Pcg64 g;
            g.load(a.env_rng);
            for (int h = 0; h < a.cfg.horizon; ++h) u_sh[h] = g.random();
        }
        env_u = u_sh;
    }
    const int A = a.cfg.n_actions, H = a.cfg.horizon, E = a.cfg.episodes, W = a.cfg.width;
    // node arrays: root + unused marks (parent -2); every CTA clears a slice
    for (int i = blockIdx.x * THREADS + tid; i < a.cfg.node_capacity; i += THREADS * (int)n_ctas) {
        tr.parent[i] = i == 0 ? -1 : -2;
        tr.first_child[i] = -1;
        tr.count[i] = 0;
        tr.meta[i] = 0xff;
        tr.vsum[i] = 0;
    }
    for (int i = blockIdx.x * THREADS + tid; i < E + W + 2; i += THREADS * (int)n_ctas) a.recip[i] = 1.0 / (double)i;
    grid_barrier(ctl, n_ctas);
    long long tp = clock64();
    auto lap = [&](int slot) {
        if (blockIdx.x == 0 && tid == 0) { const long long t1 = clock64(); ctl->prof[slot] += t1 - tp; tp = t1; }
    };
    int env_steps = 0;
    for (int w0 = 0; w0 < E; w0 += W) {
        const int nw = min(W, E - w0);
        if (blockIdx.x == 0) select_wave(a, sh, score_table, w0, nw);
        lap(0);
        grid_barrier(ctl, n_ctas);
        lap(1);
        if (hwy) {
            // one episode per 16-lane group; a small wave gives every episode a warp of its own (the two halves
            // mirror each other: no divergence between two different episodes inside a warp)
            const int n_warps = WARPS * (int)n_ctas;
            const int per_warp = nw > n_warps ? 2 : 1;
            const int half = (tid >> 4) & 1;
            const unsigned gmask = 0xFFFFu << (lane & 16);
            const int warp_global = (tid >> 5) * (int)n_ctas + (int)blockIdx.x;
            for (int j0 = warp_global * per_warp; j0 < nw; j0 += n_warps * per_warp) {
                const int j = per_warp == 2 ? j0 + half : j0;
                const bool real = j < nw, writer = real && (per_warp == 2 || half == 0);
                const int jj = real ? j : j0;
                const int e = w0 + jj;
                const int depth = __ldcg(a.plen + jj);
                hw::Lane L;
                int t, si;
                hw::load_state(a.root_state, li, L, t, si);
                double total = 0.0;
                bool terminal = false;
                int reached = 0, steps = 0;
                for (int h = 0; h < depth; ++h) {                               // mcts.py:141-149
                    const int node = __ldcg(a.paths + (int64_t)jj * H + h);
                    const int action = __ldcg(tr.meta + node) & 0xff;
                    bool term, trunc;
                    const float r = hw::step(L, li, t, si, action, term, trunc, gmask);
                    ++steps;
                    total += a.cfg.gamma_pow[h] * (double)r;
                    reached = h + 1;
                    if (term) { terminal = true; break; }
                }
                if (!terminal) {
                    if (depth < H && __ldcg(a.expands + jj)) {                  // expansion (:151-154, :237-246)
                        const float ego_y = __shfl_sync(gmask, L.y, 0, 16);
                        const int mask = hw::avail_mask(ego_y, si);
                        const int n = __popc(mask);
                        const int leaf = depth > 0 ? __ldcg(a.paths + (int64_t)jj * H + depth - 1) : 0;
                        const int base = 1 + e * A;
                        if (writer && li < n) {
                            tr.parent[base + li] = leaf;
                            tr.meta[base + li] = hw::nth_action(mask, li);
                        }
                        if (writer && li == 0) {
                            tr.first_child[leaf] = base;
                            tr.meta[leaf] = (__ldcg(tr.meta + leaf) & 0xff) | (n << 8);
                        }
                    }
                    for (int h = depth; h < H; ++h) {                           // evaluate (:160-177)
                        const float ego_y = __shfl_sync(gmask, L.y, 0, 16);
                        const int mask = hw::avail_mask(ego_y, si);
                        const int action = hw::nth_action(mask, wave_random(a.cfg.seed, e, h, 1, __popc(mask)));
                        bool term, trunc;
                        const float r = hw::step(L, li, t, si, action, term, trunc, gmask);
                        ++steps;
                        total += a.cfg.gamma_pow[h] * (double)r;
                        if (term || trunc) break;
                    }
                }
                if (writer) {
                    backup(a, jj, reached, total, li, 16, gmask);               // update_branch (:257-265)
                    env_steps += steps;                                         // mirror halves do not count
                }
            }
        } else {
            const b2_finite_mdp& m = a.cfg.mdp;
            for (int j = blockIdx.x * THREADS + tid; j < nw; j += THREADS * (int)n_ctas) {
                const int e = w0 + j;
                const int depth = __ldcg(a.plen + j);
                int s = a.root_state[0];
                double total = 0.0;
                bool terminal = false;
                int reached = 0, bad_row = -1;
                for (int h = 0; h < depth; ++h) {
                    const int node = __ldcg(a.paths + (int64_t)j * H + h);
                    const int action = __ldcg(tr.meta + node) & 0xff;
                    double r;
                    bool term;
                    if constexpr (SAMPLED) {
                        if (!sampled_step(a, env_u, h, s, action, r, term, bad_row)) break;
                    } else {
                        r = m.reward[(int64_t)s * m.n_actions + action];
                        term = m.terminal[s] != 0;
                        s = m.transition[(int64_t)s * m.n_actions + action];
                    }
                    ++env_steps;
                    total += a.cfg.gamma_pow[h] * r;
                    reached = h + 1;
                    if (term) { terminal = true; break; }
                }
                if (!terminal && bad_row < 0) {
                    if (depth < H && __ldcg(a.expands + j)) {
                        const int leaf = depth > 0 ? __ldcg(a.paths + (int64_t)j * H + depth - 1) : 0;
                        const int base = 1 + e * A;
                        for (int i = 0; i < A; ++i) { tr.parent[base + i] = leaf; tr.meta[base + i] = i; }
                        tr.first_child[leaf] = base;
                        tr.meta[leaf] = (__ldcg(tr.meta + leaf) & 0xff) | (A << 8);
                    }
                    for (int h = depth; h < H; ++h) {
                        const int action = wave_random(a.cfg.seed, e, h, 1, A);
                        double r;
                        bool term;
                        if constexpr (SAMPLED) {
                            if (!sampled_step(a, env_u, h, s, action, r, term, bad_row)) break;
                        } else {
                            r = m.reward[(int64_t)s * m.n_actions + action];
                            term = m.terminal[s] != 0;
                            s = m.transition[(int64_t)s * m.n_actions + action];
                        }
                        ++env_steps;
                        total += a.cfg.gamma_pow[h] * r;
                        if (term) break;
                    }
                }
                if (SAMPLED && bad_row >= 0)
                    atomicMax(&ctl->rejected, ~(((unsigned long long)e << 32) | (unsigned)bad_row));
                else
                    backup(a, j, reached, total, 0, 1, 0u);
            }
        }
        lap(2);
        grid_barrier(ctl, n_ctas);
        lap(3);
        if constexpr (SAMPLED) {
            if (*(volatile unsigned long long*)&ctl->rejected) break;    // the reference raises in this wave
        }
    }
    // env steps: one count per episode (lane 0 of writer groups / finite threads)
    if (hwy) {
        if (li == 0) atomicAdd(&ctl->env_steps, env_steps);
    } else {
        atomicAdd(&ctl->env_steps, env_steps);
    }
    grid_barrier(ctl, n_ctas);
    if (blockIdx.x != 0) return;
    for (int i = tid; i < a.cfg.node_capacity; i += THREADS) {
        const int c = __ldcg(tr.count + i);
        tr.value[i] = c > 0 ? ((double)__ldcg(tr.vsum + i) / FIX_SCALE) / (double)c : 0.0;
    }
    __syncthreads();
    if (tid == 0) {
        // get_plan with MCTSNode.selection_rule (mcts.py:212-218)
        int node = 0, len = 0;
        while (__ldcg(tr.first_child + node) >= 0) {
            const int fc = __ldcg(tr.first_child + node);
            const int n = (__ldcg(tr.meta + node) >> 8) & 0xff;
            int best = 0;
            for (int i = 1; i < n; ++i) {
                const int ci = __ldcg(tr.count + fc + i), cb = __ldcg(tr.count + fc + best);
                if (ci > cb || (ci == cb && tr.value[fc + i] > tr.value[fc + best])) best = i;
            }
            if (len < H) a.plan[len] = (int8_t)(__ldcg(tr.meta + fc + best) & 0xff);
            ++len;
            node = fc + best;
        }
        a.result[0] = a.cfg.node_capacity;
        a.result[1] = len;
        a.result[2] = *(volatile int*)&ctl->env_steps;
        a.result[3] = (E + W - 1) / W;
        for (int i = 0; i < 4; ++i) a.result[4 + i] = (int32_t)(ctl->prof[i] >> 8);
        if constexpr (SAMPLED) {
            const unsigned long long k = ~*(volatile unsigned long long*)&ctl->rejected;
            a.rejected[0] = ~k ? (int32_t)(k >> 32) : -1;
            a.rejected[1] = ~k ? (int32_t)(unsigned)k : -1;
        }
    }
}

static int64_t align_up(int64_t x) { return (x + 255) & ~(int64_t)255; }
struct Layout { int64_t ctl, paths, plen, expands, recip, total; };
static Layout make_layout(const b2_mcts_wave_config* c) {
    Layout l;
    l.ctl = 0;
    l.paths = align_up(sizeof(Control));
    l.plen = l.paths + align_up((int64_t)c->width * (c->horizon > 0 ? c->horizon : 1) * 4);
    l.expands = l.plen + align_up((int64_t)c->width * 4);
    l.recip = l.expands + align_up((int64_t)c->width * 4);
    l.total = l.recip + align_up(((int64_t)c->episodes + c->width + 2) * 8);
    return l;
}

}  // namespace mwave
}  // namespace b2

using namespace b2;

extern "C" int64_t b2_mcts_wave_workspace_bytes(const b2_mcts_wave_config* cfg) {
    if (!cfg || cfg->width <= 0 || cfg->horizon < 0) return -1;
    return mwave::make_layout(cfg).total;
}

static int check_wave_config(const b2_mcts_wave_config* cfg) {
    B2_REQUIRE(cfg->episodes >= 0 && cfg->horizon >= 0 && cfg->horizon <= mwave::MAX_H, "bad budget / horizon (<= 64)");
    B2_REQUIRE(cfg->width >= 1 && cfg->width <= mwave::MAX_WIDTH, "wave width must be in 1..1024");
    B2_REQUIRE(cfg->n_actions > 0 && cfg->n_actions <= mwave::MAX_A, "n_actions must be in 1..8");
    B2_REQUIRE((int64_t)cfg->node_capacity >= 1 + (int64_t)cfg->episodes * cfg->n_actions, "node_capacity too small");
    B2_REQUIRE(cfg->gamma_pow, "gamma table missing");
    B2_REQUIRE(cfg->rollout_policy == 0 && cfg->prior_policy == 0, "wavefront MCTS implements the random_available policies");
    return B2_OK;
}

// the workspace carve-up and the cooperative launch of mcts_wave_kernel<SAMPLED> on the filled-in Args
template <bool SAMPLED>
static int launch_wave(const b2_mcts_wave_config* cfg, mwave::Args& a, void* workspace, cudaStream_t stream) {
    const mwave::Layout l = mwave::make_layout(cfg);
    char* ws = (char*)workspace;
    a.ctl = (mwave::Control*)(ws + l.ctl);
    a.paths = (int32_t*)(ws + l.paths);
    a.plen = (int32_t*)(ws + l.plen);
    a.expands = (int32_t*)(ws + l.expands);
    a.recip = (double*)(ws + l.recip);
    B2_CUDA_CHECK(cudaMemsetAsync(a.ctl, 0, sizeof(mwave::Control), stream));
    const size_t smem = (size_t)mwave::TABLE_KEYS * 8;
    B2_CUDA_CHECK(cudaFuncSetAttribute(mwave::mcts_wave_kernel<SAMPLED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
    int per_sm = 0;
    B2_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, mwave::mcts_wave_kernel<SAMPLED>,
                                                                mwave::THREADS, smem));
    B2_REQUIRE(per_sm >= 1, "wave kernel does not fit on an SM");
    int grid = sm_count();
    if (cfg->max_ctas > 0 && cfg->max_ctas < grid) grid = cfg->max_ctas;
    void* params[] = {&a};
    B2_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)mwave::mcts_wave_kernel<SAMPLED>, dim3(grid),
                                              dim3(mwave::THREADS), params, smem, stream));
    return B2_OK;
}

extern "C" int b2_mcts_plan_wave(const b2_mcts_wave_config* cfg, const int32_t* root_state, const b2_mcts_wave_tree* tree,
                                 void* workspace, int8_t* plan, int32_t* result, void* stream_) {
    B2_REQUIRE(cfg && root_state && tree && workspace && plan && result, "null pointer");
    if (check_wave_config(cfg) != B2_OK) return B2_ERR_INVALID;
    if (cfg->env_kind == B2_ENV_FINITE) {
        B2_REQUIRE(cfg->mdp.transition && cfg->mdp.reward && cfg->mdp.terminal, "finite MDP tables missing");
        B2_REQUIRE(cfg->mdp.n_actions == cfg->n_actions, "mdp.n_actions != n_actions");
    } else if (cfg->env_kind == B2_ENV_HIGHWAY) {
        B2_REQUIRE(cfg->n_actions == B2_HW_ACTIONS, "HighwayLite has 5 actions");
    } else {
        set_error("unknown env_kind %d", cfg->env_kind);
        return B2_ERR_INVALID;
    }
    mwave::Args a;
    a.cfg = *cfg; a.tree = *tree; a.root_state = root_state;
    a.plan = plan; a.result = result;
    return launch_wave<false>(cfg, a, workspace, (cudaStream_t)stream_);
}

extern "C" int b2_mcts_plan_wave_sampled(const b2_mcts_wave_config* cfg, const b2_finite_mdp_sampled* mdp,
                                         const uint8_t* terminal, int32_t env_draws, const uint64_t* env_rng,
                                         const int32_t* root_state, const b2_mcts_wave_tree* tree, void* workspace,
                                         int8_t* plan, int32_t* result, int32_t* rejected, void* stream_) {
    B2_REQUIRE(cfg && mdp && env_rng && root_state && tree && workspace && plan && result && rejected, "null pointer");
    if (check_wave_config(cfg) != B2_OK) return B2_ERR_INVALID;
    if (check_sampled_entry(cfg->env_kind, *mdp, cfg->n_actions, terminal, env_draws) != B2_OK) return B2_ERR_INVALID;
    mwave::Args a;
    a.cfg = *cfg; a.tree = *tree; a.root_state = root_state;
    a.plan = plan; a.result = result;
    a.smdp = *mdp; a.terminal = terminal; a.env_draws = env_draws; a.env_rng = env_rng; a.rejected = rejected;
    return launch_wave<true>(cfg, a, workspace, (cudaStream_t)stream_);
}
