/* MCTS (rl_agents/agents/tree_search/mcts.py, open loop, random_available policies) in plain C on IntersectionLite,
 * consuming a numpy PCG64 stream exactly like Generator.choice does -- TEST INFRASTRUCTURE (oracle/).  Literal
 * restatement of oracle/planners.py::mcts_plan on il_step, the same search as mcts.c's mcts_highway_plan; lets the
 * C3 configuration (4096 episodes x horizon 20) be checked bit for bit at full size on IntersectionLite scenes.
 * Built on its own (oracle/c_mcts_intersection.py) with the Makefile's flags. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "intersection_lite.h"

typedef unsigned __int128 u128;
typedef struct { u128 state, inc; uint32_t has32, uinteger; } pcg64;

/* numpy's PCG64 (XSL-RR 128/64), next_uint32 with the buffered half, random() and integers(0, n) */
static uint64_t pcg_next64(pcg64* g) {
    const u128 mult = ((u128)0x2360ED051FC65DA4ULL << 64) | 0x4385DF649FCCF645ULL;
    g->state = g->state * mult + g->inc;
    const uint64_t hi = (uint64_t)(g->state >> 64), lo = (uint64_t)g->state, x = hi ^ lo;
    const unsigned rot = (unsigned)(hi >> 58);
    return (x >> rot) | (x << ((64 - rot) & 63));
}
static uint32_t pcg_next32(pcg64* g) {
    if (g->has32) { g->has32 = 0; return g->uinteger; }
    const uint64_t n = pcg_next64(g);
    g->has32 = 1;
    g->uinteger = (uint32_t)(n >> 32);
    return (uint32_t)n;
}
static double pcg_random(pcg64* g) { return (double)(pcg_next64(g) >> 11) * (1.0 / 9007199254740992.0); }
static uint32_t pcg_integers(pcg64* g, uint32_t n) {
    const uint32_t rng = n - 1;
    if (rng == 0) return 0;
    const uint32_t rng_excl = rng + 1;
    uint64_t m = (uint64_t)pcg_next32(g) * rng_excl;
    uint32_t leftover = (uint32_t)m;
    if (leftover < rng_excl) {
        const uint32_t threshold = (0xFFFFFFFFu - rng) % rng_excl;
        while (leftover < threshold) { m = (uint64_t)pcg_next32(g) * rng_excl; leftover = (uint32_t)m; }
    }
    return (uint32_t)(m >> 32);
}

/* rng_words: 6 x uint64 (state hi, lo, inc hi, lo, has_uint32, uinteger), advanced in place.
 * cdf: [(3+1), 3] uniform cdfs from numpy.  Arrays have capacity 1 + episodes*3.  Returns #nodes;
 * *env_steps: the transitions taken. */
int mcts_intersection_plan(const int32_t* root_words, int episodes, int horizon, double gamma, double temperature,
                           uint64_t* rng_words, const double* cdf, int32_t* parent, int32_t* action, int32_t* count,
                           int32_t* first_child, int32_t* n_children, double* value, double* prior, int64_t* env_steps) {
    pcg64 g;
    g.state = ((u128)rng_words[0] << 64) | rng_words[1];
    g.inc = ((u128)rng_words[2] << 64) | rng_words[3];
    g.has32 = (uint32_t)rng_words[4];
    g.uinteger = (uint32_t)rng_words[5];
    int n = 1;
    int64_t steps = 0;
    parent[0] = -1; action[0] = -1; count[0] = 0; first_child[0] = -1; n_children[0] = 0; value[0] = 0.0; prior[0] = 1.0;
    il_state root, st;
    memcpy(&root, root_words, sizeof(root));
    for (int ep = 0; ep < episodes; ++ep) {
        st = root;                                                                /* safe_deepcopy_env, :183 */
        int node = 0, depth = 0, terminal = 0;
        double total = 0.0;
        while (depth < horizon && n_children[node] > 0 && !terminal) {          /* mcts.py:141-149 */
            const int fc = first_child[node], k = n_children[node];
            double sc[3], best = -INFINITY;
            int ties = 0;
            for (int i = 0; i < k; ++i) {
                sc[i] = value[fc + i] + temperature * (double)k * prior[fc + i] / (double)(count[fc + i] + 1);
                if (sc[i] > best) { best = sc[i]; ties = 1; } else if (sc[i] == best) ++ties;
            }
            int pick = (int)pcg_integers(&g, (uint32_t)ties), sel = 0;          /* random_argmax */
            for (int i = 0; i < k; ++i)
                if (sc[i] == best) { if (pick == 0) sel = i; --pick; }
            int flags;
            const double r = (double)il_step(&st, action[fc + sel], &flags);
            ++steps;
            terminal = flags & 1;
            total += pow(gamma, depth) * r;
            node = fc + sel;
            depth += 1;
        }
        if (n_children[node] == 0 && depth < horizon && (!terminal || node == 0)) {   /* :151-154 */
            int acts[3];
            const int k = il_available_actions(&st, acts);
            first_child[node] = n;
            n_children[node] = k;
            for (int i = 0; i < k; ++i) {
                parent[n] = node; action[n] = acts[i]; count[n] = 0; first_child[n] = -1; n_children[n] = 0;
                value[n] = 0.0; prior[n] = 1.0 / (double)k;
                ++n;
            }
        }
        if (!terminal) {                                                          /* evaluate :160-177 */
            for (int h = depth; h < horizon; ++h) {
                int acts[3];
                const int k = il_available_actions(&st, acts);
                const double u = pcg_random(&g);
                const double* c = cdf + (size_t)k * 3;
                int idx = 0;
                for (int i = 0; i < k; ++i) idx += c[i] <= u ? 1 : 0;
                if (idx > k - 1) idx = k - 1;
                int flags;
                const double r = (double)il_step(&st, acts[idx], &flags);
                ++steps;
                total += pow(gamma, h) * r;
                if (flags & 3) break;
            }
        }
        for (int a = node; a >= 0; a = parent[a]) {                               /* update_branch :257-265 */
            count[a] += 1;
            value[a] += 1.0 / (double)count[a] * (total - value[a]);
        }
    }
    rng_words[0] = (uint64_t)(g.state >> 64); rng_words[1] = (uint64_t)g.state;
    rng_words[2] = (uint64_t)(g.inc >> 64); rng_words[3] = (uint64_t)g.inc;
    rng_words[4] = g.has32; rng_words[5] = g.uinteger;
    *env_steps = steps;
    return n;
}
