/* OPD (rl_agents/agents/tree_search/deterministic.py) in plain C on HighwayLite and IntersectionLite -- TEST
 * INFRASTRUCTURE (oracle/).  Mirrors the reference's loop literally (in-loop count walk :64-65
 * and backup_to_root :74-79); only the frontier `max(self.leaves, key=upper)` (:110) is a binary
 * heap ordered by (upper desc, node id asc), which returns the same leaf as Python's first-max
 * over the creation-ordered list.  Used as a fast checker and as the optimised-CPU baseline. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "highway_lite.h"
#include "intersection_lite.h"

/* a scene of either env: the same 136 words */
typedef struct {
    int32_t w[HL_WORDS];
} env_words;
_Static_assert(sizeof(hl_state) == sizeof(env_words) && sizeof(il_state) == sizeof(env_words), "136-word scenes");

/* what the planners need of an env: its action count (budget // n_actions expansions), get_available_actions()
 * in children order, and one step in place (reward; flags bit0 terminated) */
typedef struct {
    int n_actions;
    int (*available)(const env_words* s, int* actions);
    float (*step)(env_words* s, int action, int* flags);
} opd_env;

static int hl_available_w(const env_words* s, int* a) { return hl_available_actions((const hl_state*)s, a); }
static float hl_step_w(env_words* s, int action, int* flags) { return hl_step((hl_state*)s, action, flags); }
static int il_available_w(const env_words* s, int* a) { return il_available_actions((const il_state*)s, a); }
static float il_step_w(env_words* s, int action, int* flags) { return il_step((il_state*)s, action, flags); }
static const opd_env HIGHWAY = {5, hl_available_w, hl_step_w};
static const opd_env INTERSECTION = {3, il_available_w, il_step_w};
#define MAX_ACTIONS 5

typedef struct {
    int32_t *parent, *action, *depth, *count, *first_child, *n_children, *done;
    double *reward, *lower, *upper;
} opd_tree;

static int heap_less(const opd_tree* t, int a, int b) {   /* a worse than b ? */
    if (t->upper[a] != t->upper[b]) return t->upper[a] < t->upper[b];
    return a > b;
}
static void heap_push(const opd_tree* t, int32_t* heap, int* n, int id) {
    int i = (*n)++;
    heap[i] = id;
    while (i > 0) {
        const int p = (i - 1) / 2;
        if (!heap_less(t, heap[p], heap[i])) break;
        const int32_t tmp = heap[p]; heap[p] = heap[i]; heap[i] = tmp;
        i = p;
    }
}
static int heap_pop(const opd_tree* t, int32_t* heap, int* n) {
    const int top = heap[0];
    heap[0] = heap[--(*n)];
    int i = 0;
    for (;;) {
        int l = 2 * i + 1, r = l + 1, m = i;
        if (l < *n && heap_less(t, heap[m], heap[l])) m = l;
        if (r < *n && heap_less(t, heap[m], heap[r])) m = r;
        if (m == i) break;
        const int32_t tmp = heap[m]; heap[m] = heap[i]; heap[i] = tmp;
        i = m;
    }
    return top;
}

/* One plan().  Arrays have capacity 1 + (budget/A)*A for A = env->n_actions.  Returns the number of nodes (or -1
 * when a reward leaves [0,1]); *n_leaves receives the frontier size. */
static int opd_plan_env(const opd_env* env, const int32_t* root_words, int budget, double gamma, double terminal_reward,
                        int32_t* parent, int32_t* action, int32_t* depth, int32_t* count, int32_t* first_child,
                        int32_t* n_children, int32_t* done, double* reward, double* lower, double* upper,
                        int32_t* n_leaves) {
    const int n_exp = budget / env->n_actions, cap = 1 + n_exp * env->n_actions;
    opd_tree t = {parent, action, depth, count, first_child, n_children, done, reward, lower, upper};
    env_words* states = (env_words*)malloc((size_t)cap * sizeof(env_words));
    int32_t* heap = (int32_t*)malloc((size_t)cap * sizeof(int32_t));
    int heap_n = 0, n = 1;
    memcpy(&states[0], root_words, sizeof(env_words));
    parent[0] = -1; action[0] = -1; depth[0] = 0; count[0] = 1; first_child[0] = -1; n_children[0] = 0; done[0] = 0;
    reward[0] = lower[0] = upper[0] = 0.0;
    heap_push(&t, heap, &heap_n, 0);
    for (int it = 0; it < n_exp; ++it) {
        const int leaf = heap_pop(&t, heap, &heap_n);
        int acts[MAX_ACTIONS];
        const int na = env->available(&states[leaf], acts);
        first_child[leaf] = n;
        n_children[leaf] = na;
        const int d = depth[leaf] + 1;
        for (int k = 0; k < na; ++k) {
            const int c = n++;
            states[c] = states[leaf];
            int flags;
            const double r = (double)env->step(&states[c], acts[k], &flags);
            if (!(r >= 0.0 && r <= 1.0)) { free(states); free(heap); return -1; }
            parent[c] = leaf; action[c] = acts[k]; depth[c] = d; count[c] = 1; first_child[c] = -1; n_children[c] = 0;
            done[c] = flags & 1;
            reward[c] = r;
            lower[c] = lower[leaf] + pow(gamma, d - 1) * r;
            upper[c] = lower[c] + pow(gamma, d) / (1 - gamma);
            if (done[c]) { lower[c] = lower[c] + terminal_reward * pow(gamma, d) / (1 - gamma); upper[c] = lower[c]; }
            for (int a = c; a >= 0; a = parent[a]) count[a] += 1;
            heap_push(&t, heap, &heap_n, c);
        }
        for (int p = leaf; p >= 0; p = parent[p]) {
            double lo = lower[first_child[p]], up = upper[first_child[p]];
            for (int k = 1; k < n_children[p]; ++k) {
                const int c = first_child[p] + k;
                if (lower[c] > lo) lo = lower[c];
                if (upper[c] > up) up = upper[c];
            }
            lower[p] = lo;
            upper[p] = up;
        }
    }
    *n_leaves = heap_n;
    free(states);
    free(heap);
    return n;
}

int opd_highway_plan(const int32_t* root_words, int budget, double gamma, double terminal_reward, int32_t* parent,
                     int32_t* action, int32_t* depth, int32_t* count, int32_t* first_child, int32_t* n_children,
                     int32_t* done, double* reward, double* lower, double* upper, int32_t* n_leaves) {
    return opd_plan_env(&HIGHWAY, root_words, budget, gamma, terminal_reward, parent, action, depth, count, first_child,
                        n_children, done, reward, lower, upper, n_leaves);
}

int il_opd_plan(const int32_t* root_words, int budget, double gamma, double terminal_reward, int32_t* parent,
                int32_t* action, int32_t* depth, int32_t* count, int32_t* first_child, int32_t* n_children,
                int32_t* done, double* reward, double* lower, double* upper, int32_t* n_leaves) {
    return opd_plan_env(&INTERSECTION, root_words, budget, gamma, terminal_reward, parent, action, depth, count,
                        first_child, n_children, done, reward, lower, upper, n_leaves);
}

static int cmp_int(const void* a, const void* b) { return *(const int32_t*)a - *(const int32_t*)b; }

/* SPECIFICATION of the wavefront OPD (oracle/planners.py::opd_plan_wavefront, same statement in C): per wave
 * the k = min(width, expansions left, frontier size) best leaves by (upper desc, id asc) are expanded in
 * increasing id order; counts and backups bottom-up afterwards.  width = 1 is opd_plan_env.  `wave_end` (may be
 * NULL; capacity 1 + budget/A) receives, per wave, the number of nodes after it: wave w created the ids
 * wave_end[w-1] .. wave_end[w]-1 (wave_end[-1] = 1), in the order the device's work list simulates them. */
static int opd_plan_wave_env(const opd_env* env, const int32_t* root_words, int budget, double gamma,
                             double terminal_reward, int width, int lag, int32_t* parent, int32_t* action,
                             int32_t* depth, int32_t* count, int32_t* first_child, int32_t* n_children, int32_t* done,
                             double* reward, double* lower, double* upper, int32_t* n_leaves, int32_t* n_waves,
                             int32_t* wave_end) {
    const int n_exp = budget / env->n_actions, cap = 1 + n_exp * env->n_actions;
    opd_tree t = {parent, action, depth, count, first_child, n_children, done, reward, lower, upper};
    env_words* states = (env_words*)malloc((size_t)cap * sizeof(env_words));
    int32_t* heap = (int32_t*)malloc((size_t)cap * sizeof(int32_t));
    int32_t* chosen = (int32_t*)malloc((size_t)(width > 0 ? width : 1) * sizeof(int32_t));
    /* lag = 1 (pipelined waves): the children of a wave become eligible one wave later -- wave w is chosen
     * from the frontier as it was before wave w-1's children were added (unless nothing else is left) */
    int32_t* pending = (int32_t*)malloc((size_t)cap * sizeof(int32_t));
    int n_pending = 0;
    int heap_n = 0, n = 1, remaining = n_exp, waves = 0;
    memcpy(&states[0], root_words, sizeof(env_words));
    parent[0] = -1; action[0] = -1; depth[0] = 0; count[0] = 1; first_child[0] = -1; n_children[0] = 0; done[0] = 0;
    reward[0] = lower[0] = upper[0] = 0.0;
    heap_push(&t, heap, &heap_n, 0);
    while (remaining > 0) {
        if (heap_n == 0) {                       /* only the held-back children are left: release them */
            for (int j = 0; j < n_pending; ++j) heap_push(&t, heap, &heap_n, pending[j]);
            n_pending = 0;
        }
        int k = width < remaining ? width : remaining;
        if (k > heap_n) k = heap_n;
        for (int j = 0; j < k; ++j) chosen[j] = heap_pop(&t, heap, &heap_n);
        for (int j = 0; j < n_pending; ++j) heap_push(&t, heap, &heap_n, pending[j]);
        n_pending = 0;
        qsort(chosen, (size_t)k, sizeof(int32_t), cmp_int);
        for (int j = 0; j < k; ++j) {
            const int leaf = chosen[j];
            int acts[MAX_ACTIONS];
            const int na = env->available(&states[leaf], acts);
            first_child[leaf] = n;
            n_children[leaf] = na;
            const int d = depth[leaf] + 1;
            for (int q = 0; q < na; ++q) {
                const int c = n++;
                states[c] = states[leaf];
                int flags;
                const double r = (double)env->step(&states[c], acts[q], &flags);
                if (!(r >= 0.0 && r <= 1.0)) { free(states); free(heap); free(chosen); free(pending); return -1; }
                parent[c] = leaf; action[c] = acts[q]; depth[c] = d; count[c] = 1; first_child[c] = -1; n_children[c] = 0;
                done[c] = flags & 1;
                reward[c] = r;
                lower[c] = lower[leaf] + pow(gamma, d - 1) * r;
                upper[c] = lower[c] + pow(gamma, d) / (1 - gamma);
                if (done[c]) { lower[c] = lower[c] + terminal_reward * pow(gamma, d) / (1 - gamma); upper[c] = lower[c]; }
                if (lag) pending[n_pending++] = c; else heap_push(&t, heap, &heap_n, c);
            }
        }
        remaining -= k;
        if (wave_end) wave_end[waves] = n;
        ++waves;
    }
    for (int c = n - 1; c > 0; --c)
        for (int a = c; a >= 0; a = parent[a]) count[a] += 1;
    for (int p = n - 1; p >= 0; --p) {
        if (!n_children[p]) continue;
        double lo = lower[first_child[p]], up = upper[first_child[p]];
        for (int q = 1; q < n_children[p]; ++q) {
            const int c = first_child[p] + q;
            if (lower[c] > lo) lo = lower[c];
            if (upper[c] > up) up = upper[c];
        }
        lower[p] = lo;
        upper[p] = up;
    }
    *n_leaves = heap_n + n_pending;
    *n_waves = waves;
    free(states);
    free(heap);
    free(chosen);
    free(pending);
    return n;
}

int opd_highway_plan_wave(const int32_t* root_words, int budget, double gamma, double terminal_reward, int width, int lag,
                          int32_t* parent, int32_t* action, int32_t* depth, int32_t* count, int32_t* first_child,
                          int32_t* n_children, int32_t* done, double* reward, double* lower, double* upper,
                          int32_t* n_leaves, int32_t* n_waves) {
    return opd_plan_wave_env(&HIGHWAY, root_words, budget, gamma, terminal_reward, width, lag, parent, action, depth,
                             count, first_child, n_children, done, reward, lower, upper, n_leaves, n_waves, NULL);
}

int il_opd_plan_wave(const int32_t* root_words, int budget, double gamma, double terminal_reward, int width, int lag,
                     int32_t* parent, int32_t* action, int32_t* depth, int32_t* count, int32_t* first_child,
                     int32_t* n_children, int32_t* done, double* reward, double* lower, double* upper,
                     int32_t* n_leaves, int32_t* n_waves, int32_t* wave_end) {
    return opd_plan_wave_env(&INTERSECTION, root_words, budget, gamma, terminal_reward, width, lag, parent, action,
                             depth, count, first_child, n_children, done, reward, lower, upper, n_leaves, n_waves,
                             wave_end);
}

/* batched env steps (for parity tests of the env alone) */
void hl_step_batch(int32_t* words, const int32_t* actions, float* rewards, int32_t* flags, int n) {
    for (int i = 0; i < n; ++i) rewards[i] = hl_step((hl_state*)(words + (size_t)i * HL_WORDS), actions[i], &flags[i]);
}
