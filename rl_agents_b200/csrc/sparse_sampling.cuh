// Pieces shared by the two sparse-sampling kernels: the depth-first lane kernel (sparse_sampling.cu) and the
// level-synchronous one-decision kernel (sparse_sampling_levels.cu).
#pragma once
#include "common.cuh"
#include "pcg64.cuh"

namespace b2 {
namespace ss {

constexpr int KIND_DECISION = 0, KIND_CHANCE = 1;
constexpr int ERR_CAPACITY = 1, ERR_BAD_ROW = 2;

// DecisionNode / ChanceNode.__init__ (:32-36, :65-69): value 0, count 0
__device__ __forceinline__ void put(const b2_sparse_sampling_tree& tr, int64_t nb, int id, int parent, int kind, int key,
                                    int depth) {
    tr.parent[nb + id] = parent; tr.kind[nb + id] = kind; tr.key[nb + id] = key; tr.depth[nb + id] = depth;
    tr.count[nb + id] = 0; tr.value[nb + id] = 0.0;
}

// get_plan: root.selection_rule, random_argmax (:26-28, :53-56; abstract.py:304-311) over the root's nc available
// actions, action_at(i) the i-th of them in env order: the first maximum of root_q, or choice(indices) among the
// tied maxima, which draws from the planner's stream only for two or more ties.
template <class ActionAt>
__device__ __forceinline__ int root_plan(const double* root_q, int nc, ActionAt action_at, Pcg64& rng) {
    double m = root_q[action_at(0)];
    int ties = 1;
    for (int i = 1; i < nc; ++i) {
        const double v = root_q[action_at(i)];
        if (v > m) { m = v; ties = 1; } else if (v == m) ++ties;
    }
    int pick = (int)rng.integers((uint32_t)ties);
    for (int i = 0; i < nc; ++i) {
        const int act = action_at(i);
        if (root_q[act] == m && pick-- == 0) return act;
    }
    return -1;
}

}  // namespace ss
}  // namespace b2
