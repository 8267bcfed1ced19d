// Batched MCTS re-root (b2_mcts_reroot): step_strategy "subtree" (abstract.py:195-206) on the device, out of place.
// Destination tree j receives the sub-tree of its source tree under the root child of action[j], re-indexed breadth
// first with the children of a node contiguous and in order -- bit for bit what engine/mcts.py::reroot_arrays does.
//
// One warp per destination tree, level by level.  Level k+1 is the concatenation of the children of level k in order,
// which is the order of reroot_arrays' queue: a warp exclusive scan of the child counts of a 32-node chunk, carried
// across chunks, gives every child its position.  Until a node is processed, its destination first_child slot holds
// the source index of the node, so the walk needs no scratch.  Depth is bounded by the search horizon.
#include "common.cuh"

namespace b2 {
namespace {

constexpr int kWarps = 4;
constexpr unsigned kFull = 0xffffffffu;
constexpr int KEPT_BAD_SOURCE = -1;

struct RerootArgs {
    b2_mcts_tree src, dst;
    int32_t n_src, src_capacity, src_nodes_stride, n_dst, dst_capacity, reserve;
    const int32_t* src_nodes;
    const int32_t* src_tree;
    const int32_t* action;
    int32_t* kept;
};

__global__ void __launch_bounds__(kWarps * 32) mcts_reroot_kernel(RerootArgs a) {
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (j >= a.n_dst) return;                                   // warp-uniform
    const int s = a.src_tree ? a.src_tree[j] : j;
    int n = 0;
    if (s >= 0 && s < a.n_src) n = a.src_nodes[(int64_t)s * a.src_nodes_stride];
    if (n < 1 || n > a.src_capacity) {                          // nothing of the source is read, nothing written
        if (lane == 0) a.kept[j] = KEPT_BAD_SOURCE;
        return;
    }
    const b2_mcts_tree& src = a.src;
    const b2_mcts_tree& dst = a.dst;
    const int64_t sb = (int64_t)s * a.src_capacity, db = (int64_t)j * a.dst_capacity;
    const int act = a.action[j];

    // the root's child of action `act` (the last one, as reroot_arrays scans them all)
    int root_child = -1;
    if (act >= 0) {
        const int fc0 = src.first_child[sb];
        const int k0 = fc0 >= 0 ? (src.meta[sb] >> 8) & 0xff : 0;
        if (k0 && (fc0 < 1 || fc0 + k0 > n)) {                  // a child range outside the tree
            if (lane == 0) a.kept[j] = KEPT_BAD_SOURCE;
            return;
        }
        for (int base = 0; base < k0; base += 32) {
            const int c = base + lane;
            const unsigned hit = __ballot_sync(kFull, c < k0 && (src.meta[sb + fc0 + c] & 0xff) == act);
            if (hit) root_child = fc0 + base + 31 - __clz(hit);
        }
    }
    // kept + reserve > capacity: MCTSEngine's fall-back to a fresh tree
    const int limit = a.dst_capacity - a.reserve;
    if (root_child < 0 || limit < 1) {
        if (lane == 0) a.kept[j] = 0;
        return;
    }
    if (lane == 0) {
        dst.parent[db] = -1;
        dst.first_child[db] = root_child;
    }
    __syncwarp();

    int lo = 0, hi = 1, next = 1;                               // level [lo, hi); next: the first free position
    while (lo < hi) {
        for (int base = lo; base < hi; base += 32) {
            const int p = base + lane;
            int k = 0, sfc = -1;
            bool bad = false;
            if (p < hi) {
                const int old = dst.first_child[db + p];        // the source index of node p
                const int m = src.meta[sb + old];
                sfc = src.first_child[sb + old];
                k = sfc >= 0 ? (m >> 8) & 0xff : 0;
                bad = k && (sfc < 1 || sfc + k > n);
                dst.count[db + p] = src.count[sb + old];
                dst.meta[db + p] = p == 0 ? m | 0xff : m;       // the new root has no incoming action
                dst.value[db + p] = src.value[sb + old];
                dst.prior[db + p] = src.prior[sb + old];
            }
            if (__any_sync(kFull, bad)) {
                if (lane == 0) a.kept[j] = KEPT_BAD_SOURCE;
                return;
            }
            int incl = k;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int y = __shfl_up_sync(kFull, incl, d);
                if (lane >= d) incl += y;
            }
            const int total = __shfl_sync(kFull, incl, 31);
            if (next + total > limit) {
                if (lane == 0) a.kept[j] = 0;
                return;
            }
            if (p < hi) {
                const int first = next + incl - k;
                dst.first_child[db + p] = k ? first : -1;
                for (int c = 0; c < k; ++c) {
                    dst.parent[db + first + c] = p;
                    dst.first_child[db + first + c] = sfc + c;  // read back when the child's level is processed
                }
            }
            next += total;
            __syncwarp();
        }
        lo = hi;
        hi = next;
    }
    if (lane == 0) a.kept[j] = next;
}

bool any_shared(const b2_mcts_tree& x, const b2_mcts_tree& y) {
    const void* px[] = {x.parent, x.first_child, x.count, x.meta, x.value, x.prior};
    const void* py[] = {y.parent, y.first_child, y.count, y.meta, y.value, y.prior};
    for (const void* p : px)
        for (const void* q : py)
            if (p == q) return true;
    return false;
}

bool complete(const b2_mcts_tree& t) {
    return t.parent && t.first_child && t.count && t.meta && t.value && t.prior;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" int b2_mcts_reroot(const b2_mcts_tree* src, int32_t n_src, int32_t src_capacity, const int32_t* src_nodes,
                              int32_t src_nodes_stride, const b2_mcts_tree* dst, int32_t n_dst, int32_t dst_capacity,
                              const int32_t* src_tree, const int32_t* action, int32_t reserve, int32_t* kept,
                              void* stream) {
    B2_REQUIRE(src && dst && src_nodes && action && kept && complete(*src) && complete(*dst), "null pointer");
    B2_REQUIRE(n_dst >= 1, "n_dst must be >= 1");
    B2_REQUIRE(n_src >= 1 && src_capacity >= 1 && dst_capacity >= 1 && src_nodes_stride >= 1,
               "n_src, capacities and src_nodes_stride must be >= 1");
    B2_REQUIRE(!any_shared(*src, *dst), "the destination arena must not share an array with the source");
    B2_REQUIRE(reserve >= 0, "reserve must be >= 0");
    RerootArgs a;
    a.src = *src; a.dst = *dst;
    a.n_src = n_src; a.src_capacity = src_capacity; a.src_nodes_stride = src_nodes_stride;
    a.n_dst = n_dst; a.dst_capacity = dst_capacity; a.reserve = reserve;
    a.src_nodes = src_nodes; a.src_tree = src_tree; a.action = action; a.kept = kept;
    const int blocks = (n_dst + kWarps - 1) / kWarps;
    mcts_reroot_kernel<<<blocks, kWarps * 32, 0, (cudaStream_t)stream>>>(a);
    B2_CUDA_CHECK(cudaGetLastError());
    return B2_OK;
}
