"""How often the warp-uniform blocks of `hw::step`'s sub-step run on the C2 workload, before and after their gates
were narrowed to the vehicles that read their results.  CPU only: no GPU, no timing.

Builds the C oracle's OPD tree of each scene (`make_highway_state(seed)`, budget 10 000, gamma 0.8, as `bench.py`),
samples expansions of it, replays the children of each sampled expansion through `oracle/envs.py::highway_step` with
its `on_substep` hook, and pairs consecutive children the way the batch kernel packs them onto a warp (one child per
16-lane half).  A block runs in a warp-sub-step when its vote is true for either half.

    python benchmarks/step_path_frequencies.py [--scenes 0 1 2 100 101 102] [--samples 3] [--expansions 120]

Blocks (the vote in `hw::step`, before -> after):
  lane change  lane-entering ballots, target-lane front, abort loop:
               some present vehicle has cur != tgt -> some present, not crashed IDM vehicle (slot > 0) has cur != tgt
  a_t          IDM behind the target-lane front: some vehicle has cur != new_tgt -> some active one has
  MOBIL        the decider server: some vehicle decides -> some decider has |v| >= 1 and a_free - self_a >= 0.2
  MOBIL sides  the decider server behind the per-side own-gain screen (own_gain_shut in highway_lite.cuh): the MOBIL
               vote above -> some (decider, side) pair with the side lane on the road survives the screen.  The
               screen's threshold k comes from an approximate square root on the device and from numpy's here; it
               is checked with the same fp32 operations in both, so only the rare k at the edge of the check differs.
               Also reported: the served pairs per pass of the server (up to eight per 16-lane group).
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import c_oracle  # noqa: E402
from oracle import envs as oenvs  # noqa: E402

BLOCKS = ("lane change", "a_t", "MOBIL", "MOBIL sides")
K_SHUT = np.float32(float.fromhex("0x1.55aaaap-2"))


def served_sides(x, y, v, present, cur, ts, a_free, self_a, mobil):
    """[2, V] booleans: (decider, side) pairs that the own-gain screen leaves to the server (side 0 left, 1 right)"""
    f32 = np.float32
    gain = mobil & ~((a_free - self_a) < oenvs.MOBIL_MIN_GAIN)
    with np.errstate(all="ignore"):
        k = np.sqrt(((a_free - self_a) - oenvs.MOBIL_MIN_GAIN) * K_SHUT).astype(f32)
        k_shuts = (k >= f32(2.0 ** -8)) & ((a_free - oenvs.COMFORT_ACC_MAX * (k * k)) - self_a < oenvs.MOBIL_MIN_GAIN)
        g0 = oenvs.D0 + v * oenvs.TAU
        out = []
        for side in (-1, 1):
            lane = cur + side
            hf, f, _, _ = oenvs._neighbours(x, present, lane.astype(f32) * oenvs.LANE_W, y)
            ag = np.abs(g0 + (v * (v - v[f])) / oenvs.TWO_SQRT_AB)
            dist = np.maximum(np.abs(x[f] - x), oenvs.EPS)
            # sign of fma(k, dist, -ag): the product of two fp32 values is exact in fp64
            shut = (ag < f32(2.0 ** 32)) & (k.astype(np.float64) * dist - ag < 0)
            out.append(gain & (lane >= 0) & (lane < oenvs.N_LANES) & ~(k_shuts & hf & shut))
    return np.stack(out)


def substep_votes(state, action, pairs=None):
    """[SUBSTEPS, 2 * len(BLOCKS)] booleans per sub-step of one child: each block's vote before and after, for this
    scene alone.  Steps `state` in place.  `pairs`, when given, collects the served (decider, side) pairs of each
    sub-step."""
    rows = []
    ts = state.tgt_speed      # IDM vehicles' target speeds; the ego's (updated by the meta-action) is never read here

    def obs(x, y, v, present, crashed, cur, tgt, new_tgt, decide, **_):
        idm = np.arange(oenvs.V_SLOTS) > 0
        active = present & ~crashed & idm
        a_free = oenvs._idm(v, ts, np.zeros(oenvs.V_SLOTS, bool), x, x, v)
        hf, f, _, _ = oenvs._neighbours(x, present, cur.astype(np.float32) * oenvs.LANE_W, y)
        self_a = oenvs._idm(v, ts, hf, x, x[f], v[f])
        mobil = decide & (np.abs(v) >= np.float32(1.0)) & ~((a_free - self_a) < oenvs.MOBIL_MIN_GAIN)
        sides = served_sides(x, y, v, present, cur, ts, a_free, self_a, mobil)
        if pairs is not None:
            pairs.append(int(sides.sum()))
        rows.append([(present & (cur != tgt)).any(), (active & (cur != tgt)).any(),
                     (cur != new_tgt).any(), (active & (cur != new_tgt)).any(),
                     decide.any(), mobil.any(), mobil.any(), sides.any()])
    oenvs.highway_step(state, action, on_substep=obs)
    return np.array(rows, bool)


def children_of_sampled_expansions(root_words, tree, rng, n_expansions):
    """(parent state, action) of every child of `n_expansions` expansions drawn from the tree, in creation order"""
    parents = np.unique(tree["parent"][1:])
    pick = np.sort(rng.choice(parents, size=min(n_expansions, parents.size), replace=False))
    cache = {0: oenvs.HighwayLiteState.unpack(root_words)}

    def state_of(k):
        if k not in cache:
            s = state_of(int(tree["parent"][k])).copy()
            oenvs.highway_step(s, int(tree["action"][k]))
            cache[k] = s
        return cache[k]
    out = []
    for p in pick:
        first, n = int(tree["first_child"][p]), int(tree["n_children"][p])
        for c in range(first, first + n):
            out.append((state_of(int(p)), int(tree["action"][c])))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--scenes", type=int, nargs="+", default=[0, 1, 2, 100, 101, 102])
    ap.add_argument("--budget", type=int, default=10000)
    ap.add_argument("--gamma", type=float, default=0.8)
    ap.add_argument("--samples", type=int, default=3, help="independent samples of expansions per scene set")
    ap.add_argument("--expansions", type=int, default=120, help="expansions per sample (about 3.8 children each)")
    a = ap.parse_args()
    sys.setrecursionlimit(10000)
    trees = {s: c_oracle.opd_plan(oenvs.make_highway_state(s).pack(), a.budget, a.gamma) for s in a.scenes}
    print("C oracle OPD trees: scenes %s, budget %d, gamma %g" % (a.scenes, a.budget, a.gamma))
    print("%-8s %-12s %9s %9s %9s %9s %9s" % ("sample", "block", "children", "scene", "scene", "warp", "warp"))
    print("%-8s %-12s %9s %9s %9s %9s %9s" % ("", "", "", "before", "after", "before", "after"))
    for k in range(a.samples):
        rng = np.random.default_rng(k)
        votes, pairs = [], []
        for s in a.scenes:
            words = oenvs.make_highway_state(s).pack()
            n = max(1, a.expansions // len(a.scenes))
            for parent, action in children_of_sampled_expansions(words, trees[s], rng, n):
                votes.append(substep_votes(parent.copy(), action, pairs))
        votes = np.stack(votes)                                   # [children, SUBSTEPS, 2 * blocks]
        warps = votes[: len(votes) // 2 * 2].reshape(-1, 2, *votes.shape[1:]).any(axis=1)
        for b, name in enumerate(BLOCKS):
            print("%-8d %-12s %9d %8.1f%% %8.1f%% %8.1f%% %8.1f%%" % (
                k, name, len(votes), 100 * votes[..., 2 * b].mean(), 100 * votes[..., 2 * b + 1].mean(),
                100 * warps[..., 2 * b].mean(), 100 * warps[..., 2 * b + 1].mean()))
        pairs = np.array(pairs)
        served = pairs[pairs > 0]
        print("%-8d served (decider, side) pairs per group pass: mean %.2f, max %d; passes with more than 8: %d" % (
            k, served.mean() if served.size else 0.0, served.max() if served.size else 0, (served > 8).sum()))


if __name__ == "__main__":
    main()
