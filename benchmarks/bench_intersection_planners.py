#!/usr/bin/env python
"""MCTS and OLOP on IntersectionLite: batch throughput (decisions/s, env steps/s) of b2_mcts_plan and b2_olop_plan on
IntersectionLite scenes, at C3's search size (MCTS 4096 episodes x horizon 20, gamma 0.8, temperature 10; OLOP at the
same episodes x horizon) and at the agents' default budgets (MCTSAgent budget 100, OLOPAgent budget 500 with the KL
bound and the "uniform" continuation, gamma 0.8), each beside the HighwayLite instantiation at the same config in the
same process.  Kernel time from CUDA events around the launches after a warm-up launch.  One JSON line, with the GPU's
name and power limit; --out also writes it to a file."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.bench_mdp_gape import gpu_info  # noqa: E402

KL = {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="decisions per launch (default: 64 per SM)")
    ap.add_argument("--reps", type=int, default=5, help="timed launches at the default budgets")
    ap.add_argument("--c3-reps", type=int, default=1, help="timed launches at C3's size")
    ap.add_argument("--c3-episodes", type=int, default=4096)
    ap.add_argument("--out", default="", help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mcts import allocation
    from rl_agents_b200.engine.mcts import MCTSEngine, pcg64_words
    from rl_agents_b200.engine.olop import OLOPEngine
    from rl_agents_b200.envs import highway_lite, intersection_lite
    assert torch.cuda.is_available(), "bench_intersection_planners needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.trees or torch.cuda.get_device_properties(dev).multi_processor_count * 64
    envs = {"intersection": (_lib.ENV_INTERSECTION, 3, intersection_lite.make_scene),
            "highway": (_lib.ENV_HIGHWAY, 5, highway_lite.make_scene)}
    words = np.stack([pcg64_words(np.random.Generator(np.random.PCG64(np.random.SeedSequence(i)))) for i in range(n)])
    mcts_default = allocation(100, 0.8)
    olop_default = allocation(500, 0.8)
    # OLOP keeps episodes x horizon x actions nodes per tree (2 GB per 128 HighwayLite trees at C3's size): one
    # eighth of the batch there
    configs = (("mcts_c3", "mcts", args.c3_episodes, 20, args.c3_reps, n),
               ("mcts_default_budget100", "mcts", mcts_default[0], mcts_default[1], args.reps, n),
               ("olop_c3", "olop", args.c3_episodes, 20, args.c3_reps, n // 8),
               ("olop_default_budget500", "olop", olop_default[0], olop_default[1], args.reps, n))
    out = dict(gpu_info(), trees=n, gamma=0.8, results={})
    for name, planner, episodes, horizon, reps, trees in configs:
        row = {"planner": planner, "episodes": episodes, "horizon": horizon, "trees": trees}
        for env_name, (kind, n_actions, make_scene) in envs.items():
            scenes = torch.from_numpy(np.stack([make_scene(i) for i in range(trees)])).to(dev)

            def engine(ep):
                if planner == "mcts":
                    return MCTSEngine(kind, trees, n_actions, ep, horizon, 0.8, 10.0, device=dev)
                return OLOPEngine(kind, trees, n_actions, ep, horizon, 0.8, KL, "uniform", device=dev)
            warm = engine(2)
            warm.plan(scenes, words[:trees])
            warm.finish()
            del warm
            eng = engine(episodes)
            eng.plan(scenes, words[:trees])                # warm-up at the timed shape
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                eng.plan(scenes, words[:trees])
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            _, res, _ = eng.finish()
            r = {"ms_per_launch": ms, "decisions_per_s": trees / (ms * 1e-3), "mean_nodes": float(res[:, 0].mean())}
            if planner == "mcts":
                r["env_steps_per_s"] = float(res[:, 2].sum()) / (ms * 1e-3)
            else:
                r["env_steps_per_s"] = trees * episodes * horizon / (ms * 1e-3)
            row[env_name] = r
            del eng
            torch.cuda.empty_cache()
        row["intersection_over_highway_time"] = row["intersection"]["ms_per_launch"] / row["highway"]["ms_per_launch"]
        out["results"][name] = row
        print(name, json.dumps(row), file=sys.stderr, flush=True)
    line = json.dumps(dict(metric="MCTS / OLOP decisions/s on IntersectionLite beside HighwayLite", **out))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
