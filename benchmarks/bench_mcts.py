#!/usr/bin/env python
"""MCTS benchmark (BASELINE.json configs[2], C3): MCTSAgent on HighwayLite, episodes 4096,
horizon 20, gamma 0.8, temperature 10 -- a batch of independent decisions, strict episode
order inside every tree.  Prints one JSON line: episodes/s and env-steps/s."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="decisions per launch (default 64 per SM)")
    ap.add_argument("--episodes", type=int, default=256, help="C3 asks for 4096; 256 keeps the default run short")
    ap.add_argument("--horizon", type=int, default=20)
    ap.add_argument("--steps", type=int, default=1)
    a = ap.parse_args()
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import MCTSEngine, pcg64_words
    from rl_agents_b200.envs.highway_lite import make_scene
    dev = torch.device("cuda", 0)
    if not a.trees:
        a.trees = 64 * torch.cuda.get_device_properties(dev).multi_processor_count
    eng = MCTSEngine(_lib.ENV_HIGHWAY, a.trees, 5, a.episodes, a.horizon, 0.8, 10.0, device=dev)
    scenes = torch.from_numpy(np.stack([make_scene(i) for i in range(a.trees)])).to(dev)
    gens = [np.random.Generator(np.random.PCG64(np.random.SeedSequence(i))) for i in range(a.trees)]
    words = np.stack([pcg64_words(g) for g in gens])
    eng_small = MCTSEngine(_lib.ENV_HIGHWAY, a.trees, 5, 8, a.horizon, 0.8, 10.0, device=dev)
    eng_small.plan(scenes, words)
    eng_small.finish()                                     # warm-up launch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        eng.plan(scenes, words)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    plans, res, _ = eng.finish()
    env_steps = int(res[:, 2].sum())
    print(json.dumps({"metric": "MCTS episodes/sec on HighwayLite", "value": a.trees * a.episodes / (ms * 1e-3),
                      "unit": "episodes/s", "ms_per_step": ms, "env_steps_per_s": env_steps / (ms * 1e-3),
                      "config": {"workload": "C3: MCTS episodes=%d horizon=%d gamma 0.8, %d independent decisions"
                                             % (a.episodes, a.horizon, a.trees)},
                      "mean_nodes_per_tree": float(res[:, 0].mean())}))


if __name__ == "__main__":
    main()
