#!/usr/bin/env python
"""BRUE measurements: batch throughput (decisions/s, env steps/s) of b2_brue_plan on HighwayLite at the shipped
brue.json config (gamma 0.7, budget 200, horizon 6) and at budget 2000 / gamma 0.8, the mean number of rollouts per
decision, single-decision latency through the agent-level engine (one tree), and the CPU oracle's time per decision on
the same scenes.  One JSON line, with the GPU's name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.bench_mdp_gape import gpu_info, timed  # noqa: E402

# scripts/configs/DummyEnv/agents/brue.json of the reference (__class__ aside), and a larger budget
CONFIGS = (("brue_json_b200", {"budget": 200, "gamma": 0.7, "horizon": 6}),
           ("b2000_g0.8", {"budget": 2000, "gamma": 0.8}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="batch size (default: 64 decisions per SM)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-decisions", type=int, default=1, help="CPU oracle decisions to time per config")
    args = ap.parse_args()
    import torch
    from oracle import brue as oracle_brue
    from oracle import envs as oenvs
    from oracle import ref_loader
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.brue import BRUE
    from rl_agents_b200.engine.brue import BRUEEngine
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.envs.highway_lite import make_scene
    assert torch.cuda.is_available(), "bench_brue needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.trees or torch.cuda.get_device_properties(dev).multi_processor_count * 64
    scenes = torch.from_numpy(np.stack([make_scene(i) for i in range(n)])).to(dev)
    words = np.stack([pcg64_words(ref_loader.legacy_np_random(i)[0]) for i in range(n)])
    out = dict(gpu_info(), trees=n)
    for name, extra in CONFIGS:
        cfg = BRUE.default_config()
        BRUE.rec_update(cfg, extra)
        horizon = oracle_brue.brue_horizon(cfg, 5)

        def engine(trees):
            return BRUEEngine(_lib.ENV_HIGHWAY, trees, 5, cfg["budget"], horizon, cfg["gamma"], device=dev)
        eng = engine(n)
        ms = timed(lambda: eng.plan(scenes, words), args.reps)
        res = eng.result.cpu().numpy()
        one = engine(1)
        ms1 = timed(lambda: (one.plan(scenes[:1], words[:1]), one.finish()), args.reps)
        t0 = time.perf_counter()
        for i in range(args.oracle_decisions):
            oracle_brue.brue_plan(oenvs.LegacyStepEnv(oenvs.HighwayLite(seed=i)), cfg, ref_loader.legacy_np_random(i)[0])
        cpu_s = (time.perf_counter() - t0) / max(args.oracle_decisions, 1)
        out[name] = {"budget": cfg["budget"], "gamma": cfg["gamma"], "horizon": horizon,
                     "batch_ms": ms, "decisions_per_s": n / (ms * 1e-3),
                     "env_steps_per_s": float(res[:, 2].sum()) / (ms * 1e-3),
                     "mean_rollouts": float(res[:, 1].mean()), "mean_env_steps": float(res[:, 2].mean()),
                     "single_decision_ms": ms1, "cpu_oracle_s_per_decision": cpu_s,
                     "cpu_oracle_decisions_timed": args.oracle_decisions}
        del eng, one
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
