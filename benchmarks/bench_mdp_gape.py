#!/usr/bin/env python
"""MDP-GapE measurements: batch throughput (decisions/s) of b2_mdp_gape_plan on HighwayLite at the shipped
baseline.json config (budget 100) and at budget 1000, the mean number of episodes the stopping rule lets run,
single-decision latency through the agent-level engine (one tree), and the CPU oracle's time per decision on the
same scenes.  One JSON line, with the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# scripts/configs/HighwayEnv/agents/MDPGapEAgent/baseline.json of the reference (env_preprocessors / __class__ aside)
BASELINE = {"gamma": 0.8, "budget": 100, "accuracy": 0.1, "confidence": 1, "max_next_states_count": 1,
            "upper_bound": {"type": "kullback-leibler", "time": "global", "threshold": "1*np.log(time)"},
            "continuation_type": "uniform", "step_strategy": "reset"}


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, power = [s.strip() for s in q.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception:
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="batch size (default: 64 decisions per SM)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-decisions", type=int, default=2, help="CPU oracle decisions to time per config")
    args = ap.parse_args()
    import torch
    from oracle import envs as oenvs
    from oracle import mdp_gape as oracle_gape
    from oracle import ref_loader
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapE, budget_allocation
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.engine.mdp_gape import MDPGapEEngine
    from rl_agents_b200.envs.highway_lite import make_scene
    assert torch.cuda.is_available(), "bench_mdp_gape needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.trees or torch.cuda.get_device_properties(dev).multi_processor_count * 64
    scenes = torch.from_numpy(np.stack([make_scene(i) for i in range(n)])).to(dev)
    words = np.stack([pcg64_words(ref_loader.legacy_np_random(i)[0]) for i in range(n)])
    out = dict(gpu_info(), trees=n)
    for name, extra in (("baseline_b100", {}), ("b1000", {"budget": 1000})):
        cfg = MDPGapE.default_config()
        MDPGapE.rec_update(cfg, dict(BASELINE, **extra))
        episodes, horizon = budget_allocation(cfg, 5)

        def engine(trees):
            return MDPGapEEngine(_lib.ENV_HIGHWAY, trees, 5, episodes, horizon, cfg["gamma"], cfg["upper_bound"],
                                 cfg["accuracy"], cfg["confidence"], cfg["continuation_type"],
                                 cfg["max_next_states_count"], device=dev)
        eng = engine(n)
        ms = timed(lambda: eng.plan(scenes, words), args.reps)
        res = eng.result.cpu().numpy()
        one = engine(1)
        ms1 = timed(lambda: (one.plan(scenes[:1], words[:1]), one.finish()), args.reps)
        t0 = time.perf_counter()
        for i in range(args.oracle_decisions):
            oracle_gape.mdp_gape_plan(oenvs.LegacyStepEnv(oenvs.HighwayLite(seed=i)), cfg,
                                      ref_loader.legacy_np_random(i)[0])
        cpu_s = (time.perf_counter() - t0) / max(args.oracle_decisions, 1)
        out[name] = {"budget": cfg["budget"], "episodes_cap": episodes + 2, "horizon": horizon,
                     "batch_ms": ms, "decisions_per_s": n / (ms * 1e-3),
                     "mean_episodes_run": float(res[:, 1].mean()),
                     "stopped_early_fraction": float((res[:, 1] < episodes + 2).mean()),
                     "env_steps_per_s": float(res[:, 1].sum()) * horizon / (ms * 1e-3),
                     "single_decision_ms": ms1, "cpu_oracle_s_per_decision": cpu_s,
                     "cpu_oracle_decisions_timed": args.oracle_decisions}
        del eng, one
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
