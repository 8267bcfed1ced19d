#!/usr/bin/env python
"""MCTS-DPW measurements: batch throughput (decisions/s, env steps/s) of b2_mcts_dpw_plan on HighwayLite at
MCTSDPWAgent's default config (budget 100, gamma 0.95: 5 runs of horizon 16) and at budget 1000, and on a seeded
stochastic garnet (S = 1000, A = 4, B = 3, "sparse" mode) at budget 1000 in closed loop; single-decision latency
through the agent-level engine (one tree); and the CPU oracle's time per decision on the same inputs.  One JSON line,
with the GPU's name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.bench_mdp_gape import gpu_info, timed  # noqa: E402

CONFIGS = (("highway_default", "highway", {}),
           ("highway_budget1000", "highway", {"budget": 1000}),
           ("garnet_budget1000_closed_loop", "garnet", {"budget": 1000, "closed_loop": True}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="batch size (default: 64 decisions per SM)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-decisions", type=int, default=1, help="CPU oracle decisions to time per config")
    args = ap.parse_args()
    import torch
    from oracle import envs as oenvs
    from oracle import mcts_dpw as oracle_dpw
    from oracle import ref_loader
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPWAgent
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.engine.mcts_dpw import MCTSDPWEngine
    from rl_agents_b200.envs.highway_lite import make_scene
    assert torch.cuda.is_available(), "bench_mcts_dpw needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.trees or torch.cuda.get_device_properties(dev).multi_processor_count * 64
    P, N, R = oenvs.garnet(1000, 4, 3, seed=0)
    garnet = oenvs.FiniteMDPLite(P, R, mode="sparse", nxt=N)
    roots = {"garnet": torch.arange(n, dtype=torch.int32, device=dev) % 1000,
             "highway": torch.from_numpy(np.stack([make_scene(i) for i in range(n)])).to(dev)}
    words = np.stack([pcg64_words(ref_loader.legacy_np_random(i)[0]) for i in range(n)])
    out = dict(gpu_info(), trees=n, garnet={"states": 1000, "actions": 4, "successors": 3, "seed": 0})
    for name, env_name, config in CONFIGS:
        finite = env_name == "garnet"
        cfg = MCTSDPWAgent(garnet, dict(config)).planner.config          # the completed planner config

        def engine(trees):
            return MCTSDPWEngine(_lib.ENV_FINITE if finite else _lib.ENV_HIGHWAY, trees, 4 if finite else 5,
                                 cfg["episodes"], cfg["horizon"], cfg["gamma"], cfg["temperature"], cfg["k_action"],
                                 cfg["alpha_action"], cfg["k_state"], cfg["alpha_state"], closed_loop=cfg["closed_loop"],
                                 mdp=garnet.mdp if finite else None, device=dev)
        eng = engine(n)
        ms = timed(lambda: eng.plan(roots[env_name], words), args.reps)
        res = eng.result.cpu().numpy()
        assert (res[:, 4] == 0).all()
        one = engine(1)
        ms1 = timed(lambda: (one.plan(roots[env_name][:1], words[:1]), one.finish()), args.reps)
        t0 = time.perf_counter()
        for i in range(args.oracle_decisions):
            if finite:
                env = oenvs.FiniteMDPLite(P, R, mode="sparse", nxt=N, state=i % 1000)
            else:
                env = oenvs.HighwayLite(oenvs.HighwayLiteState.unpack(make_scene(i)))
            oracle_dpw.mcts_dpw_plan(env, cfg, ref_loader.legacy_np_random(i)[0])
        cpu_s = (time.perf_counter() - t0) / max(args.oracle_decisions, 1)
        out[name] = dict(config, episodes=cfg["episodes"], horizon=cfg["horizon"], batch_ms=ms,
                         decisions_per_s=n / (ms * 1e-3),
                         env_steps_per_s=float(res[:, 2].astype(np.int64).sum()) / (ms * 1e-3),
                         mean_nodes=float(res[:, 0].mean()), single_decision_ms=ms1, cpu_oracle_s_per_decision=cpu_s,
                         cpu_oracle_decisions_timed=args.oracle_decisions)
        del eng, one
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
