#!/usr/bin/env python
"""Time of ONE sparse-sampling decision: the depth-first lane kernel (b2_sparse_sampling_plan, one 16-lane group or one
lane) against the level-synchronous kernel (b2_sparse_sampling_plan_levels, the whole GPU), on HighwayLite at C 3,
gamma 0.7, horizons 1..6, and on a seeded deterministic garnet (S = 1000, A = 4) at C 3, gamma 0.7, horizons 1..6;
then one agent-level SparseSampling.plan() per env at the shipped sparse_sampling.json config (horizon 3, C 3), with
the engine the agent selects and with the lane engine.  Engine times are CUDA events around repeated plan() calls
after a warm-up call (each call uploads the planner's stream and launches the kernel, as an agent's decision does);
both kernels' plans, result words and streams are checked equal on every shape.  One JSON line, with the GPU's name
and power limit."""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.bench_mdp_gape import gpu_info  # noqa: E402

C, GAMMA = 3, 0.7
HORIZONS = (1, 2, 3, 4, 5, 6)


def event_ms(fn, window_s):
    """Mean over a window of about window_s seconds (at least 3 calls), after one warm-up call."""
    import torch
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    reps = max(3, min(500, int(math.ceil(window_s / max(time.perf_counter() - t0, 1e-6)))))
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps, reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=float, default=0.3, help="seconds of timed calls per shape and kernel")
    args = ap.parse_args()
    import torch
    from oracle import envs as oenvs
    from oracle import ref_loader
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search import sparse_sampling as ssmod
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.engine.sparse_sampling import SparseSamplingEngine, SparseSamplingLevelEngine
    from rl_agents_b200.envs import FiniteMDPEnv, HighwayLiteEnv
    from rl_agents_b200.envs.highway_lite import make_scene
    assert torch.cuda.is_available(), "bench_sparse_sampling_levels needs a GPU"
    dev = torch.device("cuda", 0)
    T, R = oenvs.garnet(1000, 4, 1, seed=0, deterministic=True)
    garnet = oenvs.FiniteMDPLite(T, R, mode="deterministic")
    envs = {"highway": (_lib.ENV_HIGHWAY, 5, None, torch.from_numpy(make_scene(0).reshape(1, -1).astype(np.int32)).to(dev)),
            "garnet": (_lib.ENV_FINITE, 4, garnet.mdp, torch.zeros(1, dtype=torch.int32, device=dev))}
    words = pcg64_words(ref_loader.legacy_np_random(0)[0]).reshape(1, -1)

    def agent_env(name):
        return HighwayLiteEnv(seed=0) if name == "highway" else FiniteMDPEnv(T, R, np.zeros(1000, dtype=bool))
    out = dict(gpu_info(), C=C, gamma=GAMMA, garnet={"states": 1000, "actions": 4, "seed": 0, "mode": "deterministic"},
               highway_scene="make_scene(0)", single_decision={})
    for name, (kind, A, mdp, root) in envs.items():
        rows = {}
        for H in HORIZONS:
            row = {}
            outs = []
            for label, cls in (("lane", SparseSamplingEngine), ("level", SparseSamplingLevelEngine)):
                eng = cls(kind, 1, A, H, C, GAMMA, mdp=mdp, device=dev)
                ms, reps = event_ms(lambda: eng.plan(root, words), args.window)
                plans, res, w = eng.finish()
                outs.append((plans, res.tolist(), w.tolist(), eng.root_q.cpu().numpy().tobytes()))
                row[label + "_ms"], row[label + "_reps"] = ms, reps
                row["chance_nodes"] = int(res[0, 1])
                del eng
            assert outs[0] == outs[1], (name, H)
            row["speedup"] = row["lane_ms"] / row["level_ms"]
            row["level_engine_selected"] = ssmod.use_level_engine(ssmod.describe(agent_env(name)), H, C)
            rows["h%d" % H] = row
            torch.cuda.empty_cache()
        out["single_decision"][name] = rows

    # agent level: one SparseSampling.plan() at the shipped config, with the selected engine and on the lane engine
    out["agent_plan_ms"] = {}
    for name in ("highway", "garnet"):
        res = {}
        for label, rule in (("selected", ssmod.use_level_engine), ("lane", lambda *a: False)):
            ssmod.use_level_engine, saved = rule, ssmod.use_level_engine
            try:
                env = agent_env(name)
                agent = ssmod.SparseSamplingAgent(env, {"gamma": GAMMA, "horizon": 3, "C": C})
                agent.seed(0)
                obs = None if name == "highway" else 0
                agent.plan(obs)
                ts = []
                for _ in range(20):
                    t0 = time.perf_counter()
                    agent.plan(obs)                       # returns host data: ends in a device synchronise
                    ts.append(time.perf_counter() - t0)
                res[label + "_ms"] = float(np.median(ts)) * 1e3
                res[label + "_engine"] = type(agent.planner.engine).__name__
            finally:
                ssmod.use_level_engine = saved
        out["agent_plan_ms"][name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
