#!/usr/bin/env python
"""Sparse-sampling measurements: batch throughput (decisions/s, samples/s) of b2_sparse_sampling_plan on a seeded
"sparse" garnet (S = 1000, A = 4, B = 3) at the shipped sparse_sampling.json config (gamma 0.7, horizon 3, C 3) and at
horizon 5, C 3, and on HighwayLite at the shipped config; single-decision latency through the agent-level engine (one
tree, no tree dump); and the CPU oracle's time per decision on the same inputs.  One JSON line, with the GPU's name
and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.bench_mdp_gape import gpu_info, timed  # noqa: E402

# scripts/configs/FiniteMDPEnv/agents/sparse_sampling.json of the reference (__class__ aside), and a deeper search
CONFIGS = (("garnet_shipped_h3_c3", "garnet", {"gamma": 0.7, "horizon": 3, "C": 3}),
           ("garnet_h5_c3", "garnet", {"gamma": 0.7, "horizon": 5, "C": 3}),
           ("highway_shipped_h3_c3", "highway", {"gamma": 0.7, "horizon": 3, "C": 3}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="batch size (default: 64 decisions per SM)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-decisions", type=int, default=1, help="CPU oracle decisions to time per config")
    args = ap.parse_args()
    import torch
    from oracle import envs as oenvs
    from oracle import ref_loader
    from oracle import sparse_sampling as oracle_ss
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.engine.sparse_sampling import SparseSamplingEngine
    from rl_agents_b200.envs.highway_lite import make_scene
    assert torch.cuda.is_available(), "bench_sparse_sampling needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.trees or torch.cuda.get_device_properties(dev).multi_processor_count * 64
    P, N, R = oenvs.garnet(1000, 4, 3, seed=0)
    garnet = oenvs.FiniteMDPLite(P, R, mode="sparse", nxt=N)
    roots = {"garnet": torch.arange(n, dtype=torch.int32, device=dev) % 1000,
             "highway": torch.from_numpy(np.stack([make_scene(i) for i in range(n)])).to(dev)}
    words = np.stack([pcg64_words(ref_loader.legacy_np_random(i)[0]) for i in range(n)])
    out = dict(gpu_info(), trees=n, garnet={"states": 1000, "actions": 4, "successors": 3, "seed": 0})
    for name, env_name, cfg in CONFIGS:
        finite = env_name == "garnet"

        def engine(trees):
            return SparseSamplingEngine(_lib.ENV_FINITE if finite else _lib.ENV_HIGHWAY, trees, 4 if finite else 5,
                                        cfg["horizon"], cfg["C"], cfg["gamma"], mdp=garnet.mdp if finite else None,
                                        device=dev)
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
            oracle_ss.sparse_sampling_plan(oenvs.LegacyStepEnv(env), cfg, ref_loader.legacy_np_random(i)[0])
        cpu_s = (time.perf_counter() - t0) / max(args.oracle_decisions, 1)
        out[name] = dict(cfg, batch_ms=ms, decisions_per_s=n / (ms * 1e-3),
                         samples_per_s=float(res[:, 2].astype(np.int64).sum()) / (ms * 1e-3),
                         mean_nodes=float(res[:, 0].mean()), mean_chance_nodes=float(res[:, 1].mean()),
                         single_decision_ms=ms1, cpu_oracle_s_per_decision=cpu_s,
                         cpu_oracle_decisions_timed=args.oracle_decisions)
        del eng, one
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
