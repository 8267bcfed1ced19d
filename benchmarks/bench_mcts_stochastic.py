#!/usr/bin/env python
"""MCTS on a stochastic finite MDP: batch throughput (decisions/s) of b2_mcts_plan_sampled on a seeded sparse garnet
(S = 1000, A = 4, B = 3 successors per row) at MCTSAgent's default budget (100) and at budget 2000 (gamma 0.9), beside
the same garnet made deterministic (its first successor) through b2_mcts_plan, which shows what the per-episode reload
of the env generator's words and the per-step draws cost; single-decision latency; one decision of the wavefront
kernel (b2_mcts_plan_wave_sampled, waves of 64 episodes); and the CPU oracle's time per decision.  One JSON line, with
the GPU's name and power limit read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from bench_mdp_gape import gpu_info, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="batch size (default: 64 decisions per SM)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--width", type=int, default=64, help="wavefront episodes per wave")
    ap.add_argument("--oracle-decisions", type=int, default=2, help="CPU oracle decisions to time per config")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    from oracle import envs as oenvs
    from oracle import planners
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mcts import allocation
    from rl_agents_b200.engine.mcts import MCTSEngine, MCTSWaveEngine, pcg64_words
    assert torch.cuda.is_available(), "bench_mcts_stochastic needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.trees or torch.cuda.get_device_properties(dev).multi_processor_count * 64
    P, N, R = oenvs.garnet(1000, 4, 3, seed=0)
    sparse = oenvs.FiniteMDPLite(P, R, None, mode="sparse", nxt=N, seed=1)
    det = oenvs.FiniteMDPLite(N[:, :, 0], R, None)
    roots = torch.arange(n, dtype=torch.int32, device=dev) % 1000

    def gen(i):
        return np.random.Generator(np.random.PCG64(np.random.SeedSequence(i)))
    words = np.stack([pcg64_words(gen(i)) for i in range(n)])
    env_words = np.stack([pcg64_words(gen(10 ** 6 + i)) for i in range(n)])
    out = dict(gpu_info(), trees=n, mdp="garnet(1000, 4, 3, seed=0)")
    for name, budget, gamma in (("b100_g0.8", 100, 0.8), ("b2000_g0.9", 2000, 0.9)):
        episodes, horizon = allocation(budget, gamma)
        temperature = 2 / (1 - 0.8)           # MCTS.default_config: from the default gamma (mcts.py:120-127)
        row = {"budget": budget, "gamma": gamma, "episodes": episodes, "horizon": horizon}
        for mode, env in (("sparse", sparse), ("deterministic", det)):
            def engine(trees):
                return MCTSEngine(_lib.ENV_FINITE, trees, 4, episodes, horizon, gamma, temperature, mdp=env.mdp,
                                  device=dev)
            eng = engine(n)
            assert eng.sampled == (mode == "sparse")
            ms = timed(lambda: eng.plan(roots, words, None, env_words), args.reps)
            res = eng.result.cpu().numpy()
            assert mode == "deterministic" or (res[:, 3] == 0).all()
            one = engine(1)
            ms1 = timed(lambda: (one.plan(roots[:1], words[:1], None, env_words[:1]), one.finish()), args.reps)
            row[mode] = {"batch_ms": ms, "decisions_per_s": n / (ms * 1e-3),
                         "env_steps_per_s": float(res[:, 2].sum()) / (ms * 1e-3), "single_decision_ms": ms1}
            del eng, one
            torch.cuda.empty_cache()
        row["sparse_over_deterministic_batch_ms"] = row["sparse"]["batch_ms"] / row["deterministic"]["batch_ms"]
        weng = MCTSWaveEngine(_lib.ENV_FINITE, 4, episodes, horizon, gamma, temperature, args.width, mdp=sparse.mdp,
                              device=dev)
        root1 = roots[:1].contiguous()
        row["sparse"]["wavefront_decision_ms"] = timed(lambda: (weng.plan(root1, 7, env_words[0]), weng.finish()),
                                                       args.reps)
        row["sparse"]["wavefront_width"] = weng.width
        del weng
        t0 = time.perf_counter()
        for i in range(args.oracle_decisions):
            sparse.mdp.state = i
            planners.mcts_plan(sparse, episodes, horizon, gamma, temperature, gen(i))
        sparse.mdp.state = 0
        row["sparse"]["cpu_oracle_s_per_decision"] = (time.perf_counter() - t0) / max(args.oracle_decisions, 1)
        row["sparse"]["cpu_oracle_decisions_timed"] = args.oracle_decisions
        out[name] = row
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
