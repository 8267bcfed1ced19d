#!/usr/bin/env python
"""MDP-GapE on a stochastic finite MDP: batch throughput (decisions/s) of b2_mdp_gape_plan_sampled on a seeded sparse
garnet (S = 1000, A = 4, B = 3 successors per row, max_next_states_count 3) at mdp-gape.json and at budget 2000,
beside the same garnet made deterministic (its first successor) through b2_mdp_gape_plan, which shows what the
several-next-state backups with their Newton solves cost; the mean number of episodes run; single-decision latency;
and the CPU oracle's time per decision.  One JSON line, with the GPU's name and power limit read in the same run.
mdp-gape.json sets max_next_states_count 2, which a garnet with three successors per row overflows (the reference's
ValueError), so it runs here at 3."""
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

# scripts/configs/DummyEnv/agents/mdp-gape.json of the reference (`__class__` aside; its "threshold_transition" key
# is a typo the agent ignores), with max_next_states_count 3
MDP_GAPE_JSON = {"gamma": 0.7, "budget": 200, "max_depth": 4, "accuracy": 0.0, "confidence": 1.0,
                 "max_next_states_count": 3,
                 "upper_bound": {"type": "kullback-leibler", "time": "global", "threshold": "1*np.log(time)",
                                 "threshold_transition": "0.1*np.log(time)", "max_next_states_count": 1},
                 "continuation_type": "uniform"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="batch size (default: 64 decisions per SM)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-decisions", type=int, default=2, help="CPU oracle decisions to time per config")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    from oracle import envs as oenvs
    from oracle import mdp_gape_stochastic as oracle_gape
    from oracle import ref_loader
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapE, budget_allocation
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.engine.mdp_gape import MDPGapEEngine
    assert torch.cuda.is_available(), "bench_mdp_gape_stochastic needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.trees or torch.cuda.get_device_properties(dev).multi_processor_count * 64
    P, N, R = oenvs.garnet(1000, 4, 3, seed=0)
    sparse = oenvs.FiniteMDPLite(P, R, None, mode="sparse", nxt=N)
    det = oenvs.FiniteMDPLite(N[:, :, 0], R, None)
    roots = torch.arange(n, dtype=torch.int32, device=dev) % 1000
    words = np.stack([pcg64_words(ref_loader.legacy_np_random(i)[0]) for i in range(n)])
    out = dict(gpu_info(), trees=n, mdp="garnet(1000, 4, 3, seed=0)")
    for name, extra in (("mdp_gape_json", {}), ("b2000", {"budget": 2000, "gamma": 0.8, "accuracy": 1.0,
                                                           "confidence": 0.9})):
        cfg = MDPGapE.default_config()
        MDPGapE.rec_update(cfg, dict(MDP_GAPE_JSON, **extra))
        episodes, horizon = budget_allocation(cfg, 4)
        row = {"budget": cfg["budget"], "episodes_cap": episodes + 2, "horizon": horizon}
        for mode, env in (("sparse", sparse), ("deterministic", det)):
            def engine(trees):
                return MDPGapEEngine(_lib.ENV_FINITE, trees, 4, episodes, horizon, cfg["gamma"], cfg["upper_bound"],
                                     cfg["accuracy"], cfg["confidence"], cfg["continuation_type"],
                                     cfg["max_next_states_count"], mdp=env.mdp, device=dev)
            eng = engine(n)
            ms = timed(lambda: eng.plan(roots, words), args.reps)
            res = eng.result.cpu().numpy()
            assert (res[:, 2] == 0).all()
            one = engine(1)
            ms1 = timed(lambda: (one.plan(roots[:1], words[:1]), one.finish()), args.reps)
            row[mode] = {"batch_ms": ms, "decisions_per_s": n / (ms * 1e-3),
                         "mean_episodes_run": float(res[:, 1].mean()),
                         "env_steps_per_s": float(res[:, 1].sum()) * horizon / (ms * 1e-3),
                         "single_decision_ms": ms1}
            del eng, one
            torch.cuda.empty_cache()
        t0 = time.perf_counter()
        for i in range(args.oracle_decisions):
            sparse.mdp.state = i
            oracle_gape.mdp_gape_plan(oenvs.LegacyStepEnv(sparse), cfg, ref_loader.legacy_np_random(i)[0])
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
