#!/usr/bin/env python
"""OLOP on a stochastic finite MDP: batch throughput (decisions/s) of b2_olop_plan_sampled on a seeded sparse garnet
(S = 1000, A = 4, B = 3 successors per row) at the shipped FiniteMDPEnv/agents/kl-olop.json and at budget 2000
(gamma 0.8), beside the same garnet made deterministic (its first successor) through b2_olop_plan, which shows what the
per-episode env seeding and the per-step draws cost; single-decision latency; and the CPU oracle's time per decision.
One JSON line, with the GPU's name and power limit read in the same run."""
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

# scripts/configs/FiniteMDPEnv/agents/kl-olop.json of the reference (`__class__` aside; OLOP ignores max_depth and
# lazy_tree_construction)
KL_OLOP_JSON = {"gamma": 0.9, "budget": 100, "max_depth": 2,
                "upper_bound": {"type": "kullback-leibler", "time": "global"}, "lazy_tree_construction": True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="batch size (default: 64 decisions per SM)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-decisions", type=int, default=2, help="CPU oracle decisions to time per config")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    from oracle import envs as oenvs
    from oracle import planners
    from oracle import ref_loader
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mcts import allocation
    from rl_agents_b200.agents.tree_search.olop import OLOP
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.engine.olop import OLOPEngine
    assert torch.cuda.is_available(), "bench_olop_stochastic needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.trees or torch.cuda.get_device_properties(dev).multi_processor_count * 64
    P, N, R = oenvs.garnet(1000, 4, 3, seed=0)
    sparse = oenvs.FiniteMDPLite(P, R, None, mode="sparse", nxt=N)
    det = oenvs.FiniteMDPLite(N[:, :, 0], R, None)
    roots = torch.arange(n, dtype=torch.int32, device=dev) % 1000
    words = np.stack([pcg64_words(ref_loader.legacy_np_random(i)[0]) for i in range(n)])
    out = dict(gpu_info(), trees=n, mdp="garnet(1000, 4, 3, seed=0)")
    for name, extra in (("kl_olop_json", {}), ("b2000", {"budget": 2000, "gamma": 0.8})):
        cfg = OLOP.default_config()
        OLOP.rec_update(cfg, dict(KL_OLOP_JSON, **extra))
        episodes, horizon = allocation(max(4, cfg["budget"]), cfg["gamma"])
        row = {"budget": cfg["budget"], "gamma": cfg["gamma"], "episodes": episodes, "horizon": horizon}
        for mode, env in (("sparse", sparse), ("deterministic", det)):
            def engine(trees):
                return OLOPEngine(_lib.ENV_FINITE, trees, 4, episodes, horizon, cfg["gamma"], cfg["upper_bound"],
                                  cfg["continuation_type"], mdp=env.mdp, device=dev)
            eng = engine(n)
            assert eng.sampled == (mode == "sparse")
            ms = timed(lambda: eng.plan(roots, words), args.reps)
            res = eng.result.cpu().numpy()
            assert (res[:, 2] == 0).all()
            one = engine(1)
            ms1 = timed(lambda: (one.plan(roots[:1], words[:1]), one.finish()), args.reps)
            row[mode] = {"batch_ms": ms, "decisions_per_s": n / (ms * 1e-3),
                         "env_steps_per_s": n * episodes * horizon / (ms * 1e-3), "single_decision_ms": ms1}
            del eng, one
            torch.cuda.empty_cache()
        t0 = time.perf_counter()
        for i in range(args.oracle_decisions):
            sparse.mdp.state = i
            planners.olop_plan(oenvs.LegacyStepEnv(sparse), cfg["budget"], cfg["gamma"],
                               ref_loader.legacy_np_random(i)[0], upper_bound=cfg["upper_bound"],
                               continuation_type=cfg["continuation_type"])
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
