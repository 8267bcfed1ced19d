#!/usr/bin/env python
"""PlaTyPOOS measurements: batch throughput (decisions/s, env steps/s) of b2_platypoos_plan on HighwayLite at the
shipped baseline.json (budget 2500, gamma 0.9: h_max 2) and at budgets 50 000 and 200 000 (gamma 0.9), and on a
deterministic garnet (S = 1000, A = 4) at budget 200 000; single-decision latency through a one-tree engine; and the CPU
oracle's time per decision on the same inputs.  One JSON line, with the GPU's name and power limit; --out also writes it
to a file."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.bench_mdp_gape import gpu_info, timed  # noqa: E402

CONFIGS = (("highway_baseline", "highway", 2500),
           ("highway_budget50000", "highway", 50000),
           ("highway_budget200000", "highway", 200000),
           ("garnet_budget200000", "garnet", 200000))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=0, help="batch size (default: 64 decisions per SM)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-decisions", type=int, default=1, help="CPU oracle decisions to time per config")
    ap.add_argument("--oracle-max-budget", type=int, default=50000,
                    help="skip the CPU oracle above this budget on HighwayLite (the reference takes minutes there)")
    ap.add_argument("--out", default="", help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    from oracle import envs as oenvs
    from oracle import platypoos as oracle_pl
    from oracle import ref_loader
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.engine.platypoos import PlaTyPOOSEngine, horizon_of
    from rl_agents_b200.envs.highway_lite import make_scene
    assert torch.cuda.is_available(), "bench_platypoos needs a GPU"
    dev = torch.device("cuda", 0)
    n = args.trees or torch.cuda.get_device_properties(dev).multi_processor_count * 64
    T, R = oenvs.garnet(1000, 4, 1, seed=0, deterministic=True)
    garnet = oenvs.FiniteMDPLite(T, R)
    roots = {"garnet": torch.arange(n, dtype=torch.int32, device=dev) % 1000,
             "highway": torch.from_numpy(np.stack([make_scene(i) for i in range(n)])).to(dev)}
    words = np.stack([pcg64_words(ref_loader.legacy_np_random(i)[0]) for i in range(n)])
    out = dict(gpu_info(), trees=n, gamma=0.9, garnet={"states": 1000, "actions": 4, "deterministic": True, "seed": 0})
    for name, env_name, budget in CONFIGS:
        finite = env_name == "garnet"
        n_actions = 4 if finite else 5
        horizon = horizon_of(budget, n_actions)

        def engine(trees):
            return PlaTyPOOSEngine(_lib.ENV_FINITE if finite else _lib.ENV_HIGHWAY, trees, n_actions, horizon, 0.9,
                                   mdp=garnet.mdp if finite else None, device=dev)
        eng = engine(n)
        ms = timed(lambda: eng.plan(roots[env_name], words), args.reps)
        res = eng.result.cpu().numpy()
        assert (res[:, 3] == 0).all()
        one = engine(1)
        ms1 = timed(lambda: (one.plan(roots[env_name][:1], words[:1]), one.finish()), args.reps)
        cpu_s = None
        if finite or budget <= args.oracle_max_budget:
            t0 = time.perf_counter()
            for i in range(args.oracle_decisions):
                if finite:
                    env = oenvs.FiniteMDPLite(T, R, state=i % 1000)
                else:
                    env = oenvs.HighwayLite(oenvs.HighwayLiteState.unpack(make_scene(i)))
                oracle_pl.platypoos_plan(env, {"horizon": horizon, "gamma": 0.9, "step_strategy": "reset"},
                                         ref_loader.legacy_np_random(i)[0])
            cpu_s = (time.perf_counter() - t0) / max(args.oracle_decisions, 1)
        out[name] = dict(budget=budget, horizon=horizon, batch_ms=ms, decisions_per_s=n / (ms * 1e-3),
                         env_steps_per_s=float(res[:, 5].astype(np.int64).sum()) / (ms * 1e-3),
                         mean_nodes=float(res[:, 0].mean()), max_nodes=int(res[:, 0].max()),
                         mean_openings=float(res[:, 1].mean()), mean_plan_length=float(res[:, 2].mean()),
                         node_capacity=eng.node_capacity, layer_capacity=eng.layer_capacity,
                         single_decision_ms=ms1, cpu_oracle_s_per_decision=cpu_s,
                         cpu_oracle_decisions_timed=args.oracle_decisions if cpu_s is not None else 0)
        del eng, one
        torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
