#!/usr/bin/env python
"""Budget sweep of closed-loop episodes on finite MDPs, in the shape of the reference's planners_evaluation.py:
run_batched_episodes(..., env="finite") for every finite-MDP planner on a seeded sparse garnet (S = 1000, A = 4, B = 3,
the garnet of bench_mdp_gape_stochastic.py) and on the same garnet made deterministic (its first successor), 8 448
episodes x 20 steps per planner and budget.  Per run: decisions/s (decisions taken over the host wall time of the
whole run, engine set-up included), the share of that time spent in b2_finite_step (CUDA events around each call),
and the mean return with its standard error.  Each run follows a one-step warm-up run of the same configuration.
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

from bench_mdp_gape import gpu_info  # noqa: E402

KL = {"upper_bound": {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)"},
      "continuation_type": "uniform"}
BUDGETS = (100, 400)
# planner -> (modes, [(budget, keywords)]).  MDP-GapE keeps up to the garnet's 3 next states per chance node (with the
# default 1 it raises the reference's placeholder ValueError on the sparse garnet).  Sparse sampling and PlaTyPOOS are
# swept over their horizon (PlaTyPOOS's h_max from a budget of 400 over 4 actions is 0).  VI runs 100 iterations.
SWEEP = {
    "opd": (("deterministic",), [(b, {}) for b in BUDGETS]),
    "gbop": (("deterministic",), [(b, {}) for b in BUDGETS]),
    "gbopd": (("deterministic",), [(b, {}) for b in BUDGETS]),
    "brue": (("deterministic",), [(b, {}) for b in BUDGETS]),
    "mcts": (("deterministic", "sparse"), [(b, {}) for b in BUDGETS]),
    "olop": (("deterministic", "sparse"), [(b, KL) for b in BUDGETS]),
    "mdp_gape": (("deterministic", "sparse"), [(b, {"max_next_states_count": 3}) for b in BUDGETS]),
    "mcts_dpw": (("deterministic", "sparse"), [(b, {}) for b in BUDGETS]),
    "sparse_sampling": (("deterministic", "sparse"), [(0, {"horizon": h, "C": 3}) for h in (2, 3)]),
    "platypoos": (("deterministic", "sparse"), [(0, {"horizon": h}) for h in (3, 4)]),
    "vi": (("deterministic", "sparse"), [(100, {})]),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--episodes", type=int, default=8448)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--gamma", type=float, default=0.8)
    ap.add_argument("--planners", default=",".join(SWEEP))
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    from oracle import envs as oenvs
    from rl_agents_b200.envs import FiniteMDPEnv
    from rl_agents_b200.evaluation import run_batched_episodes
    assert torch.cuda.is_available(), "bench_eval_finite needs a GPU"
    P, N, R = oenvs.garnet(1000, 4, 3, seed=0)
    envs = {"sparse": FiniteMDPEnv(P, R, None, mode="sparse", nxt=N), "deterministic": FiniteMDPEnv(N[:, :, 0], R)}
    starts = np.arange(args.episodes) % 1000
    out = dict(gpu_info(), episodes=args.episodes, steps=args.steps, gamma=args.gamma,
               mdp="garnet(1000, 4, 3, seed=0)", runs=[])
    for planner in args.planners.split(","):
        modes, configs = SWEEP[planner]
        for mode in modes:
            for budget, kw in configs:
                def run(steps):
                    return run_batched_episodes(planner, range(args.episodes), budget, args.gamma, max_steps=steps,
                                                env="finite", mdp=envs[mode], start_states=starts, env_seed=0, **kw)
                run(1)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = run(args.steps)
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                decisions = int(res["lengths"].sum())
                ret = res["returns"]
                out["runs"].append({"planner": planner, "mode": mode, "budget": budget, **kw,
                                    "decisions_per_s": decisions / wall, "wall_s": wall,
                                    "step_share": res["step_ms"] * res["actions"].shape[1] * 1e-3 / wall,
                                    "decision_ms": res["decision_ms"], "step_ms": res["step_ms"],
                                    "mean_return": float(ret.mean()),
                                    "return_stderr": float(ret.std(ddof=1) / np.sqrt(ret.size))})
                print(json.dumps(out["runs"][-1]), file=sys.stderr)
                del res
                torch.cuda.empty_cache()
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
