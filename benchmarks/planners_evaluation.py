#!/usr/bin/env python
"""Budget sweep of the device planners on HighwayLite (closed loop, batched episodes); one CSV row
per (planner, budget): mean return, crash rate, mean episode length, ms per batched decision.
Planners: opd, mcts, olop, mdp_gape, brue, vi (ValueIterationAgent on the scenes' TTC-grid MDPs; its "budget" is the
agent's `iterations`, e.g. `--planners vi --budgets 10 --gamma 1.0` = the reference's shipped highway config)."""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--planners", default="opd,mcts,olop")
    ap.add_argument("--budgets", default="75,300,1000,3000")
    ap.add_argument("--episodes", type=int, default=256)
    ap.add_argument("--gamma", type=float, default=0.8)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--step-strategy", default="reset",
                    help='"subtree": MCTS keeps the sub-tree under the played action (the other planners reset)')
    a = ap.parse_args()
    from rl_agents_b200.evaluation import run_batched_episodes
    print("planner,budget,episodes,mean_return,crash_rate,mean_length,ms_per_batched_decision")
    for planner in a.planners.split(","):
        for budget in [int(b) for b in a.budgets.split(",")]:
            out = run_batched_episodes(planner, list(range(a.episodes)), budget, a.gamma, max_steps=a.steps,
                                       step_strategy=a.step_strategy)
            print("%s,%d,%d,%.4f,%.4f,%.2f,%.2f" % (planner, budget, a.episodes, out["returns"].mean(),
                                                    out["crashed"].mean(), out["lengths"].mean(), out["decision_ms"]))
            sys.stdout.flush()


if __name__ == "__main__":
    main()
