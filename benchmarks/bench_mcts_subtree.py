#!/usr/bin/env python
"""MCTS with step_strategy "subtree" (the reference's step-strategy benchmark, benchmark_step_strategy.json, at batch
scale).  One JSON line, with the GPU's name and power limit read in the same run:

- `reroot_kernel`: b2_mcts_reroot over 8 448 trees of a first decision (HighwayLite at MCTSAgent's default budget 100
  and at budget 2000, gamma 0.8, and the seeded sparse garnet of bench_mcts_stochastic.py at budget 100, gamma 0.8 and
  2000, gamma 0.9), every tree re-rooted at its planned action into a second arena: CUDA events over many launches
  after a warm-up launch, and the bytes the kernel moves (68 per kept node: five source fields read, the node's source
  index read back, six destination fields and the child's source index written) against the 3.35 TB/s data-sheet HBM
  peak.
- `closed_loop`: run_batched_episodes("mcts", ...) over 8 448 episodes x 20 steps for "reset" and "subtree" on the
  same shapes: decisions/s over the host wall time of each run (engine set-up included, after a one-step warm-up run
  of the same configuration), mean return with its standard error, and the share of decisions that resumed a kept
  sub-tree.
- `agent` (also alone with --agent-only, which uses only what MCTSAgent offered before the device re-root, so the same
  command times the host re-root at an earlier commit): ONE MCTSAgent decision on HighwayLite with "subtree" at
  budgets 100 and 2000: median agent.act() time and median time of its step_tree() (the re-root) over consecutive
  decisions of one episode, after warm-up decisions."""
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

HBM_PEAK_GBS = 3350.0           # data sheet (H100 SXM, 700 W): the roofline denominator, not a measurement
BYTES_PER_NODE = 68
SHAPES = (("highway_b100", "highway", 100, 0.8), ("highway_b2000", "highway", 2000, 0.8),
          ("garnet_b100", "garnet", 100, 0.8), ("garnet_b2000", "garnet", 2000, 0.9))


def gen(i):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(i)))


def agent_decisions(budget, decisions, warmup):
    """-> median ms of agent.act() and of its step_tree() over the `decisions` decisions after `warmup` that resumed a
    re-rooted tree; an episode that ends is followed by a new one (scene seeds 0, 1, ...) with a new agent."""
    import torch
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    from rl_agents_b200.envs import HighwayLiteEnv
    act_ms, step_ms, scene = [], [], 0
    while len(act_ms) < decisions + warmup and scene < 100:
        env = HighwayLiteEnv(seed=scene)
        agent = MCTSAgent(env, {"budget": budget, "gamma": 0.8, "step_strategy": "subtree"})
        agent.seed(scene)
        planner, timing = agent.planner, {}
        step_tree = planner.step_tree

        def timed_step_tree(actions, step_tree=step_tree, planner=planner, timing=timing):
            t0 = time.perf_counter()
            step_tree(actions)
            torch.cuda.synchronize()
            timing["ms"], timing["resumed"] = 1e3 * (time.perf_counter() - t0), getattr(planner, "_resume", 0) > 0
        planner.step_tree = timed_step_tree
        done = False
        while not done and len(act_ms) < decisions + warmup:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            a = agent.act(None)
            torch.cuda.synchronize()
            if timing.get("resumed"):
                act_ms.append(1e3 * (time.perf_counter() - t0))
                step_ms.append(timing["ms"])
            _, _, term, trunc, _ = env.step(a)
            done = term or trunc
        scene += 1
    act_ms, step_ms = act_ms[warmup:], step_ms[warmup:]
    return {"budget": budget, "gamma": 0.8, "resumed_decisions": len(act_ms), "episodes": scene,
            "act_ms_median": float(np.median(act_ms)), "step_tree_ms_median": float(np.median(step_ms)),
            "step_tree_ms_max": float(np.max(step_ms))}


def engine_for(kind, n, budget, gamma, dev):
    from oracle import envs as oenvs
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mcts import MCTS, allocation, subtree_capacity
    from rl_agents_b200.engine.mcts import MCTSEngine
    episodes, horizon = allocation(budget, gamma)
    temperature = MCTS.default_config()["temperature"]
    if kind == "highway":
        return MCTSEngine(_lib.ENV_HIGHWAY, n, 5, episodes, horizon, gamma, temperature, device=dev,
                          capacity=subtree_capacity(episodes, horizon, 5))
    P, N, R = oenvs.garnet(1000, 4, 3, seed=0)
    mdp = oenvs.FiniteMDPLite(P, R, None, mode="sparse", nxt=N, seed=1).mdp
    return MCTSEngine(_lib.ENV_FINITE, n, 4, episodes, horizon, gamma, temperature, mdp=mdp, device=dev,
                      capacity=subtree_capacity(episodes, horizon, 4))


def reroot_kernel(kind, n, budget, gamma, launches, dev):
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.envs import highway_lite
    eng = engine_for(kind, n, budget, gamma, dev)
    if kind == "highway":
        roots = torch.from_numpy(np.stack([highway_lite.make_scene(s) for s in range(n)])).to(dev)
    else:
        roots = torch.arange(n, dtype=torch.int32, device=dev) % 1000
    env_words = np.stack([pcg64_words(gen(10 ** 6 + i)) for i in range(n)]) if eng.sampled else None
    eng.plan(roots, np.stack([pcg64_words(gen(i)) for i in range(n)]), None, env_words)
    _, res, _ = eng.finish()
    dst = [torch.empty_like(getattr(eng, k)) for k in _lib.MCTS_TREE_FIELDS]
    dst_tree = _lib.MCTSTree(*[t.data_ptr() for t in dst])
    act = eng.plan_buf[:, 0].to(torch.int32).contiguous()
    kept = torch.empty(n, dtype=torch.int32, device=dev)

    def launch():
        _lib.check(eng.lib.b2_mcts_reroot(eng.tree, n, eng.capacity, _lib.ptr(eng.result), _lib.MCTS_RESULT_WORDS,
                                          dst_tree, n, eng.capacity, None, _lib.ptr(act),
                                          eng.episodes * eng.n_actions, _lib.ptr(kept), _lib.current_stream()))
    launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / launches
    k = kept.cpu().numpy()
    moved = BYTES_PER_NODE * float(k[k > 0].sum())
    out = {"trees": n, "episodes": eng.episodes, "horizon": eng.horizon, "capacity": eng.capacity,
           "mean_source_nodes": float(res[:, 0].mean()), "mean_kept_nodes": float(k.mean()),
           "kept_share": float((k > 0).mean()), "launches": launches, "ms_per_launch": ms,
           "bytes_moved": moved, "gb_per_s": moved / (ms * 1e-3) / 1e9}
    out["share_of_hbm_peak"] = out["gb_per_s"] / HBM_PEAK_GBS
    del eng, dst
    torch.cuda.empty_cache()
    return out


def closed_loop(kind, n, budget, gamma, steps, strategy):
    import torch
    from rl_agents_b200.envs import FiniteMDPEnv
    from oracle import envs as oenvs
    from rl_agents_b200.evaluation import run_batched_episodes
    if kind == "highway":
        run = lambda s: run_batched_episodes("mcts", range(n), budget, gamma, max_steps=s, step_strategy=strategy)
    else:
        P, N, R = oenvs.garnet(1000, 4, 3, seed=0)
        env = FiniteMDPEnv(P, R, None, mode="sparse", nxt=N)
        starts = np.arange(n) % 1000
        run = lambda s: run_batched_episodes("mcts", range(n), budget, gamma, max_steps=s, env="finite", mdp=env,
                                             start_states=starts, env_seed=0, step_strategy=strategy)
    run(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = run(steps)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ret, decisions = res["returns"], int(res["lengths"].sum())
    out = {"decisions_per_s": decisions / wall, "wall_s": wall, "decision_ms": res["decision_ms"],
           "mean_return": float(ret.mean()), "return_stderr": float(ret.std(ddof=1) / np.sqrt(ret.size)),
           "mean_length": float(res["lengths"].mean())}
    if "resumed" in res:
        out["resumed_share"] = float(res["resumed"].sum()) / decisions
    del res
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=8448)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--decisions", type=int, default=20, help="timed agent decisions per budget")
    ap.add_argument("--agent-only", action="store_true", help="only the single-agent decision timing")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_mcts_subtree needs a GPU"
    dev = torch.device("cuda", 0)
    out = dict(gpu_info())
    out["agent"] = [agent_decisions(b, args.decisions, 3) for b in (100, 2000)]
    print(json.dumps(out["agent"]), file=sys.stderr)
    if not args.agent_only:
        out["reroot_kernel"], out["closed_loop"] = {}, {}
        for name, kind, budget, gamma in SHAPES:
            out["reroot_kernel"][name] = dict(reroot_kernel(kind, args.trees, budget, gamma, args.launches, dev),
                                              budget=budget, gamma=gamma)
            print(json.dumps({name: out["reroot_kernel"][name]}), file=sys.stderr)
        for name, kind, budget, gamma in SHAPES:
            row = {"budget": budget, "gamma": gamma, "episodes": args.trees, "steps": args.steps}
            for strategy in ("reset", "subtree"):
                row[strategy] = closed_loop(kind, args.trees, budget, gamma, args.steps, strategy)
            row["subtree_over_reset_decisions_per_s"] = (row["subtree"]["decisions_per_s"] /
                                                         row["reset"]["decisions_per_s"])
            out["closed_loop"][name] = row
            print(json.dumps({name: row}), file=sys.stderr)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
