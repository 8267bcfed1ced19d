#!/usr/bin/env python
"""Secondary measurements for DESIGN.md: single-decision latencies through the agent-level
engines (one tree), finite-MDP OPD batch throughput, OLOP batch throughput.  One JSON line."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, reps=5):
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def main():
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import MCTSEngine, pcg64_words
    from rl_agents_b200.engine.olop import OLOPEngine
    from rl_agents_b200.engine.opd import OPDEngine
    from rl_agents_b200.envs.finite_mdp import FiniteMDP
    from rl_agents_b200.envs.highway_lite import make_scene
    dev = torch.device("cuda", 0)
    out = {}
    scene = torch.from_numpy(make_scene(0)).reshape(1, -1).to(dev)
    gen = np.random.Generator(np.random.PCG64(np.random.SeedSequence(0)))

    # --- one decision at a time (what agent.plan() does) ---
    eng = OPDEngine(_lib.ENV_HIGHWAY, 1, 5, 10000, 0.8, keys_in_smem=True)
    out["opd_highway_b10000_single_decision_ms"] = timed(lambda: (eng.plan(scene), eng.finish([gen])))
    eng = OPDEngine(_lib.ENV_HIGHWAY, 1, 5, 75, 0.7, keys_in_smem=True)
    out["opd_highway_b75_single_decision_ms"] = timed(lambda: (eng.plan(scene), eng.finish([gen])))
    g = np.load(os.path.join(ROOT, "tests", "golden", "finite_mdps.npz"))
    mdp = FiniteMDP("deterministic", g["large1_T"], g["large1_R"], g["large1_term"])
    root1 = torch.zeros(1, dtype=torch.int32, device=dev)
    eng = OPDEngine(_lib.ENV_FINITE, 1, 5, 10000, 0.9, mdp=mdp, keys_in_smem=True)
    out["opd_finite_b10000_single_decision_ms"] = timed(lambda: (eng.plan(root1), eng.finish([gen])))
    meng = MCTSEngine(_lib.ENV_HIGHWAY, 1, 5, 4096, 20, 0.8, 10.0)
    w1 = pcg64_words(gen).reshape(1, -1)
    out["mcts_highway_4096x20_single_decision_ms"] = timed(lambda: (meng.plan(scene, w1), meng.finish()), reps=3)

    rp = MCTSEngine(_lib.ENV_HIGHWAY, 64, 5, 64, 20, 0.8, 10.0)            # root_parallel = 64: 64 trees x 64 episodes
    scenes64 = scene.repeat(64, 1).contiguous()
    w64 = np.stack([pcg64_words(g) for g in gen.spawn(64)])
    out["mcts_highway_4096x20_root_parallel64_ms"] = timed(lambda: (rp.plan(scenes64, w64), rp.finish()), reps=3)

    # --- C5-sized single decision: budget 1e6 (200 000 expansions), strict single tree and sub-tree sharded ---
    if "--big" in sys.argv:
        big = OPDEngine(_lib.ENV_HIGHWAY, 1, 5, 1_000_000, 0.9)
        out["opd_highway_b1e6_single_tree_ms"] = timed(lambda: (big.plan(scene), big.finish([gen])), reps=1)
        out["opd_highway_b1e6_max_depth"] = int(big.result[0, 2].item())
        del big
        from rl_agents_b200.distributed import ShardedOPD
        sh = ShardedOPD(1_000_000, 0.9, device=dev)
        t0 = time.perf_counter()
        d = sh.decide(make_scene(0))
        torch.cuda.synchronize()
        out["opd_highway_b1e6_sharded_1gpu_ms"] = (time.perf_counter() - t0) * 1e3
        out["opd_highway_b1e6_sharded_subtrees"] = d["n_subtrees"]

    # --- batches ---
    n = torch.cuda.get_device_properties(dev).multi_processor_count * 256
    roots = torch.randint(0, 100, (n,), dtype=torch.int32, device=dev)
    eng = OPDEngine(_lib.ENV_FINITE, n, 5, 10000, 0.9, mdp=mdp)
    ms = timed(lambda: eng.plan(roots), reps=3)
    out["opd_finite_b10000_batch"] = {"trees": n, "ms": ms, "expansions_per_s": n * 2000 / (ms * 1e-3)}
    ub = {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)"}
    n = torch.cuda.get_device_properties(dev).multi_processor_count * 64
    scenes = torch.from_numpy(np.stack([make_scene(i) for i in range(n)])).to(dev)
    oeng = OLOPEngine(_lib.ENV_HIGHWAY, n, 5, 72, 6, 0.7, ub, "uniform")      # budget 500, gamma 0.7 (shipped KL-OLOP config)
    words = np.stack([pcg64_words(np.random.Generator(np.random.PCG64(i))) for i in range(n)])
    ms = timed(lambda: oeng.plan(scenes, words), reps=3)
    out["olop_highway_b500_batch"] = {"trees": n, "ms": ms, "episodes_per_s": n * 72 / (ms * 1e-3),
                                      "env_steps_per_s": n * 72 * 6 / (ms * 1e-3)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
