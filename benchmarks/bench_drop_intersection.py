#!/usr/bin/env python
"""DROP on IntersectionLite: the time of ONE DiscreteRobustPlanner decision (b2_opd_plan_wave with n_models = 3) over
the three route hypotheses of routes_behaviours.json (the other vehicles on their approach turning left / straight /
right), at budgets 20 (the shipped config), 200 and 2 000, gamma 0.9, in waves of 1 leaf (the reference's order) and
of 64; beside plain OPD (n_models = 0) on the same scene, budget and width.  GPU arm: the host clock around plan() +
finish() (launch, synchronise, result copy, host tie-break) and CUDA events around the launch alone, best of --reps
after a warm-up at the timed shape.  CPU arm: oracle.planners.robust_plan (numpy, the reference's algorithm) per
decision, pinned to one core; its plans are compared with the kernel's.  One JSON line with the GPU's name and
power limit; --out also writes it to a file."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from benchmarks.bench_mdp_gape import gpu_info  # noqa: E402

GAMMA = 0.9
BUDGETS = (20, 200, 2000)
WIDTHS = (1, 64)
TURNS = (0, 1, 2)


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", type=int, default=0, help="make_scene seed")
    ap.add_argument("--reps", type=int, default=20, help="timed decisions per config (best is reported)")
    ap.add_argument("--cpu-reps", type=int, default=3, help="CPU decisions per budget below 2000 (2000: one)")
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--out", default="", help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDWaveEngine
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv, make_scene
    assert torch.cuda.is_available(), "bench_drop_intersection needs a GPU"
    dev = torch.device("cuda", 0)
    env = IntersectionLiteEnv(make_scene(args.scene))
    models = np.stack([env.set_route_at_intersection(k).words for k in TURNS])
    roots = {"drop_m3": torch.tensor(models, dtype=torch.int32, device=dev),
             "opd": torch.tensor(env.words, dtype=torch.int32, device=dev)}
    out = dict(gpu_info(), scene=args.scene, gamma=GAMMA, n_models=len(TURNS), results={})
    plans = {}
    for budget in BUDGETS:
        for width in WIDTHS:
            row = {"budget": budget, "width": width}
            for name, root in roots.items():
                m = len(TURNS) if name == "drop_m3" else 0
                eng = OPDWaveEngine(_lib.ENV_INTERSECTION, 3, budget, GAMMA, width, device=dev, n_models=m)
                eng.plan(root)
                eng.finish([np_random(0)])                       # warm-up at the timed shape
                wall, kern = [], []
                for _ in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    e0.record()
                    eng.plan(root)
                    e1.record()
                    p, res = eng.finish([np_random(0)])
                    wall.append((time.perf_counter() - t0) * 1e3)
                    kern.append(e0.elapsed_time(e1))
                row[name] = {"ms_per_decision": min(wall), "kernel_ms": min(kern), "nodes": int(res[0, 0]),
                             "waves": int(res[0, 7]), "plan": p[0]}
                if name == "drop_m3":
                    plans[(budget, width)] = p[0]
                del eng
            row["drop_over_opd_time"] = row["drop_m3"]["ms_per_decision"] / row["opd"]["ms_per_decision"]
            out["results"]["b%d_w%d" % (budget, width)] = row
            print(json.dumps(row), file=sys.stderr, flush=True)
    if not args.no_cpu:
        from oracle import intersection as oit
        from oracle import planners
        from oracle.intersection_routes import IntersectionLiteRoutes
        if hasattr(os, "sched_setaffinity"):
            os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
        oenv = IntersectionLiteRoutes(oit.IntersectionLiteState.unpack(env.words))
        cpu = {}
        for budget in BUDGETS:
            times = []
            for _ in range(1 if budget >= 2000 else args.cpu_reps):
                t0 = time.perf_counter()
                plan, _ = planners.robust_plan([oenv.set_route_at_intersection(k) for k in TURNS], budget, GAMMA,
                                               np_random=np_random(0))
                times.append((time.perf_counter() - t0) * 1e3)
            cpu["b%d" % budget] = {"ms_per_decision": min(times), "plan_equals_kernel_w1": plan == plans[(budget, 1)],
                                   "gpu_speedup_w1": min(times) / out["results"]["b%d_w1" % budget]["drop_m3"][
                                       "ms_per_decision"]}
            print(budget, json.dumps(cpu["b%d" % budget]), file=sys.stderr, flush=True)
        out["cpu_one_core_robust_plan"] = cpu
    line = json.dumps(dict(metric="ONE DROP decision (M = 3 route hypotheses) on IntersectionLite beside plain OPD",
                           **out))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
