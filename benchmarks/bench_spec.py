#!/usr/bin/env python
"""ONE strict OPD decision on HighwayLite: the one-CTA kernel (b2_opd_plan) against the speculative whole-GPU kernel
(b2_opd_plan_spec, the same tree bit for bit) over candidate widths.  CUDA-event median per decision, the kernel's own
clock64 breakdown (CTA 0, 256-cycle units -> us at the SM clock).

    python benchmarks/bench_spec.py [--budgets 10000,15625] [--gammas 0.8,0.95] [--widths 16,64,256] [--reps 5]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budgets", default="10000")
    ap.add_argument("--gammas", default="0.8")
    ap.add_argument("--widths", default="16,64,256")
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--strict", type=int, default=1)
    ap.add_argument("--sm-mhz", type=float, default=0.0, help="SM clock for the clock64 profile (default: the device's)")
    a = ap.parse_args()
    import numpy as np
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDEngine, OPDSpeculativeEngine
    from rl_agents_b200.envs.highway_lite import make_scene
    scenes = [torch.tensor(make_scene(s), dtype=torch.int32, device="cuda") for s in range(a.seeds)]
    sm_mhz = a.sm_mhz or torch.cuda.get_device_properties(0).clock_rate / 1e3

    def med_ms(fn):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return sorted(ts)[len(ts) // 2]

    rows = []
    for budget in [int(x) for x in a.budgets.split(",")]:
        for gamma in [float(x) for x in a.gammas.split(",")]:
            n_exp = budget // 5
            strict_ms = None
            if a.strict:
                eng = OPDEngine(_lib.ENV_HIGHWAY, 1, 5, budget, gamma)
                strict_ms = float(np.median([med_ms(lambda: eng.plan(s.reshape(1, -1))) for s in scenes]))
                rows.append({"budget": budget, "gamma": gamma, "kernel": "b2_opd_plan (one CTA)", "ms": strict_ms,
                             "expansions_per_s": n_exp / (strict_ms * 1e-3)})
                del eng
            for width in [int(x) for x in a.widths.split(",")]:
                eng = OPDSpeculativeEngine(_lib.ENV_HIGHWAY, 5, budget, gamma, width)
                ms = float(np.median([med_ms(lambda: eng.plan(s)) for s in scenes]))
                res = eng.result.cpu().numpy()[0]
                waves = int(res[7])
                names = ["commit", "select", "sort_worklist", "barrier_after_select", "simulate", "barrier_after_simulate",
                         "bottom_up_plan"]
                per_wave = {n: float(res[8 + i]) * 256.0 / sm_mhz / max(waves, 1) for i, n in enumerate(names)}
                rows.append({"budget": budget, "gamma": gamma, "kernel": "b2_opd_plan_spec", "candidates": width, "ms": ms,
                             "expansions_per_s": n_exp / (ms * 1e-3), "waves": waves,
                             "commits_per_wave": n_exp / float(max(waves, 1)), "max_depth": int(res[2]),
                             "speedup_vs_one_cta": (strict_ms / ms) if strict_ms else None,
                             "us_per_wave_cta0": per_wave})
                del eng
    print(json.dumps({"workload": "ONE strict OPD decision on HighwayLite", "rows": rows}))


if __name__ == "__main__":
    main()
