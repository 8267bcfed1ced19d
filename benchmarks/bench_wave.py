#!/usr/bin/env python
"""Latency of ONE OPD decision searched by the whole GPU (b2_opd_plan_wave) vs the strict one-CTA kernel."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rl_agents_b200 import _lib                                  # noqa: E402
from rl_agents_b200.engine.opd import OPDEngine, OPDWaveEngine    # noqa: E402
from rl_agents_b200.envs.highway_lite import make_scene          # noqa: E402


def sm_mhz():
    return torch.cuda.get_device_properties(0).clock_rate / 1e3


def time_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--budget", type=int, default=10000)
    ap.add_argument("--gamma", type=float, default=0.8)
    ap.add_argument("--widths", default="1,16,32,64,128,256")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seeds", type=int, default=3)
    ap.add_argument("--strict", type=int, default=1)
    ap.add_argument("--max-ctas", type=int, default=0)
    a = ap.parse_args()
    n_exp = a.budget // 5
    out = {"budget": a.budget, "gamma": a.gamma, "expansions": n_exp, "rows": []}
    scenes = [torch.tensor(make_scene(s), dtype=torch.int32, device="cuda") for s in range(a.seeds)]
    if a.strict:
        eng = OPDEngine(_lib.ENV_HIGHWAY, 1, 5, a.budget, a.gamma, keys_in_smem=True)
        ms = np.median([time_ms(lambda: eng.plan(s.reshape(1, -1)), a.reps) for s in scenes])
        strict_lower = [None] * a.seeds
        strict_action = [None] * a.seeds
        for i, s in enumerate(scenes):
            eng.plan(s.reshape(1, -1))
            plans, _ = eng.finish([np.random.default_rng(0)])
            strict_lower[i] = float(eng.lower[0, 0].item())
            strict_action[i] = plans[0][0]
        out["rows"].append({"kernel": "opd_highway_kernel (strict, one CTA)", "ms": float(ms),
                            "expansions_per_s": n_exp / (ms * 1e-3)})
        del eng
    for w in [int(x) for x in a.widths.split(",")]:
        eng = OPDWaveEngine(_lib.ENV_HIGHWAY, 5, a.budget, a.gamma, w, max_ctas=a.max_ctas)
        ms = np.median([time_ms(lambda: eng.plan(s), a.reps) for s in scenes])
        row = {"kernel": "opd_wave_kernel", "width": w, "ms": float(ms), "expansions_per_s": n_exp / (ms * 1e-3)}
        agree, gaps, waves = 0, [], []
        for i, s in enumerate(scenes):
            eng.plan(s)
            plans, res = eng.finish([np.random.default_rng(0)])
            waves.append(int(res[0, 7]))
            if a.strict:
                agree += int(plans[0][0] == strict_action[i])
                gaps.append(strict_lower[i] - float(eng.lower[0, 0].item()))
        names = ["stage", "bisect", "compact_layout", "barrier_after_select", "simulate", "barrier_after_simulate", "finish"]
        prof = res[0, 8:16].astype(float)
        row["prof_us_per_wave"] = {n: round(float(prof[i]) * 256 / sm_mhz() / waves[-1], 2) for i, n in enumerate(names)}
        row["bisection_steps_per_wave"] = float(prof[7]) / waves[-1]
        row["waves"] = float(np.mean(waves))
        row["us_per_wave"] = 1e3 * float(ms) / row["waves"]
        if a.strict:
            row["root_action_agreement"] = agree / float(a.seeds)
            row["value_lower_gap_vs_strict_mean"] = float(np.mean(gaps))
            row["value_lower_gap_vs_strict_max"] = float(np.max(gaps))
        out["rows"].append(row)
        del eng
    print(json.dumps(out))


if __name__ == "__main__":
    main()
