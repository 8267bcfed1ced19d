#!/usr/bin/env python
"""Latency of ONE C3 MCTS decision (4096 episodes x horizon 20): strict kernel, root-parallel, wavefront."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rl_agents_b200 import _lib                                        # noqa: E402
from rl_agents_b200.engine.mcts import MCTSEngine, MCTSWaveEngine, pcg64_words   # noqa: E402
from rl_agents_b200.envs.highway_lite import make_scene                # noqa: E402


def med_ms(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def main():
    E, H = 4096, 20
    scene = torch.tensor(make_scene(0), dtype=torch.int32, device="cuda")
    rows = []
    if "--strict" in sys.argv:
        eng = MCTSEngine(_lib.ENV_HIGHWAY, 1, 5, E, H, 0.8, 10.0)
        words = pcg64_words(np.random.Generator(np.random.PCG64(0))).reshape(1, -1)
        ms = med_ms(lambda: eng.plan(scene.reshape(1, -1), words), reps=2)
        rows.append({"mode": "strict (reference episode order)", "ms": ms})
        del eng
    for width in (128, 256, 512, 1024):
        eng = MCTSWaveEngine(_lib.ENV_HIGHWAY, 5, E, H, 0.8, 10.0, width)
        ms = med_ms(lambda: eng.plan(scene, 0))
        eng.plan(scene, 0)
        plan, res = eng.finish()
        waves = int(res[3])
        prof = res[4:8].astype(float) * 256 / (torch.cuda.get_device_properties(0).clock_rate / 1e3) / waves
        counts, values = eng.root_statistics()
        rows.append({"mode": "wavefront", "width": width, "ms": ms, "episodes_per_s": E / (ms * 1e-3),
                     "env_steps": int(res[2]), "env_steps_per_s": int(res[2]) / (ms * 1e-3), "waves": waves,
                     "us_per_wave": {"select": prof[0], "barrier": prof[1], "simulate": prof[2], "barrier2": prof[3]},
                     "root_counts": counts.tolist(), "plan": plan[:5]})
        del eng
    print(json.dumps({"workload": "C3: MCTS HighwayLite 4096 episodes x horizon 20, one decision", "rows": rows}))


if __name__ == "__main__":
    main()
