#!/usr/bin/env python
"""Value-iteration sweep benchmark (BASELINE.json configs[3], C4 shape on one GPU, or
slab-sharded under torchrun): sparse garnet MDP, fp64 P / int32 N.  Prints one JSON line:
sweeps/s, achieved algorithmic GB/s against the measured HBM peak, and numpy's time
for the same sweep on the host (the reference's bellman_expectation)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--states", type=int, default=1_000_000)
    ap.add_argument("--actions", type=int, default=8)
    ap.add_argument("--next", type=int, default=4)
    ap.add_argument("--sweeps", type=int, default=100)
    ap.add_argument("--mode", default="sparse", choices=["sparse", "deterministic"])
    ap.add_argument("--cpu-sweeps", type=int, default=3)
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    from rl_agents_b200.distributed import allgather_slabs, shard_range
    from rl_agents_b200.engine.vi import VIEngine
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    S, A, B = a.states, a.actions, a.next
    b, e = shard_range(S, rank, world)
    rng = np.random.default_rng(1000 + rank)          # each rank generates only its slab (synthetic)
    rows = e - b
    R = rng.uniform(size=(rows, A)) * (rng.uniform(size=(rows, A)) >= 0.5)
    term = np.zeros(rows, bool)
    if a.mode == "sparse":
        N = rng.integers(0, S, size=(rows, A, B), dtype=np.int64)
        P = rng.uniform(size=(rows, A, B))
        P /= P.sum(-1, keepdims=True)
        eng = VIEngine("sparse", P, R, term, nxt=N, gamma=0.95, device=dev, row_begin=b, row_end=e, n_states=S)
    else:
        T = rng.integers(0, S, size=(rows, A), dtype=np.int64)
        eng = VIEngine("deterministic", T, R, term, gamma=0.95, device=dev, row_begin=b, row_end=e, n_states=S)
        P = N = None
    eng.problem.rtol = 0.0                               # timing run: never converge early (SURVEY 8d)
    eng.problem.atol = -1.0

    def run(n):
        eng.reset(n)
        for k in range(n):
            eng.sweep(k)
            if world > 1:
                allgather_slabs(eng.v[(k + 1) & 1], S)
                dist.all_reduce(eng.viol[k:k + 1])

    run(5)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run(a.sweeps)
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item())
    assert int(eng.viol.min().item()) > 0               # every sweep did its work
    per_sweep_ms = ms / a.sweeps
    slab_bytes = eng.bytes_per_sweep()
    from bench import HBM_PEAK_GBS
    peak = HBM_PEAK_GBS
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    out = {"metric": "VI Bellman sweeps/sec", "value": 1e3 / per_sweep_ms, "unit": "sweeps/s", "n_gpus": world,
           "ms_per_sweep": per_sweep_ms, "config": {"workload": "C4: %s VI, S=%d A=%d B=%d fp64/int32, gamma 0.95"
                                                                 % (a.mode, S, A, B), "sweeps": a.sweeps},
           "roofline": {"bound": "hbm", "achieved": slab_bytes / (per_sweep_ms * 1e-3) / 1e9, "peak": peak,
                        "unit": "GB/s", "frac": slab_bytes / (per_sweep_ms * 1e-3) / 1e9 / peak,
                        "bytes_per_sweep_per_gpu": slab_bytes}}
    if rank == 0 and world == 1 and a.cpu_sweeps > 0 and a.mode == "sparse":
        v = np.zeros(S)
        t0 = time.perf_counter()
        for _ in range(a.cpu_sweeps):      # the reference's sparse Bellman operator in numpy (value_iteration.py:56-63)
            next_v = (P * np.take(v, N)).sum(axis=-1)
            next_v[term] = 0
            q = R + 0.95 * next_v
            v = q.max(axis=-1)
        dt = (time.perf_counter() - t0) / a.cpu_sweeps
        out["cpu_baseline"] = {"value": 1.0 / dt, "unit": "sweeps/s", "cores": 1, "kind": "port",
                               "sample": "%d numpy sweeps (value_iteration.py:56-63 arithmetic)" % a.cpu_sweeps}
    if rank == 0:
        print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
