"""Multi-GPU parity (needs >= 2 GPUs on the box; skipped otherwise)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus():
    import torch
    return torch.cuda.device_count()


def test_two_rank_vi_and_root_parallel_mcts():
    if _gpus() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29531", os.path.join(ROOT, "tests", "dist_gpu_worker.py")]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:]
    line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])
    assert all(r["vi_ok"] for r in res)
    assert all(r["vi_local_ok"] for r in res) and all(r["vi_check_every_ok"] for r in res)
    assert all(r["vi_p2p_ok_0"] and r["vi_p2p_ok_1"] for r in res)
    assert all(r["vi_p2p_nonfinite_ok"] for r in res)
    assert res[0]["vi_sweeps"] == res[1]["vi_sweeps"] < 80          # converged early, same sweep on both ranks
    # every episode of both trees counted once; the episode that expands a root descends into no child
    assert res[0]["mcts_total"] == res[1]["mcts_total"] == 64.0 - 2
    assert res[0]["mcts_action"] == res[1]["mcts_action"]
    # sharded OPD: both ranks agree, and equal the single-GPU run of the same decomposition bit for bit
    import torch
    from oracle import envs as oenvs
    from rl_agents_b200.distributed import ShardedOPD
    assert res[0]["sharded_children"] == res[1]["sharded_children"] and res[0]["sharded_action"] == res[1]["sharded_action"]
    torch.cuda.set_device(0)
    single = ShardedOPD(3000, 0.85, device="cuda:0").decide(oenvs.make_highway_state(5).pack())
    assert {str(k): list(v) for k, v in single["children"].items()} == res[0]["sharded_children"]
    assert int(single["action"]) == res[0]["sharded_action"]
    assert [single["root_lower"], single["root_upper"], single["n_subtrees"]] == res[0]["sharded_root"]
    # the same on IntersectionLite (C5's env model), sub-trees searched in waves
    from rl_agents_b200.envs.intersection_lite import make_scene as make_intersection
    single_il = ShardedOPD(3000, 0.9, device="cuda:0", env="intersection", wave_width=16).decide(make_intersection(1))
    assert res[0]["sharded_il"] == res[1]["sharded_il"]
    assert res[0]["sharded_il"] == [int(single_il["action"]), single_il["root_lower"], single_il["root_upper"],
                                    single_il["n_subtrees"]]


def test_sharded_opd_single_rank_is_consistent_with_plain_opd():
    """world == 1: the decomposition's bounds bracket / agree with a plain OPD search of the scene."""
    import numpy as np
    from oracle import envs as oenvs
    from rl_agents_b200 import _lib
    from rl_agents_b200.distributed import ShardedOPD
    from rl_agents_b200.engine.opd import OPDEngine
    import torch
    words = oenvs.make_highway_state(6).pack()
    d = ShardedOPD(2000, 0.8, device="cuda").decide(words)
    assert d["action"] in d["children"] and d["root_lower"] <= d["root_upper"]
    eng = OPDEngine(_lib.ENV_HIGHWAY, 1, 5, 2000, 0.8)
    eng.plan(torch.tensor(words, dtype=torch.int32, device="cuda").reshape(1, -1))
    plans, _ = eng.finish([np.random.default_rng(0)])
    lo, up = float(eng.lower[0, 0]), float(eng.upper[0, 0])
    # both are valid brackets of the same optimal value: the intervals must intersect
    assert max(lo, d["root_lower"]) <= min(up, d["root_upper"]) + 1e-12
    assert plans[0][0] in d["children"]
