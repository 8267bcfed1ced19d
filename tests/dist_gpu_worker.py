"""torchrun worker for tests/test_gpu_multi.py (one rank per GPU, NCCL)."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    from oracle import envs as oenvs
    from oracle import planners
    from rl_agents_b200 import _lib
    from rl_agents_b200.distributed import DistributedVI, merge_root_statistics, recommend, shard_range
    from rl_agents_b200.engine.mcts import MCTSEngine, pcg64_words
    out = {}
    # --- slab-sharded VI vs the single-process oracle ---
    S, A, B = 3001, 4, 3
    P, N, R = oenvs.garnet(S, A, B, seed=5)
    term = np.zeros(S, bool)
    term[::101] = True
    dvi = DistributedVI("sparse", P, R, term, nxt=N, gamma=0.6, device=dev)
    q, sweeps = dvi.solve(80)
    q_ref, sweeps_ref = planners.value_iteration("sparse", P, R, term, 0.6, 80, nxt=N)
    b, e = shard_range(S, rank, world)
    out["vi_ok"] = bool(np.array_equal(q.cpu().numpy(), q_ref[b:e])) and sweeps == sweeps_ref
    out["vi_sweeps"] = sweeps
    # --- tables_are_local: every rank hands over only its own slab, as device tensors ---
    slab = dict(transition=torch.as_tensor(P[b:e]).to(dev), reward=torch.as_tensor(R[b:e]).to(dev),
                terminal=torch.as_tensor(term[b:e].astype(np.uint8)).to(dev),
                nxt=torch.as_tensor(N[b:e].astype(np.int32)).to(dev))
    dvi2 = DistributedVI("sparse", gamma=0.6, device=dev, tables_are_local=True, n_states=S, **slab)
    q2, sweeps2 = dvi2.solve(80)
    out["vi_local_ok"] = bool(np.array_equal(q2.cpu().numpy(), q_ref[b:e])) and sweeps2 == sweeps_ref
    # violation counters exchanged every 4 sweeps: same fixed point within the allclose tolerance
    dvi3 = DistributedVI("sparse", gamma=0.6, device=dev, tables_are_local=True, n_states=S, check_every=4, **slab)
    q3, sweeps3 = dvi3.solve(80)
    out["vi_check_every_ok"] = bool(np.allclose(q3.cpu().numpy(), q_ref[b:e], rtol=1e-4, atol=1e-7)) \
        and sweeps_ref <= sweeps3 <= sweeps_ref + 4
    # --- exchange fused into the sweep kernel over peer memory (no NCCL in the loop): bit-exact, same sweep count ---
    S2, A2, B2 = 4096, 8, 4
    Pp, Np, Rp = oenvs.garnet(S2, A2, B2, seed=6)
    termp = np.zeros(S2, bool)
    termp[::97] = True
    qp_ref, sweeps_p_ref = planners.value_iteration("sparse", Pp, Rp, termp, 0.7, 60, nxt=Np)
    bp, ep = shard_range(S2, rank, world)
    dvi4 = DistributedVI("sparse", Pp, Rp, termp, nxt=Np, gamma=0.7, device=dev, exchange="p2p", max_iterations=64)
    for rep in range(2):                       # twice: the flags / counters are reset correctly between solves
        q4, sweeps4 = dvi4.solve(60)
        out["vi_p2p_ok_%d" % rep] = bool(np.array_equal(q4.cpu().numpy(), qp_ref[bp:ep])) and sweeps4 == sweeps_p_ref
    dvi4.close()
    # the same exchange on an MDP with +-inf rewards and zero probabilities: the NaN that numpy's max over actions
    # keeps crosses the slabs within 3 sweeps (NaN matches any NaN, every other value bit for bit)
    from tests import vi_cases
    Pn, Rn, termn, Nn = vi_cases.nonfinite_mdp("sparse", S2, A2, B2, seed=8)
    with np.errstate(invalid="ignore", over="ignore"):
        qn_ref, sweeps_n_ref = planners.value_iteration("sparse", Pn, Rn, termn, 0.9, 3, nxt=Nn)
    dvi5 = DistributedVI("sparse", Pn, Rn, termn, nxt=Nn, gamma=0.9, device=dev, exchange="p2p", max_iterations=8)
    qn, sweeps_n = dvi5.solve(3)
    out["vi_p2p_nonfinite_ok"] = bool(np.array_equal(qn.cpu().numpy(), qn_ref[bp:ep], equal_nan=True)) \
        and sweeps_n == sweeps_n_ref
    dvi5.close()
    # --- root-parallel MCTS: one all-reduce of root statistics ---
    words = oenvs.make_highway_state(3).pack()
    ss = np.random.SeedSequence(11).spawn(world)[rank]
    gen = np.random.Generator(np.random.PCG64(ss))
    eng = MCTSEngine(_lib.ENV_HIGHWAY, 1, 5, 64 // world, 6, 0.8, 10.0, device=dev)
    eng.plan(torch.tensor(words, dtype=torch.int32, device=dev).reshape(1, -1), pcg64_words(gen).reshape(1, -1))
    eng.finish()
    d = eng.tree_dict(0)
    n = int(d["n_children"][0])
    counts = torch.zeros(5, dtype=torch.int32, device=dev)
    values = torch.zeros(5, dtype=torch.float64, device=dev)
    for c in range(d["first_child"][0], d["first_child"][0] + n):
        counts[d["action"][c]] = int(d["count"][c])
        values[d["action"][c]] = float(d["value"][c])
    mc, mv = merge_root_statistics(counts, values)
    out["mcts_total"] = float(mc.sum().item())
    out["mcts_action"] = recommend(mc.cpu().numpy(), mv.cpu().numpy())
    # --- sub-tree sharded OPD: one all-reduce(max); must equal the same decomposition run on one GPU ---
    from rl_agents_b200.distributed import ShardedOPD
    sharded = ShardedOPD(3000, 0.85, device=dev).decide(oenvs.make_highway_state(5).pack())
    out["sharded_action"] = int(sharded["action"])
    out["sharded_children"] = {str(k): list(v) for k, v in sharded["children"].items()}
    out["sharded_root"] = [sharded["root_lower"], sharded["root_upper"], sharded["n_subtrees"]]
    from rl_agents_b200.envs.intersection_lite import make_scene as make_intersection
    sh_il = ShardedOPD(3000, 0.9, device=dev, env="intersection", wave_width=16).decide(make_intersection(1))
    out["sharded_il"] = [int(sh_il["action"]), sh_il["root_lower"], sh_il["root_upper"], sh_il["n_subtrees"]]
    gathered = [None] * world
    dist.all_gather_object(gathered, out)
    if rank == 0:
        print("RESULT " + json.dumps(gathered))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
