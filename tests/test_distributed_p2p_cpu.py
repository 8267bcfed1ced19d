"""world_size-2 gloo test (CPU) of DistributedVI(exchange="p2p")'s constructor: the refusals every rank must make alike
before anything touches a device (the single-GPU tests of the exchange itself are tests/test_gpu_vi_p2p.py)."""
import numpy as np

from rl_agents_b200.distributed import shard_range
from tests.test_distributed_cpu import run_world


def _p2p_fewer_states_than_ranks(rank, world):
    """DistributedVI(exchange="p2p") with S = 1 < world: a rank without a state would have its sweep refused while
    its peers wait for its arrival flag.  Every rank must refuse in the constructor, before the VIEngine touches a
    device (there is none here), with full tables and with its own (possibly empty) slab."""
    from oracle import envs as oenvs
    from rl_agents_b200.distributed import DistributedVI
    P, N, R = oenvs.garnet(1, 4, 2, seed=0)
    term = np.zeros(1, bool)
    b, e = shard_range(1, rank, world)
    out = []
    for kw in (dict(transition=P, reward=R, terminal=term, nxt=N),
               dict(transition=P[b:e], reward=R[b:e], terminal=term[b:e], nxt=N[b:e], tables_are_local=True,
                    n_states=1)):
        try:
            DistributedVI("sparse", gamma=0.9, device="cuda", exchange="p2p", **kw)
            out.append(None)
        except ValueError as ex:
            out.append(str(ex))
    return out


def test_p2p_value_iteration_refuses_fewer_states_than_ranks():
    out = run_world(_p2p_fewer_states_than_ranks)
    assert all(msg is not None and "a state for every rank" in msg for o in out for msg in o), out
