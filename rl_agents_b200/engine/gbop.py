"""Batched GBOP-T and GBOP-D engines (device side of StateAwarePlannerAgent and GraphBasedPlannerAgent).

Both GBOP kernels keep their breadth-first backup queue as a linear array of `queue_capacity` entries per tree and
report a backup that would push past it in result word 7.  How many entries one backup needs is not bounded by any
fixed multiple of the tree or state count (it grows faster than the budget), so the engines recover: finish() doubles
the queue, reallocates it and relaunches the same search until no tree overflows.  The kernels are deterministic,
so the relaunched search is bit for bit the one a large enough queue would have run, and the grown size is kept for
the engine's later searches.  A queue thus holds fewer than twice the entries of the largest backup the engine has
run (or its first size), n_trees times over.  Only a queue that would need more than 2**31 - 1 entries (the kernels
index it with int32) is an error."""
import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import FiniteTables
from rl_agents_b200.engine.tree_engine import HostTieEngine, TreeEngine, decode_action

QUEUE_CAPACITY_MAX = 2 ** 31 - 1


def grown_queue_capacity(capacity, name):
    """The next backup queue size after an overflow at `capacity` entries: double, up to int32 indexing."""
    if capacity >= QUEUE_CAPACITY_MAX:
        raise _lib.B2Error("%s backup queue overflow: one backup needs more than 2**31 - 1 queue entries, "
                           "beyond the kernel's int32 queue indexing" % name)
    return min(2 * capacity, QUEUE_CAPACITY_MAX)


class GBOPEngine(HostTieEngine):
    """n_trees independent GBOP-T decisions per launch (one warp per tree) on a deterministic finite MDP.
    queue_factor: the first backup queue size per tree, in multiples of the node capacity (grown on overflow)."""
    # StateAwarePlanner.plan runs get_plan() twice (state_aware.py:124, :130; the first inside super().plan()): a tie
    # consumes the planner RNG on both walks, the second is returned
    TIE_WALKS = 2

    def __init__(self, n_trees, n_actions, budget, gamma, mdp, terminal_reward=0.0, backup_aggregated_nodes=True,
                 prune_suboptimal_leaves=True, accuracy=0, device="cuda", queue_factor=64):
        super(GBOPEngine, self).__init__(n_trees, n_actions, budget, gamma, terminal_reward, device)
        gamma = float(gamma)
        self.tables = FiniteTables(mdp, self.device)
        self.n_states = self.tables.n_states
        self.cfg = _lib.GBOPConfig(self.n_trees, self.n_actions, self.n_expansions, self.capacity, self.plan_capacity,
                                   min(int(queue_factor) * self.capacity, QUEUE_CAPACITY_MAX),
                                   1 if backup_aggregated_nodes else 0, 1 if prune_suboptimal_leaves else 0, gamma,
                                   1 / (1 - gamma), accuracy * (1 - gamma), self.gamma_pow.data_ptr(),
                                   self.terminal_bonus.data_ptr(), self.tables.struct())
        self.tree = _lib.GBOPTree(*self._alloc_tree(_lib.GBOP_TREE_FIELDS, self.capacity))
        self._alloc_workspace()
        self.relaunches = 0          # searches run again after a queue overflow, over the engine's life
        self._roots = None

    @property
    def queue_capacity(self):
        return int(self.cfg.queue_capacity)

    def _alloc_workspace(self):
        """Per-tree workspace: state values, per-state node lists, expansion order, then the backup queue."""
        ws = self.lib.b2_gbop_workspace_bytes(self.cfg)
        if ws < 0:
            raise _lib.B2Error("unsupported GBOP configuration")
        self.ws_per_tree = int(ws) // self.n_trees
        self.workspace = self.torch.empty(int(ws), dtype=self.torch.uint8, device=self.device)

    def plan(self, root_states):
        assert root_states.dtype == self.torch.int32 and root_states.is_cuda and root_states.is_contiguous()
        self._roots = root_states            # kept for a relaunch after a queue overflow
        _lib.check(self.lib.b2_gbop_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.workspace),
                                         _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def _result(self):
        res = super(GBOPEngine, self)._result()
        while (res[:, 7] != 0).any():
            self.cfg.queue_capacity = grown_queue_capacity(self.queue_capacity, "GBOP")
            self.workspace = None
            self._alloc_workspace()
            self.relaunches += 1
            self.plan(self._roots)
            res = super(GBOPEngine, self)._result()
        return res

    def state_values(self, tree=0):
        off = tree * self.ws_per_tree
        return self.workspace[off:off + 8 * self.n_states].view(self.torch.float64).cpu().numpy()

    def tree_dict(self, tree=0):
        n = int(self.result[tree, 0].item())
        meta = self.meta[tree, :n].cpu().numpy()
        return {"parent": self.parent[tree, :n].cpu().numpy(), "action": decode_action(meta),
                "count": self.count[tree, :n].cpu().numpy(), "depth": self.depth[tree, :n].cpu().numpy(),
                "first_child": self.first_child[tree, :n].cpu().numpy(), "n_children": (meta >> 8) & 0xff,
                "done": ((meta >> 16) & 1).astype(bool), "leaf": ((meta >> 17) & 1).astype(bool),
                "reward": self.reward[tree, :n].cpu().numpy(), "lower": self.lower[tree, :n].cpu().numpy(),
                "obs": self.obs[tree, :n].cpu().numpy()}


class GBOPDEngine(TreeEngine):
    """n_trees independent GBOP-D decisions per launch (GraphBasedPlanner, one warp per decision).
    queue_factor: the first backup queue size per tree, in multiples of the state count (grown on overflow)."""

    def __init__(self, n_trees, n_actions, budget, gamma, mdp, accuracy=1e-2, sampling_timeout=100, device="cuda",
                 queue_factor=256):
        super(GBOPDEngine, self).__init__(n_trees, _lib.OPD_RESULT_WORDS, device)
        torch = self.torch
        self.n_actions = int(n_actions)
        self.tables = FiniteTables(mdp, self.device)
        S = self.n_states = self.tables.n_states
        T = np.asarray(mdp.transition, dtype=np.int64)
        # reverse transitions (the potential parents of every state), ascending and unique
        pairs = np.unique(np.stack([T.reshape(-1), np.repeat(np.arange(S), self.n_actions)], axis=1), axis=0)
        ptr = np.zeros(S + 1, dtype=np.int32)
        np.add.at(ptr, pairs[:, 0] + 1, 1)
        self.rev_ptr = torch.as_tensor(np.cumsum(ptr).astype(np.int32), device=self.device)
        self.rev_idx = torch.as_tensor(pairs[:, 1].astype(np.int32), device=self.device)
        self.timeout = int(sampling_timeout)
        gamma = float(gamma)
        self.cfg = _lib.GBOPDConfig(self.n_trees, self.n_actions, int(budget) // self.n_actions, self.timeout, self.timeout,
                                    min(int(queue_factor) * S, QUEUE_CAPACITY_MAX), gamma, 1 / (1 - gamma),
                                    float(accuracy), self.tables.struct(), self.rev_ptr.data_ptr(), self.rev_idx.data_ptr())
        self.lower = torch.empty((self.n_trees, S), dtype=torch.float64, device=self.device)
        self.upper = torch.empty((self.n_trees, S), dtype=torch.float64, device=self.device)
        self.flags = torch.empty((self.n_trees, S), dtype=torch.uint8, device=self.device)
        self.queue = torch.empty((self.n_trees, self.queue_capacity), dtype=torch.int32, device=self.device)
        self.plan_buf = torch.empty((self.n_trees, self.timeout), dtype=torch.int8, device=self.device)
        self.relaunches = 0          # searches run again after a queue overflow, over the engine's life
        self._roots = self._rng_words = None

    @property
    def queue_capacity(self):
        return int(self.cfg.queue_capacity)

    def plan(self, root_states, rng_words):
        # kept for a relaunch after a queue overflow: the kernel advances the device copy of the words in place
        self._roots, self._rng_words = root_states, np.array(rng_words, copy=True)
        self._load_rng(rng_words)
        _lib.check(self.lib.b2_gbopd_plan(self.cfg, _lib.ptr(root_states), _lib.ptr(self.lower), _lib.ptr(self.upper),
                                          _lib.ptr(self.flags), _lib.ptr(self.queue), _lib.ptr(self.rng),
                                          _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def _result(self):
        res = super(GBOPDEngine, self)._result()
        while (res[:, 7] != 0).any():
            self.cfg.queue_capacity = grown_queue_capacity(self.queue_capacity, "GBOP-D")
            self.queue = None
            self.queue = self.torch.empty((self.n_trees, self.queue_capacity), dtype=self.torch.int32,
                                          device=self.device)
            self.relaunches += 1
            self.plan(self._roots, self._rng_words)
            res = super(GBOPDEngine, self)._result()
        return res

    def _plans(self, res):
        """The plan words up to result word 5."""
        plans_dev = self.plan_buf.cpu().numpy()
        return [plans_dev[i, :res[i, 5]].astype(int).tolist() for i in range(self.n_trees)]

    def nodes(self, tree=0):
        fl = self.flags[tree].cpu().numpy()
        lo, up = self.lower[tree].cpu().numpy(), self.upper[tree].cpu().numpy()
        return {int(s): dict(lower=float(lo[s]), upper=float(up[s]), expanded=bool(fl[s] & 2)) for s in np.nonzero(fl & 1)[0]}
