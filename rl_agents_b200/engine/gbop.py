"""Batched GBOP-T engine (device side of StateAwarePlannerAgent)."""
import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import FiniteTables
from rl_agents_b200.engine.tree_engine import HostTieEngine, TreeEngine, decode_action


class GBOPEngine(HostTieEngine):
    """n_trees independent GBOP-T decisions per launch (one warp per tree) on a deterministic finite MDP."""
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
                                   int(queue_factor) * self.capacity, 1 if backup_aggregated_nodes else 0,
                                   1 if prune_suboptimal_leaves else 0, gamma, 1 / (1 - gamma), accuracy * (1 - gamma),
                                   self.gamma_pow.data_ptr(), self.terminal_bonus.data_ptr(), self.tables.struct())
        self.tree = _lib.GBOPTree(*self._alloc_tree(_lib.GBOP_TREE_FIELDS, self.capacity))
        ws = self.lib.b2_gbop_workspace_bytes(self.cfg)
        if ws < 0:
            raise _lib.B2Error("unsupported GBOP configuration")
        self.ws_per_tree = int(ws) // self.n_trees
        self.workspace = self.torch.empty(int(ws), dtype=self.torch.uint8, device=self.device)

    def plan(self, root_states):
        assert root_states.dtype == self.torch.int32 and root_states.is_cuda and root_states.is_contiguous()
        _lib.check(self.lib.b2_gbop_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.workspace),
                                         _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def _check(self, res):
        super(GBOPEngine, self)._check(res)
        if (res[:, 7] != 0).any():
            raise _lib.B2Error("GBOP backup queue overflow: raise queue_factor")

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
    """n_trees independent GBOP-D decisions per launch (GraphBasedPlanner, one warp per decision)."""

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
        self.queue_capacity = int(queue_factor) * S
        self.cfg = _lib.GBOPDConfig(self.n_trees, self.n_actions, int(budget) // self.n_actions, self.timeout, self.timeout,
                                    self.queue_capacity, gamma, 1 / (1 - gamma), float(accuracy), self.tables.struct(),
                                    self.rev_ptr.data_ptr(), self.rev_idx.data_ptr())
        self.lower = torch.empty((self.n_trees, S), dtype=torch.float64, device=self.device)
        self.upper = torch.empty((self.n_trees, S), dtype=torch.float64, device=self.device)
        self.flags = torch.empty((self.n_trees, S), dtype=torch.uint8, device=self.device)
        self.queue = torch.empty((self.n_trees, self.queue_capacity), dtype=torch.int32, device=self.device)
        self.plan_buf = torch.empty((self.n_trees, self.timeout), dtype=torch.int8, device=self.device)

    def plan(self, root_states, rng_words):
        self._load_rng(rng_words)
        _lib.check(self.lib.b2_gbopd_plan(self.cfg, _lib.ptr(root_states), _lib.ptr(self.lower), _lib.ptr(self.upper),
                                          _lib.ptr(self.flags), _lib.ptr(self.queue), _lib.ptr(self.rng),
                                          _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def _check(self, res):
        if (res[:, 7] != 0).any():
            raise _lib.B2Error("GBOP-D backup queue overflow: raise queue_factor")

    def _plans(self, res):
        """The plan words up to result word 5."""
        plans_dev = self.plan_buf.cpu().numpy()
        return [plans_dev[i, :res[i, 5]].astype(int).tolist() for i in range(self.n_trees)]

    def nodes(self, tree=0):
        fl = self.flags[tree].cpu().numpy()
        lo, up = self.lower[tree].cpu().numpy(), self.upper[tree].cpu().numpy()
        return {int(s): dict(lower=float(lo[s]), upper=float(up[s]), expanded=bool(fl[s] & 2)) for s in np.nonzero(fl & 1)[0]}
