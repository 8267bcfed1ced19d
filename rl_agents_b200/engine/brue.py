"""Batched BRUE engine (device side of BRUEAgent)."""
import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import FiniteTables, gamma_tables
from rl_agents_b200.engine.tree_engine import TreeEngine, decode_action


class BRUEEngine(TreeEngine):
    def __init__(self, env_kind, n_trees, n_actions, budget, horizon, gamma, mdp=None, device="cuda"):
        super(BRUEEngine, self).__init__(n_trees, _lib.BRUE_RESULT_WORDS, device)
        torch = self.torch
        if env_kind not in (_lib.ENV_FINITE, _lib.ENV_HIGHWAY):
            raise NotImplementedError("BRUE runs on finite MDPs and HighwayLite")
        self.n_actions = int(n_actions)
        self.budget, self.horizon = int(budget), int(horizon)
        if self.budget < 1 or self.horizon < 1:
            # budget < 1: the reference runs no rollout and its get_plan raises; horizon < 1: its rollouts never
            # spend budget, so its plan() never returns
            raise ValueError("BRUE needs budget >= 1 and horizon >= 1 (got %d, %d)" % (self.budget, self.horizon))
        # every env step creates at most one chance and one decision node; the last rollout may overshoot the budget
        self.capacity = 1 + 2 * (self.budget + self.horizon - 1)
        if self.capacity >= 2 ** 31:
            raise ValueError("budget + horizon too large for one tree's node arena (%d nodes)" % self.capacity)
        gamma = float(gamma)
        self.gamma_pow = torch.as_tensor(gamma_tables(gamma, self.horizon)[0], device=self.device)   # gamma**d, brue.py:63
        self.tables = FiniteTables(mdp, self.device) if env_kind == _lib.ENV_FINITE else None
        nodes = self._alloc_tree(_lib.BRUE_TREE_FIELDS, self.capacity)
        self.path = torch.empty((self.n_trees, self.horizon), dtype=torch.int32, device=self.device)
        self.path_reward = torch.empty((self.n_trees, self.horizon), dtype=torch.float64, device=self.device)
        self.cfg = _lib.BRUEConfig(env_kind, self.n_trees, self.n_actions, self.budget, self.horizon, self.capacity,
                                   gamma, self.gamma_pow.data_ptr(), self.tables.struct() if self.tables else _lib.FiniteMDP())
        self.tree = _lib.BRUETree(*nodes, self.path.data_ptr(), self.path_reward.data_ptr())
        self.plan_buf = torch.empty(self.n_trees, dtype=torch.int8, device=self.device)

    def plan(self, root_states, rng_words):
        """root_states: [n_trees] state ids (finite) or [n_trees, 136] words (HighwayLite), on the device."""
        self._load_rng(rng_words)
        _lib.check(self.lib.b2_brue_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.rng),
                                         _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def _check(self, res):
        if (res[:, 4] != 0).any():
            raise RuntimeError("BRUE node arena exhausted (error word %d)" % int(res[:, 4].max()))

    def tree_dict(self, tree=0):
        """Every node array of one tree, in creation order, with the fields of oracle.brue.tree_dict: kind, action
        (-1 on decision nodes), depth, count, value."""
        n = int(self.result[tree, 0].item())
        out = {k: getattr(self, k)[tree, :n].cpu().numpy() for k in _lib.BRUE_TREE_FIELDS}
        meta = out["meta"]
        depth = np.zeros(n, dtype=int)
        kind = (meta >> 8) & 1
        for i in range(1, n):            # parents precede their children; a chance node has its parent's depth
            depth[i] = depth[out["parent"][i]] + (1 - kind[i])
        out.update(action=decode_action(meta), kind=kind, depth=depth)
        return out
