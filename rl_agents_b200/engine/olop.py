"""Batched OLOP / KL-OLOP engine (device side of OLOPAgent).

A finite MDP in mode "deterministic" runs b2_olop_plan on FiniteTables; in mode "stochastic" or "sparse" it runs
b2_olop_plan_sampled on SampledFiniteTables, where every step of an episode draws its next state from the episode's
env generator."""
import logging

import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import finite_model
from rl_agents_b200.engine.tree_engine import TreeEngine, decode_action

logger = logging.getLogger(__name__)


def thresholds_for(upper_bound, episodes):
    """compute_reward_ucb's `threshold = eval(config string)` per episode (olop.py:144-160)."""
    out = np.zeros(max(episodes, 1), dtype=np.float64)
    for episode in range(episodes):
        if upper_bound["time"] == "local":
            time = episode + 1
        elif upper_bound["time"] == "global":
            time = episodes
        else:
            time = np.nan
            logger.error("Unknown upper-bound time reference")
        out[episode] = eval(upper_bound["threshold"], {"np": np, "time": time})
    return out


class OLOPEngine(TreeEngine):
    def __init__(self, env_kind, n_trees, n_actions, episodes, horizon, gamma, upper_bound, continuation_type="zeros",
                 mdp=None, device="cuda"):
        super(OLOPEngine, self).__init__(n_trees, _lib.OLOP_RESULT_WORDS, device)
        torch = self.torch
        self.n_actions = int(n_actions)
        self.episodes, self.horizon = int(episodes), int(horizon)
        self.capacity = 1 + self.episodes * self.horizon * self.n_actions
        self.kl = upper_bound["type"] == "kullback-leibler"
        if not self.kl:
            logger.error("Unknown upper-bound type")          # olop.py:162-163: mu_ucb stays inf
        gamma = float(gamma)
        init_upper = np.array([(1 - gamma ** (self.horizon + 1 - d)) / (1 - gamma) for d in range(self.horizon + 2)],
                              dtype=np.float64)             # olop.py:118-119
        self.init_upper = torch.as_tensor(init_upper, device=self.device)
        self.thresholds = torch.as_tensor(thresholds_for(upper_bound, self.episodes) if self.kl
                                          else np.zeros(max(self.episodes, 1)), device=self.device)
        self.sampled, self.tables, finite_mdp = finite_model(env_kind, mdp, self.device)
        if self.sampled:
            self.terminal = self.tables.terminal
        self.tree = _lib.OLOPTree(*self._alloc_tree(_lib.OLOP_TREE_FIELDS, self.capacity))
        self.cfg = _lib.OLOPConfig(env_kind, self.n_trees, self.n_actions, self.episodes, self.horizon, self.capacity,
                                   1 if self.kl else 0, 1 if continuation_type == "uniform" else 0, gamma,
                                   self.thresholds.data_ptr(), self.init_upper.data_ptr(),
                                   finite_mdp)
        self.plan_buf = torch.empty((self.n_trees, max(self.horizon, 1)), dtype=torch.int8, device=self.device)

    def plan(self, root_states, rng_words):
        self._load_rng(rng_words)
        if self.sampled:
            _lib.check(self.lib.b2_olop_plan_sampled(
                self.cfg, self.tables.struct(), _lib.ptr(self.terminal), self.tables.env_draws,
                _lib.ptr(root_states), self.tree,
                _lib.ptr(self.rng), _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))
            return
        _lib.check(self.lib.b2_olop_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.rng),
                                         _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def _check(self, res):
        bad = np.nonzero(res[:, 2] == 3)[0]
        if bad.size:
            self.tables.raise_rejected_row(int(res[bad[0], 3]))
        if (res[:, 2] == 1).any():
            raise ValueError("This planner assumes that all rewards are normalized in [0, 1]")   # olop.py:133-134
        if (res[:, 2] == 2).any():
            raise KeyError(0)                         # "zeros" continuation, action 0 unavailable (olop.py:82,88)

    def _plans(self, res):
        plans = self.plan_buf.cpu().numpy()
        return [plans[i, :res[i, 1]].astype(int).tolist() for i in range(self.n_trees)]

    def tree_dict(self, tree=0):
        n = int(self.result[tree, 0].item())
        meta = self.meta[tree, :n].cpu().numpy()
        return {"parent": self.parent[tree, :n].cpu().numpy(), "action": decode_action(meta),
                "count": self.count[tree, :n].cpu().numpy(), "done": ((meta >> 16) & 1).astype(bool),
                "cumulative_reward": self.cumulative[tree, :n].cpu().numpy(),
                "mu_ucb": self.mu_ucb[tree, :n].cpu().numpy(), "upper": self.upper[tree, :n].cpu().numpy()}
