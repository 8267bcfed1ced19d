"""Batched MDP-GapE engine (device side of MDPGapEAgent).

A finite MDP in mode "deterministic" runs b2_mdp_gape_plan on FiniteTables; in mode "stochastic" or "sparse" it runs
b2_mdp_gape_plan_sampled on SampledFiniteTables, where chance nodes observe several next states."""
import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import finite_model
from rl_agents_b200.engine.tree_engine import TreeEngine, decode_action


def count_table(expression, episodes, horizon, n_actions, confidence):
    """`eval(expression)` for count = 0 .. episodes + 2 with the names compute_reward_ucb / transition_threshold
    put in scope (mdp_gape.py:200-213, 307-313; `time` is always the global episode budget).  Entry 0 is never
    read; an exception of the expression surfaces as the reference's would."""
    out = np.zeros(episodes + 3, dtype=np.float64)
    scope = {"np": np, "horizon": horizon, "actions": n_actions, "confidence": confidence, "time": episodes}
    for count in range(1, episodes + 3):
        out[count] = eval(expression, dict(scope, count=count))
    return out


PLACEHOLDERS_MESSAGE = ("No more placeholder nodes available, we observed more next states than the "
                        "'max_next_states_count' config")


class MDPGapEEngine(TreeEngine):
    def __init__(self, env_kind, n_trees, n_actions, episodes, horizon, gamma, upper_bound, accuracy, confidence,
                 continuation_type="uniform", max_next_states_count=1, mdp=None, device="cuda"):
        super(MDPGapEEngine, self).__init__(n_trees, _lib.MDP_GAPE_RESULT_WORDS, device)
        torch = self.torch
        if env_kind not in (_lib.ENV_FINITE, _lib.ENV_HIGHWAY):
            raise NotImplementedError("MDP-GapE runs on finite MDPs and HighwayLite")
        if upper_bound["type"] != "kullback-leibler":
            # the reference only implements the KL bounds (mdp_gape.py:200-212); any other type leaves infinite
            # bounds whose backups are NaN
            raise NotImplementedError("MDP-GapE supports the kullback-leibler upper bound only")
        self.n_actions = int(n_actions)
        self.episodes, self.horizon = int(episodes), int(horizon)
        self.n_next = int(max_next_states_count)
        self.capacity = 1 + (self.episodes + 2) * self.horizon * (self.n_actions + self.n_next)
        gamma = float(gamma)
        init_upper = np.array([(1 - gamma ** (self.horizon - d)) / (1 - gamma) for d in range(self.horizon + 1)],
                              dtype=np.float64)                              # mdp_gape.py:145-147
        table = lambda expr: torch.as_tensor(count_table(expr, self.episodes, self.horizon, self.n_actions, confidence),
                                             device=self.device)
        self.thresholds = table(upper_bound["threshold"])
        self.transition_thresholds = table(upper_bound["transition_threshold"])
        self.init_upper = torch.as_tensor(init_upper, device=self.device)
        self.sampled, self.tables, finite_mdp = finite_model(env_kind, mdp, self.device)
        self.keys = None
        if self.sampled:
            self.terminal = self.tables.terminal
            self.keys = torch.empty((self.n_trees, self.capacity), dtype=torch.int32, device=self.device)
        self.tree = _lib.MDPGapETree(*self._alloc_tree(_lib.MDP_GAPE_TREE_FIELDS, self.capacity))
        self.cfg = _lib.MDPGapEConfig(env_kind, self.n_trees, self.n_actions, self.episodes, self.horizon,
                                      self.capacity, self.n_next, 1 if continuation_type == "uniform" else 0, gamma,
                                      float(accuracy), self.thresholds.data_ptr(),
                                      self.transition_thresholds.data_ptr(), self.init_upper.data_ptr(),
                                      finite_mdp)
        self.plan_buf = torch.empty(self.n_trees, dtype=torch.int8, device=self.device)

    def plan(self, root_states, rng_words):
        """root_states: [n_trees] state ids (finite) or [n_trees, 136] words (HighwayLite), on the device."""
        self._load_rng(rng_words)
        if self.sampled:
            _lib.check(self.lib.b2_mdp_gape_plan_sampled(
                self.cfg, self.tables.struct(), _lib.ptr(self.terminal), self.tables.env_draws,
                _lib.ptr(root_states), self.tree,
                _lib.ptr(self.keys), _lib.ptr(self.rng), _lib.ptr(self.plan_buf), _lib.ptr(self.result),
                _lib.current_stream()))
            return
        _lib.check(self.lib.b2_mdp_gape_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.rng),
                                             _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def _check(self, res):
        bad = np.nonzero(res[:, 2] == 4)[0]
        if bad.size:
            self.tables.raise_rejected_row(int(res[bad[0], 6]))
        if (res[:, 2] == 3).any():
            raise ValueError(PLACEHOLDERS_MESSAGE)                                   # mdp_gape.py:283-285
        if (res[:, 2] == 1).any():
            raise ValueError("This planner assumes that all rewards are normalized in [0, 1]")   # olop.py:133-134
        if (res[:, 2] == 2).any():
            raise ValueError("max() arg is an empty sequence")       # one available root action (mdp_gape.py:247)

    def tree_dict(self, tree=0):
        """Every node array of one tree, in creation order; `action` is the env action of a chance node, the
        placeholder index of a decision node below one, -1 at the root.  `order` maps each expanded chance node to
        its children in the reference's dict order (the unobserved placeholders, then the observed ones in the
        order they were observed); on a sampled MDP `key` is the state id a decision node was observed under, -1
        elsewhere."""
        n = int(self.result[tree, 0].item())
        out = {k: getattr(self, k)[tree, :n].cpu().numpy() for k in _lib.MDP_GAPE_TREE_FIELDS}
        meta = out["meta"]
        out.update(action=decode_action(meta), n_children=(meta >> 8) & 0xff, done=((meta >> 16) & 1).astype(bool),
                   kind=(meta >> 17) & 1, cumulative_reward=out["cumulative"])
        if self.sampled:
            out["key"] = self.keys[tree, :n].cpu().numpy()
        out["order"] = {}
        for c in np.nonzero((out["kind"] == 1) & (out["first_child"] >= 0))[0]:
            fc, k = int(out["first_child"][c]), int(out["n_children"][c])
            n_obs = int((out["key"][fc:fc + k] >= 0).sum()) if self.sampled else 1
            out["order"][int(c)] = list(range(fc + n_obs, fc + k)) + list(range(fc, fc + n_obs))
        return out
