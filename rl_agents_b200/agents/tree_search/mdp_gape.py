"""MDP-GapE agent on the device engine.  Drop-in for
rl_agents.agents.tree_search.mdp_gape.MDPGapEAgent (mdp_gape.py:11-344) with step_strategy "reset", on HighwayLite and
on finite MDPs in every mode ("stochastic" and "sparse" ones with several observed next states per chance node)."""
import numpy as np

from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.common.factory import preprocess_env
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner, AbstractTreeSearchAgent, refuse_intersection
from rl_agents_b200.agents.tree_search.mcts import allocation
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


def budget_allocation(config, n_actions):
    """MDPGapE.allocate_budget (mdp_gape.py:47-58) -> (episodes, horizon): from the accuracy when
    horizon_from_accuracy is set, else OLOP's split of max(n_actions, budget)."""
    if config["horizon_from_accuracy"]:
        gamma = config["gamma"]
        horizon = int(np.ceil(np.log(config["accuracy"] * (1 - gamma) / 2) / np.log(gamma)))
        episodes = config["budget"] // horizon
        assert episodes > 1
        return episodes, horizon
    return allocation(max(n_actions, config["budget"]), config["gamma"])


class MDPGapE(AbstractPlanner):
    def __init__(self, env, config=None):
        self.env = env
        self.next_observation = None
        self.budget_used = 0
        super(MDPGapE, self).__init__(config)
        # the tree is rebuilt at every decision; the reference's "subtree" re-rooting on the observed next state
        # (mdp_gape.py:112-127) is not reproduced, so refuse it instead of silently planning differently
        if self.config["step_strategy"] == "subtree":
            raise NotImplementedError("MDP-GapE on the device supports step_strategy 'reset' only")
        if self.config["upper_bound"]["type"] != "kullback-leibler":
            raise NotImplementedError("MDP-GapE supports the kullback-leibler upper bound only")
        refuse_intersection("MDP-GapE", env)

    @classmethod
    def default_config(cls):
        cfg = super(MDPGapE, cls).default_config()
        cfg.update({"continuation_type": "zeros"})                          # OLOP (olop.py:20-34)
        cfg.update({"accuracy": 1.0,                                         # mdp_gape.py:20-40
                    "confidence": 0.9,
                    "continuation_type": "uniform",
                    "horizon_from_accuracy": False,
                    "max_next_states_count": 1,
                    "upper_bound": {"type": "kullback-leibler",
                                    "time": "global",
                                    "threshold": "3*np.log(1 + np.log(count))"
                                                 "+ horizon*np.log(actions)"
                                                 "+ np.log(1/(1-confidence))",
                                    "transition_threshold": "0.1*np.log(time)"}})
        return cfg

    def reset(self):
        if "horizon" not in self.config:
            self.config["episodes"], self.config["horizon"] = budget_allocation(self.config, self.env.action_space.n)
        super(MDPGapE, self).reset()

    def plan(self, state, observation):
        from rl_agents_b200.engine.mdp_gape import MDPGapEEngine
        d = describe(state)
        refuse_intersection("MDP-GapE", state)
        c = self.config
        ub = c["upper_bound"]
        key = (d.kind, d.n_actions, c["episodes"], c["horizon"], c["gamma"], c["accuracy"], c["confidence"],
               c["continuation_type"], c["max_next_states_count"], ub["type"], ub["threshold"],
               ub["transition_threshold"], mdp_fingerprint(d.mdp))
        eng = self.cached_engine(key, lambda: MDPGapEEngine(d.kind, 1, d.n_actions, c["episodes"], c["horizon"],
                                                            c["gamma"], ub, c["accuracy"], c["confidence"],
                                                            c["continuation_type"], c["max_next_states_count"],
                                                            mdp=d.mdp))
        plan, res = self.search_one_tree(eng, d)
        self.budget_used = int(res[1]) * self.config["horizon"]             # mdp_gape.py:109
        return plan


@register_with_reference
class MDPGapEAgent(AbstractTreeSearchAgent):
    """An agent that uses best-arm-identification to plan a sequence of actions in an MDP."""
    PLANNER_TYPE = MDPGapE

    def plan(self, observation):
        self.steps += 1
        self.step(self.previous_actions)
        env = preprocess_env(self.env, self.config["env_preprocessors"])
        self._queue.actions = self.planner.plan(state=env, observation=observation)
        return self._queue.actions

    def step(self, actions):
        """MDPGapEAgent.step (mdp_gape.py:322-341) under step_strategy "reset": the tree is reset and rebuilt at
        every call whatever receding_horizon is (a plan is one action); remaining_horizon counts down as there."""
        queue = self._queue
        queue.credit = self.config["receding_horizon"] - 1 if queue.credit == 0 else queue.credit - 1
        self.planner.step_by_reset()
        return True

    def record(self, state, action, reward, next_state, done, info):
        self.planner.next_observation = next_state                          # mdp_gape.py:343-344
