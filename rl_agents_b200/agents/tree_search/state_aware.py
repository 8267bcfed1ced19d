"""GBOP-T agent on the device engine.  Drop-in for
rl_agents.agents.tree_search.state_aware.StateAwarePlannerAgent (state_aware.py:71-137) on deterministic finite
MDPs (the observation the reference keys its tables on, `str(observation)`, is the state id there)."""
from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner
from rl_agents_b200.agents.tree_search.deterministic import DeterministicPlannerAgent
from rl_agents_b200 import _lib
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


class StateAwarePlanner(AbstractPlanner):
    def __init__(self, env, config=None):
        super(StateAwarePlanner, self).__init__(config)
        self.env = env

    @classmethod
    def default_config(cls):
        cfg = super(StateAwarePlanner, cls).default_config()
        cfg.update({"backup_aggregated_nodes": True, "prune_suboptimal_leaves": True, "accuracy": 0})   # :79-86
        return cfg

    def plan(self, state, observation):
        from rl_agents_b200.engine.gbop import GBOPEngine
        d = describe(state)
        if d.kind != _lib.ENV_FINITE:
            raise TypeError("the device GBOP-T planner aggregates nodes by state id: it needs a finite-MDP env")
        key = (d.n_actions, self.config["budget"], self.config["gamma"], self.config.get("terminal_reward", 0),
               self.config["backup_aggregated_nodes"], self.config["prune_suboptimal_leaves"], self.config["accuracy"],
               mdp_fingerprint(d.mdp))
        eng = self.cached_engine(key, lambda: GBOPEngine(1, d.n_actions, self.config["budget"], self.config["gamma"],
                                                         d.mdp, self.config.get("terminal_reward", 0),
                                                         self.config["backup_aggregated_nodes"],
                                                         self.config["prune_suboptimal_leaves"], self.config["accuracy"]))
        plan = self.search_host_ties(eng, d.root)
        self.state_values = eng.state_values(0)
        return plan


@register_with_reference
class StateAwarePlannerAgent(DeterministicPlannerAgent):
    """An agent that performs state-aware optimistic planning in deterministic MDPs."""
    PLANNER_TYPE = StateAwarePlanner
