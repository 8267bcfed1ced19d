"""GBOP-D agent on the device engine.  Drop-in for
rl_agents.agents.tree_search.graph_based.GraphBasedPlannerAgent (graph_based.py:84-150) on deterministic finite MDPs."""
from rl_agents_b200 import _lib
from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner, AbstractTreeSearchAgent
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


class GraphBasedPlanner(AbstractPlanner):
    def __init__(self, env, config=None):
        super(GraphBasedPlanner, self).__init__(config)
        self.env = env

    def plan(self, state, observation):
        from rl_agents_b200.engine.gbop import GBOPDEngine
        d = describe(state)
        if d.kind != _lib.ENV_FINITE:
            raise TypeError("the device GBOP-D planner builds a graph over state ids: it needs a finite-MDP env")
        key = (d.n_actions, self.config["budget"], self.config["gamma"], self.config["accuracy"],
               self.config["sampling_timeout"], mdp_fingerprint(d.mdp))
        eng = self.cached_engine(key, lambda: GBOPDEngine(1, d.n_actions, self.config["budget"], self.config["gamma"],
                                                          d.mdp, self.config["accuracy"],
                                                          self.config["sampling_timeout"]))
        return self.search_one_tree(eng, d)[0]          # the tie-breaks consume the planner's stream


@register_with_reference
class GraphBasedPlannerAgent(AbstractTreeSearchAgent):
    PLANNER_TYPE = GraphBasedPlanner

    @classmethod
    def default_config(cls):
        cfg = super(GraphBasedPlannerAgent, cls).default_config()
        cfg.update({"sampling_timeout": 100, "accuracy": 1e-2})        # graph_based.py:143-150
        return cfg
