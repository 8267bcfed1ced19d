"""OLOP / KL-OLOP agent on the device engine.  Drop-in for
rl_agents.agents.tree_search.olop.OLOPAgent (olop.py:11-200), on HighwayLite, IntersectionLite and finite MDPs in every
mode ("stochastic" and "sparse" ones draw a next state at every step of an episode)."""
from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner, AbstractTreeSearchAgent
from rl_agents_b200.agents.tree_search.mcts import allocation
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


class OLOP(AbstractPlanner):
    def __init__(self, env, config=None):
        self.env = env
        super(OLOP, self).__init__(config)

    @classmethod
    def default_config(cls):
        cfg = super(OLOP, cls).default_config()
        cfg.update({"upper_bound": {"type": "hoeffding", "time": "global", "threshold": "4*np.log(time)"},
                    "continuation_type": "zeros"})          # olop.py:20-34
        return cfg

    def reset(self):
        if "horizon" not in self.config:                     # olop.py:36-48
            budget = max(self.env.action_space.n, self.config["budget"])
            self.config["episodes"], self.config["horizon"] = allocation(budget, self.config["gamma"])
        # the reference builds its root OLOPNode here, which reads upper_bound["type"] (olop.py:115): a config whose
        # "upper_bound" is a bare string, as the shipped FiniteMDPEnv/agents/olop.json has, raises that TypeError
        self.config["upper_bound"]["type"]
        super(OLOP, self).reset()

    def plan(self, state, observation):
        from rl_agents_b200.engine.olop import OLOPEngine
        d = describe(state)
        ub = self.config["upper_bound"]
        key = (d.kind, d.n_actions, self.config["episodes"], self.config["horizon"], self.config["gamma"],
               ub["type"], ub["time"], ub["threshold"], self.config["continuation_type"], mdp_fingerprint(d.mdp))
        eng = self.cached_engine(key, lambda: OLOPEngine(d.kind, 1, d.n_actions, self.config["episodes"],
                                                         self.config["horizon"], self.config["gamma"], ub,
                                                         self.config["continuation_type"], mdp=d.mdp))
        return self.search_one_tree(eng, d)[0]


@register_with_reference
class OLOPAgent(AbstractTreeSearchAgent):
    """An agent that uses Open Loop Optimistic Planning to plan a sequence of actions in an MDP."""
    PLANNER_TYPE = OLOP
