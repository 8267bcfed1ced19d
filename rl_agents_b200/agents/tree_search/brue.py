"""BRUE agent on the device engine.  Drop-in for rl_agents.agents.tree_search.brue.BRUEAgent (brue.py:11-123) with
step_strategy "reset"."""
from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import AbstractTreeSearchAgent, refuse_intersection
from rl_agents_b200.agents.tree_search.olop import OLOP
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint

# what the reference raises when no rollout ran (budget < 1): np.amax of the root's empty value list
EMPTY_ROOT_MESSAGE = "zero-size array to reduction operation maximum which has no identity"


class BRUE(OLOP):
    """Best Recommendation with Uniform Exploration.  Like the reference it is an OLOP planner: it inherits OLOP's
    default config and, without a configured "horizon", OLOP's budget allocation (brue.py:19-22)."""

    def __init__(self, env, config=None):
        self.available_budget = 0
        super(BRUE, self).__init__(env, config)
        # the reference's "subtree" re-roots on a chance node, whose next plan() raises AttributeError
        if self.config["step_strategy"] == "subtree":
            raise NotImplementedError("BRUE on the device supports step_strategy 'reset' only")
        refuse_intersection("BRUE", env)

    def plan(self, state, observation):
        from rl_agents_b200.engine.brue import BRUEEngine
        if self.config["horizon"] < 1:
            # the reference's rollouts would never take a step, so its budget loop would never end
            raise ValueError("BRUE needs horizon >= 1 (got %r)" % self.config["horizon"])
        if self.config["budget"] < 1:
            raise ValueError(EMPTY_ROOT_MESSAGE)                     # no rollout: get_plan has nothing to choose
        d = describe(state)
        refuse_intersection("BRUE", state)
        c = self.config
        key = (d.kind, d.n_actions, c["budget"], c["horizon"], c["gamma"], mdp_fingerprint(d.mdp))
        eng = self.cached_engine(key, lambda: BRUEEngine(d.kind, 1, d.n_actions, c["budget"], c["horizon"], c["gamma"],
                                                         mdp=d.mdp))
        plan, res = self.search_one_tree(eng, d)
        self.available_budget = self.config["budget"] - int(res[2])        # <= 0: the last rollout overshoots
        return plan


@register_with_reference
class BRUEAgent(AbstractTreeSearchAgent):
    """An agent that uses BRUE to plan a sequence of actions in an MDP.  Its plans hold one action, so it replans at
    every step whatever receding_horizon is."""
    PLANNER_TYPE = BRUE
