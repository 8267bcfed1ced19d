"""Sparse-sampling agent on the device engine.  Drop-in for
rl_agents.agents.tree_search.sparse_sampling.SparseSamplingAgent (sparse_sampling.py:11-103) with step_strategy
"reset", on finite MDPs in every mode ("deterministic", "stochastic", "sparse") and on HighwayLite."""
from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner, AbstractTreeSearchAgent, refuse_intersection
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


class SparseSampling(AbstractPlanner):
    """Kearns, Mansour and Ng's sparse sampling: C sampled next states per (state, action), down to `horizon`.
    The config has no defaults of its own: `horizon` and `C` must be given (a KeyError at plan time otherwise, as in
    the reference)."""

    def __init__(self, env, config=None):
        super(SparseSampling, self).__init__(config)
        # the reference's "subtree" re-roots on a chance node, whose next plan() fails
        if self.config["step_strategy"] == "subtree":
            raise NotImplementedError("sparse sampling on the device supports step_strategy 'reset' only")
        refuse_intersection("sparse sampling", env)
        self.root_values = None

    def plan(self, state, observation):
        from rl_agents_b200.engine.sparse_sampling import EMPTY_ROOT_MESSAGE, SparseSamplingEngine, check_horizon_and_c
        horizon = self.config["horizon"]            # KeyError without one, as the reference's estimateV (:45)
        if horizon == 0:
            raise ValueError(EMPTY_ROOT_MESSAGE)    # a childless root, before C is ever read
        C = self.config["C"]                        # KeyError without one, as estimateQ (:76)
        check_horizon_and_c(horizon, C)
        d = describe(state)
        refuse_intersection("sparse sampling", state)
        key = (d.kind, d.n_actions, horizon, C, self.config["gamma"], mdp_fingerprint(d.mdp))
        eng = self.cached_engine(key, lambda: SparseSamplingEngine(d.kind, 1, d.n_actions, horizon, C,
                                                                   self.config["gamma"], mdp=d.mdp))
        plan, _ = self.search_one_tree(eng, d)
        self.root_values = eng.root_q[0].cpu().numpy()       # the root's chance values by action (NaN: unavailable)
        return plan


@register_with_reference
class SparseSamplingAgent(AbstractTreeSearchAgent):
    """An agent that uses SparseSampling to plan in an MDP.  Its plans hold one action, so it replans at every step
    whatever receding_horizon is."""
    PLANNER_TYPE = SparseSampling
