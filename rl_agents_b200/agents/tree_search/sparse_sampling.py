"""Sparse-sampling agent on the device engine.  Drop-in for
rl_agents.agents.tree_search.sparse_sampling.SparseSamplingAgent (sparse_sampling.py:11-103) with step_strategy
"reset", on finite MDPs in every mode ("deterministic", "stochastic", "sparse") and on HighwayLite."""
from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner, AbstractTreeSearchAgent, refuse_intersection
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint

# The level-synchronous engine's workspace is sized for a tree in which every decision node has all actions; above this
# many bytes a decision keeps the lane engine, which needs no node storage and plans the same bits.
LEVEL_WORKSPACE_CAP = 1 << 30
# A finite-MDP transition is two loads, so a small tree is searched faster on one lane than through the level kernel's
# grid barriers.  On one H100 80GB HBM3 (700 W power limit), deterministic garnet, A = 4, C 3: 20 chance nodes
# (horizon 2) take 0.047 ms on the lane kernel and 0.053 ms on the level kernel, 84 (horizon 3) 0.133 and 0.069 ms
# (benchmarks/bench_sparse_sampling_levels.py).  A HighwayLite step is dear enough that the level kernel is faster
# from horizon 1 (5 chance nodes: 0.150 against 0.074 ms).
FINITE_LEVEL_MIN_CHANCE_NODES = 64


def use_level_engine(d, horizon, C):
    """Whether a decision on `d` (describe()) runs on SparseSamplingLevelEngine -- ONE decision on the whole GPU, level
    by level -- rather than on one lane group: on HighwayLite, or on a finite MDP in mode "deterministic" whose tree
    has at least FINITE_LEVEL_MIN_CHANCE_NODES chance nodes, when the worst-case workspace is at most
    LEVEL_WORKSPACE_CAP.  Both engines return the same bits."""
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.sparse_sampling import deterministic_nodes, level_workspace_bytes
    if d.kind == _lib.ENV_FINITE:
        # every action of a finite MDP is expanded: the tree is the full-width one
        if d.mdp.mode != "deterministic" or \
                (deterministic_nodes(d.n_actions, horizon) - 1) // 2 < FINITE_LEVEL_MIN_CHANCE_NODES:
            return False
    elif d.kind != _lib.ENV_HIGHWAY:
        return False
    n = level_workspace_bytes(d.kind, d.n_actions, horizon, C)
    return n is not None and n <= LEVEL_WORKSPACE_CAP


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
        from rl_agents_b200.engine.sparse_sampling import (EMPTY_ROOT_MESSAGE, SparseSamplingEngine,
                                                           SparseSamplingLevelEngine, check_horizon_and_c)
        horizon = self.config["horizon"]            # KeyError without one, as the reference's estimateV (:45)
        if horizon == 0:
            raise ValueError(EMPTY_ROOT_MESSAGE)    # a childless root, before C is ever read
        C = self.config["C"]                        # KeyError without one, as estimateQ (:76)
        check_horizon_and_c(horizon, C)
        d = describe(state)
        refuse_intersection("sparse sampling", state)
        engine = SparseSamplingLevelEngine if use_level_engine(d, horizon, C) else SparseSamplingEngine
        key = (engine, d.kind, d.n_actions, horizon, C, self.config["gamma"], mdp_fingerprint(d.mdp))
        eng = self.cached_engine(key, lambda: engine(d.kind, 1, d.n_actions, horizon, C, self.config["gamma"],
                                                     mdp=d.mdp))
        plan, _ = self.search_one_tree(eng, d)
        self.root_values = eng.root_q[0].cpu().numpy()       # the root's chance values by action (NaN: unavailable)
        return plan


@register_with_reference
class SparseSamplingAgent(AbstractTreeSearchAgent):
    """An agent that uses SparseSampling to plan in an MDP.  Its plans hold one action, so it replans at every step
    whatever receding_horizon is."""
    PLANNER_TYPE = SparseSampling
