"""MCTS with double progressive widening on the device engine.  Drop-in for
rl_agents.agents.tree_search.mcts_dpw.MCTSDPWAgent (mcts_dpw.py:10-194) with step_strategy "reset", on finite MDPs in
every mode ("deterministic", "stochastic", "sparse") and on HighwayLite, open or closed loop.

Where the reference cannot run as written, the port takes these positions:
- MCTSDPW.run unpacks a 4-tuple `step` (:76) while the inherited MCTS.evaluate unpacks a 5-tuple (mcts.py:171), so the
  unmodified classes cannot finish a rollout against either env API.  Here the descent drops truncation and the rollout
  stops on terminal or truncated, which is what each of the two methods does on the env API it expects.
- DecisionNode.get_child calls `state.get_available_actions()` with no fallback (:121); a finite MDP has no such
  method.  Every action of a finite MDP is available, the fallback unexplored_actions itself uses (:110-113).
- get_plan returns root.selection_rule(), a bare action, so the reference agent's act() (`plan(...)[0]`) fails on its
  first decision.  Here plan() returns [action] and the agent works.
- step_strategy "subtree" re-roots the tree on a ChanceNode, and the next run fails there: NotImplementedError.
- horizon < 1 leaves the root childless and the reference's plan returns None: ValueError.
- The MCTS-only extensions "wavefront" and "root_parallel" are not available: NotImplementedError when set.
On HighwayLite and deterministic finite MDPs every chance node has exactly one child, open or closed loop.
"""
from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import refuse_intersection
from rl_agents_b200.agents.tree_search.mcts import MCTS, MCTSAgent
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


class MCTSDPW(MCTS):
    """UCT with double progressive widening: a decision node adds an action while k_action * N**alpha_action >=
    #children, a chance node a next state while k_state * N**alpha_state >= #children."""

    def __init__(self, env, prior_policy, rollout_policy, config=None):
        super(MCTSDPW, self).__init__(env, prior_policy, rollout_policy, config)
        if self.config["step_strategy"] == "subtree":
            raise NotImplementedError("MCTS-DPW on the device supports step_strategy 'reset' only: the reference's "
                                      "'subtree' re-roots on a chance node, where its next run fails")
        for ext in ("wavefront", "root_parallel"):
            if self.config.get(ext):
                raise NotImplementedError("%r is an MCTS extension that MCTS-DPW does not implement" % ext)
        refuse_intersection("MCTS-DPW", env)

    @classmethod
    def default_config(cls):
        cfg = super(MCTSDPW, cls).default_config()
        cfg.update({"temperature": 1, "closed_loop": False, "k_state": 1, "alpha_state": 0.3, "k_action": 3,
                    "alpha_action": 0.3})                                       # mcts_dpw.py:43-54
        return cfg

    def plan(self, state, observation):
        from rl_agents_b200.engine.mcts_dpw import MCTSDPWEngine
        c = self.config
        episodes, horizon = c["episodes"], c["horizon"]      # KeyError without episodes, as the reference's plan
        if horizon < 1:
            raise ValueError("MCTS-DPW needs horizon >= 1 (got %r): the root would stay childless and the reference's "
                             "plan returns None" % horizon)
        d = describe(state)
        refuse_intersection("MCTS-DPW", state)
        key = (d.kind, d.n_actions, episodes, horizon, c["gamma"], c["temperature"], c["k_action"], c["alpha_action"],
               c["k_state"], c["alpha_state"], bool(c["closed_loop"]), repr(self.rollout_policy), mdp_fingerprint(d.mdp))
        eng = self.cached_engine(key, lambda: MCTSDPWEngine(
            d.kind, 1, d.n_actions, episodes, horizon, c["gamma"], c["temperature"], c["k_action"], c["alpha_action"],
            c["k_state"], c["alpha_state"], closed_loop=c["closed_loop"], mdp=d.mdp,
            rollout_policy=self.rollout_policy))
        plan, _ = self.search_one_tree(eng, d)
        return plan


@register_with_reference
class MCTSDPWAgent(MCTSAgent):
    """An agent that uses MCTSDPW to plan in an MDP.  Its plans hold one action, so it replans at every step whatever
    receding_horizon is."""

    def make_planner(self):
        return MCTSDPW(self.env, MCTSAgent.policy_factory(self.config["prior_policy"]),
                       MCTSAgent.policy_factory(self.config["rollout_policy"]), self.config)

    @classmethod
    def default_config(cls):
        config = super(MCTSDPWAgent, cls).default_config()
        config.update({"budget": 100, "gamma": 0.95})                         # mcts_dpw.py:20-27
        return config
