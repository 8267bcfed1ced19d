"""PlaTyPOOS on the device engine.  Drop-in for rl_agents.agents.tree_search.platypoos.PlaTyPOOSAgent
(platypoos.py:11-197) with step_strategy "reset", on finite MDPs in every mode ("deterministic", "stochastic", "sparse")
and on HighwayLite.  plan() returns the whole action sequence to the best candidate, so `receding_horizon` serves its
later actions without replanning.

Where the reference cannot run as written, or misbehaves, the port takes these positions:
- Root value.  The root is built without a `value` attribute, so the first child update (`self.parent.value`, :129)
  raises AttributeError and the reference's plan() never completes.  Here the root's value is 0.0, so a depth-1
  child's value is its mean reward.
- Legacy env API.  The reference steps a 4-tuple `step` and draws `np_random.randint(2**30)` to seed each sample's env
  copy.  The device replays those draws on the planner's numpy PCG64 stream, and the seeded env's Generator.choice on a
  stochastic finite MDP.
- Finite MDPs skip action 0.  A finite MDP has no get_available_actions, so the reference falls back to
  range(1, n) (:145-147) and never expands action 0.  The port keeps that, the reference's own behaviour; a finite MDP
  with one action gives the root no child.
- Empty candidates.  When h_max < 2, or the root has no child, the reference's get_plan takes max() of an empty
  sequence and raises ValueError.  Here plan() raises ValueError with a message that says why, before any device work.
  The default budget 500 gives h_max 0 on HighwayLite.  A negative budget fails at construction, as in the reference,
  because the host evaluates the same expression.
- step_strategy "subtree".  The re-rooted tree's existing children never reach the next plan's layer, so its
  get_plan finds no candidate: NotImplementedError at construction.
- IntersectionLite: NotImplementedError.
"""
from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner, AbstractTreeSearchAgent, refuse_intersection
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


class PlaTyPOOS(AbstractPlanner):
    """Planning with gamma Plus an Online Optimization Strategy (scale-free adaptive planning for deterministic dynamics
    and discounted rewards): the tree is explored one depth at a time, the best nodes of a layer expanded with more
    evaluations, and the best node of each evaluation level cross-validated up to the root."""

    def __init__(self, env, config=None):
        from rl_agents_b200.engine.platypoos import horizon_of
        super(PlaTyPOOS, self).__init__(config)
        if self.config["step_strategy"] == "subtree":
            raise NotImplementedError("PlaTyPOOS on the device supports step_strategy 'reset' only: after the "
                                      "reference's 'subtree' re-rooting, the next plan finds no candidate")
        refuse_intersection("PlaTyPOOS", env)
        self.env = env
        self.openings = 0
        self.candidates = []
        if "horizon" not in self.config:                             # platypoos.py:22-25
            self.config["horizon"] = horizon_of(self.config["budget"], env.action_space.n)

    def plan(self, state, observation):
        from rl_agents_b200 import _lib
        from rl_agents_b200.engine.platypoos import PlaTyPOOSEngine, check_plannable
        horizon, gamma = self.config["horizon"], self.config["gamma"]
        d = describe(state)
        refuse_intersection("PlaTyPOOS", state)
        check_plannable(horizon, d.n_actions, d.kind == _lib.ENV_FINITE)
        key = (d.kind, d.n_actions, horizon, gamma, mdp_fingerprint(d.mdp))
        eng = self.cached_engine(key, lambda: PlaTyPOOSEngine(d.kind, 1, d.n_actions, horizon, gamma, mdp=d.mdp))
        plan, res = self.search_one_tree(eng, d)
        self.openings = int(res[1])                                  # the reference logs them (:95)
        self.candidates = [(int(p), int(n)) for p, n in eng.candidates[0].cpu().numpy().reshape(-1, 2)[:int(res[6])]]
        return plan


@register_with_reference
class PlaTyPOOSAgent(AbstractTreeSearchAgent):
    """An agent that uses PlaTyPOOS to plan a sequence of actions in an MDP."""
    PLANNER_TYPE = PlaTyPOOS
