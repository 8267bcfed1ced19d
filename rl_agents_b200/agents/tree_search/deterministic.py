"""OPD agent on the device engine.  Drop-in for
rl_agents.agents.tree_search.deterministic.DeterministicPlannerAgent
(deterministic.py:91-139): same constructor, config keys and defaults, same
plan()/act() results on identical seeds."""
from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner, AbstractTreeSearchAgent
from rl_agents_b200 import _lib
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


class OptimisticDeterministicPlanner(AbstractPlanner):
    """plan(): one OPD decision, searched by libb2planner (b2_opd_plan)."""

    def __init__(self, env, config=None):
        super(OptimisticDeterministicPlanner, self).__init__(config)
        self.env = env

    SPEC_MAX_NODES = 24576      # one shared-memory tile of frontier keys (opd_wave.cu: STAGE_CAP)

    def _speculative_width(self, d, wavefront):
        """`"speculative"`: K in 1..256 forces b2_opd_plan_spec, 0 / False the one-CTA kernel; "auto" (default)
        takes it for the scene models when the tree fits and gamma <= 0.9 -- with a larger discount the best
        child nearly always outranks the second-best leaf, the strict order is a chain and nothing commits
        ahead (measured: 2.4x faster at gamma 0.8, 2x slower at 0.95; docs/DESIGN.md section 4c)."""
        spec = self.config.get("speculative", "auto")
        n_exp = int(self.config["budget"]) // d.n_actions
        fits = 1 + n_exp * d.n_actions <= self.SPEC_MAX_NODES
        if spec == "auto":
            if wavefront > 0 or not fits or d.kind == _lib.ENV_FINITE:
                return 0
            if d.kind == _lib.ENV_INTERSECTION:
                return 256
            return 256 if float(self.config["gamma"]) <= 0.9 else 0
        spec = int(spec or 0)
        if spec > 0 and not fits:
            raise ValueError("speculative search holds trees of at most %d nodes" % self.SPEC_MAX_NODES)
        return spec

    def _engine_for(self, d):
        """Default: the reference's strict best-first order, bit-exact with deterministic.py -- by the speculative
        whole-GPU kernel (b2_opd_plan_spec) where that pays, else one CTA (b2_opd_plan).
        Extension `"wavefront": K` (K >= 1): the whole GPU searches the ONE decision in waves of K leaves
        (b2_opd_plan_wave; K = 1 is again the strict order) -- 30-60x lower latency at K = 64..128."""
        from rl_agents_b200.engine.opd import OPDEngine, OPDSpeculativeEngine, OPDWaveEngine
        width = int(self.config.get("wavefront", 0) or 0)
        spec = self._speculative_width(d, width)
        if d.kind == _lib.ENV_INTERSECTION and spec == 0:
            width = max(width, 1)          # IntersectionLite lives in the whole-GPU kernels (width 1 = strict order)
        key = (d.kind, d.n_actions, self.config["budget"], self.config["gamma"],
               self.config.get("terminal_reward", 0), width, spec, mdp_fingerprint(d.mdp))

        def make():
            if spec > 0:
                return OPDSpeculativeEngine(d.kind, d.n_actions, self.config["budget"], self.config["gamma"], spec,
                                            self.config.get("terminal_reward", 0), mdp=d.mdp)
            if width > 0:
                return OPDWaveEngine(d.kind, d.n_actions, self.config["budget"], self.config["gamma"], width,
                                     self.config.get("terminal_reward", 0), mdp=d.mdp)
            return OPDEngine(d.kind, 1, d.n_actions, self.config["budget"], self.config["gamma"],
                             self.config.get("terminal_reward", 0), mdp=d.mdp,
                             keys_in_smem=self.config.get("keys_in_smem", True))
        return self.cached_engine(key, make)

    def plan(self, state, observation):
        d = describe(state)
        return self.search_host_ties(self._engine_for(d), d.root)


@register_with_reference
class DeterministicPlannerAgent(AbstractTreeSearchAgent):
    """An agent that performs optimistic planning in deterministic MDPs."""
    PLANNER_TYPE = OptimisticDeterministicPlanner
