"""DROP agent on the device engine.  Drop-in for
rl_agents.agents.robust.robust.DiscreteRobustPlannerAgent (robust.py:50-71): `config["models"]` lists one
env-preprocessor chain per model; every decision plans on the joint env of the M resulting models with
OPD on the minima over the models of the per-model bounds (RobustNode, robust.py:40-47).

The reference's JointEnv.step (robust.py:13-16) returns the legacy 4-tuple, which its own
DeterministicNode.expand (deterministic.py:41) cannot unpack; the golden vectors this agent is pinned
against come from the unmodified planner classes with that tuple re-packed (tests/golden/make_golden.py)."""
import numpy as np

from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.common.factory import preprocess_env
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner
from rl_agents_b200.agents.tree_search.deterministic import DeterministicPlannerAgent
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


class DiscreteRobustPlanner(AbstractPlanner):
    """plan(): one DROP decision, searched by libb2planner (b2_opd_plan_wave with n_models = M)."""

    def __init__(self, env, config=None):
        super(DiscreteRobustPlanner, self).__init__(config)
        self.env = env

    def plan(self, state, observation):
        """state: the list of the M model envs (what JointEnv holds as joint_state)."""
        from rl_agents_b200.engine.opd import OPDWaveEngine
        models = list(state)
        descs = [describe(m) for m in models]
        kinds = set(d.kind for d in descs)
        if len(kinds) != 1 or len(set(d.n_actions for d in descs)) != 1:
            raise ValueError("the models of a joint env must share the env kind and the action space")
        d0 = descs[0]
        width = max(1, int(self.config.get("wavefront", 1) or 1))          # 1: the reference's strict order
        key = (d0.kind, d0.n_actions, len(models), self.config["budget"], self.config["gamma"],
               self.config.get("terminal_reward", 0), width, tuple(mdp_fingerprint(d.mdp) for d in descs))
        eng = self.cached_engine(key, lambda: OPDWaveEngine(d0.kind, d0.n_actions, self.config["budget"],
                                                            self.config["gamma"], width,
                                                            self.config.get("terminal_reward", 0), n_models=len(models),
                                                            model_mdps=[d.mdp for d in descs] if d0.mdp is not None
                                                            else None))
        return self.search_host_ties(eng, np.stack([d.root.reshape(-1) for d in descs]))


@register_with_reference
class DiscreteRobustPlannerAgent(DeterministicPlannerAgent):
    """An agent that plans robustly over a finite set of dynamics models (DROP)."""
    PLANNER_TYPE = DiscreteRobustPlanner

    def __init__(self, env, config=None):
        self.true_env = env
        super(DiscreteRobustPlannerAgent, self).__init__(env, config)

    @classmethod
    def default_config(cls):
        config = super(DiscreteRobustPlannerAgent, cls).default_config()
        config.update(dict(models=[]))
        return config

    def plan(self, observation):
        # robust.py:66-68: one preprocessed copy of the true env per model; the joint env is what is planned on
        self.env = [preprocess_env(self.true_env, preprocessors) for preprocessors in self.config["models"]]
        return super(DiscreteRobustPlannerAgent, self).plan(observation)
