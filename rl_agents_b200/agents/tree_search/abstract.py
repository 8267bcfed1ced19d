"""Agent / planner shells shared by the device tree-search planners.

Same observable behaviour as rl_agents/agents/tree_search/abstract.py
(AbstractTreeSearchAgent :15-106, AbstractPlanner :109-206) -- receding-horizon
schedule, env pre-processing, planner seeding through a numpy PCG64 Generator
(what gymnasium's seeding.np_random builds), `reset` tree-step strategy --
written independently of it.  The search itself lives on the device
(rl_agents_b200.engine).
"""
import logging
from collections import defaultdict

import numpy as np

from rl_agents_b200.agents.common.abstract import AbstractAgent
from rl_agents_b200.agents.common.factory import preprocess_env
from rl_agents_b200.configuration import Configurable

logger = logging.getLogger(__name__)


def np_random(seed=None):
    """gymnasium.utils.seeding.np_random: Generator(PCG64(SeedSequence(seed)))."""
    seed_seq = np.random.SeedSequence(seed)
    return np.random.Generator(np.random.PCG64(seed_seq)), seed_seq.entropy


def refuse_intersection(name, env):
    """BRUE, MDP-GapE and sparse sampling model finite MDPs and HighwayLite only: refuse an IntersectionLite env, both
    when the planner is built and when it is handed the env to plan on."""
    if getattr(getattr(env, "unwrapped", env), "b2_env_kind", None) == "intersection":
        raise NotImplementedError("%s runs on finite MDPs and HighwayLite, not on IntersectionLite" % name)


class _OpenLoopQueue(object):
    """Receding-horizon bookkeeping of a tree-search agent.

    A plan is an open-loop action sequence; config["receding_horizon"] = H lets H consecutive decisions be
    served from one plan before the planner runs again (H = 1, the default: replan at every step).  The
    queue is also spent when fewer than two actions are left.  Same observable schedule as the reference
    agent's plan()/step() pair (rl_agents/agents/tree_search/abstract.py:49-82)."""

    def __init__(self):
        self.actions = []     # what the last plan() call returned
        self.credit = 0       # decisions that may still be served without replanning

    def clear(self):
        self.credit = 0

    def must_replan(self):
        return self.credit == 0 or len(self.actions) < 2

    def refill(self, actions, horizon):
        self.actions, self.credit = actions, horizon - 1
        return actions

    def advance(self):
        self.actions, self.credit = self.actions[1:], self.credit - 1
        return self.actions


class AbstractTreeSearchAgent(AbstractAgent):
    """(env, config) plugin shell of the device planners: owns one planner (PLANNER_TYPE or
    make_planner()), hands it the pre-processed env at every replanning step, serves the rest of an
    open-loop plan for `receding_horizon` steps."""
    PLANNER_TYPE = None

    def __init__(self, env, config=None):
        super(AbstractTreeSearchAgent, self).__init__(config)
        self.env = env
        self.steps = 0
        self._queue = _OpenLoopQueue()
        self.planner = self.make_planner()

    @classmethod
    def default_config(cls):
        return dict(env_preprocessors=[], display_tree=False, receding_horizon=1, terminal_reward=0)

    def make_planner(self):
        if self.PLANNER_TYPE is None:
            raise NotImplementedError()
        return self.PLANNER_TYPE(self.env, self.config)

    # the reference exposes these two names; keep them readable for tools written against it
    @property
    def previous_actions(self):
        return self._queue.actions

    @property
    def remaining_horizon(self):
        return self._queue.credit

    def plan(self, observation):
        self.steps += 1
        replan = self.step(self._queue.actions)
        if not replan:
            return self._queue.advance()
        planning_env = preprocess_env(self.env, self.config["env_preprocessors"])
        return self._queue.refill(self.planner.plan(state=planning_env, observation=observation),
                                  self.config["receding_horizon"])

    def step(self, actions):
        """Tell the planner the env moved on by actions[0] (tree reuse / reset); -> whether to replan."""
        replan = self._queue.must_replan()
        self.planner.step_tree(actions)
        return replan

    def act(self, state):
        return self.plan(state)[0]

    def reset(self):
        self.planner.step_by_reset()
        self._queue.clear()
        self.steps = 0

    def seed(self, seed=None):
        return self.planner.seed(seed)

    def record(self, state, action, reward, next_state, done, info):
        pass        # planners do not learn

    def save(self, filename):
        return False

    def load(self, filename):
        return False


class AbstractPlanner(Configurable):
    def __init__(self, config=None):
        super(AbstractPlanner, self).__init__(config)
        self.np_random = None
        self.engine = None
        self._engine_key = None
        self.last_tree = None
        self.reset()
        self.seed()

    @classmethod
    def default_config(cls):
        return dict(budget=500, gamma=0.8, step_strategy="reset")

    def seed(self, seed=None):
        self.np_random, seed = np_random(seed)
        return [seed]

    def plan(self, state, observation):
        raise NotImplementedError()

    def cached_engine(self, key, make):
        """The engine make() built for `key`; a new one only when the key differs from the last call's."""
        if key != self._engine_key:
            self.engine = make()
            self._engine_key = key
        return self.engine

    def search_one_tree(self, engine, d, *plan_args):
        """One tree from the root of `d` (describe()) on the planner's own PCG64 stream, which the device
        advances -> (plan, result words of the tree)."""
        import torch
        from rl_agents_b200.engine.mcts import pcg64_words, set_pcg64_words
        root = torch.from_numpy(d.root.reshape(1, -1) if d.root.size > 1 else d.root).to(engine.device)
        engine.plan(root.contiguous(), pcg64_words(self.np_random).reshape(1, -1), *plan_args)
        plans, res, rng_words = engine.finish()
        set_pcg64_words(self.np_random, rng_words[0])
        self.last_tree = engine
        return plans[0], res[0]

    def search_host_ties(self, engine, root):
        """One tree from `root` (int32 host array: the root's state id or words; DROP: one row per model) on a
        value-bound engine, which completes its plan past a tie with the planner's generator -> the plan."""
        import torch
        engine.plan(torch.from_numpy(root).to(engine.device).contiguous())
        plans, _ = engine.finish([self.np_random])
        self.last_tree = engine
        return plans[0]

    def get_visits(self):
        return defaultdict(int)

    def get_updates(self):
        return defaultdict(int)

    def step_tree(self, actions):
        # the device planners rebuild the tree per decision: only "reset" applies
        # (OPD "subtree" crashes in the reference, SURVEY appendix B)
        if self.config["step_strategy"] != "reset":
            logger.warning("step strategy {} is not supported by the device planners: "
                           "resetting".format(self.config["step_strategy"]))
        self.step_by_reset()

    def step_by_reset(self):
        self.reset()

    def reset(self):
        self.last_tree = None
