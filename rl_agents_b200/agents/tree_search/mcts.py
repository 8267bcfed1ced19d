"""MCTS / UCT agent on the device engine.  Drop-in for
rl_agents.agents.tree_search.mcts.MCTSAgent (mcts.py:12-305, open loop)."""
import numpy as np

from rl_agents_b200.agents.common.abstract import register_with_reference
from rl_agents_b200.agents.tree_search.abstract import AbstractPlanner, AbstractTreeSearchAgent
from rl_agents_b200.envs.adapters import describe, mdp_fingerprint


def horizon_for(episodes, gamma):
    # OLOP.horizon (olop.py:42-44)
    return max(int(np.ceil(np.log(episodes) / (2 * np.log(1 / gamma)))), 1)


def allocation(budget, gamma):
    """OLOP.allocation (olop.py:50-62): budget -> (episodes, horizon)."""
    for episodes in range(1, int(budget)):
        if episodes * horizon_for(episodes, gamma) > budget:
            episodes = max(episodes - 1, 1)
            horizon = horizon_for(episodes, gamma)
            break
    else:
        raise ValueError("Could not split budget {} with gamma {}".format(budget, gamma))
    return episodes, horizon


def subtree_capacity(episodes, horizon, n_actions):
    """Nodes per tree under step_strategy "subtree": a node at depth d survives d re-rootings, so a tree holds up to
    horizon + 1 searches' expansions."""
    return 1 + (horizon + 1) * episodes * n_actions


class MCTS(AbstractPlanner):
    def __init__(self, env, prior_policy, rollout_policy, config=None):
        super(MCTS, self).__init__(config)
        self.env = env
        self.prior_policy = prior_policy
        self.rollout_policy = rollout_policy
        if not self.config["horizon"]:                                   # mcts.py:116-118
            self.config["episodes"], self.config["horizon"] = allocation(self.config["budget"], self.config["gamma"])
        # closed_loop (mcts.py:125,147,267-273) keys an extra node level on str(observation).  Within one plan() the
        # successor after a given action prefix is fixed: HighwayLite, IntersectionLite and deterministic finite MDPs
        # are deterministic, and the env copies of a stochastic finite MDP all replay the live env's generator (the
        # reference never reseeds them).  Every action node then has exactly one observation child carrying the same
        # statistics, so visit counts, values and the recommended action equal the open-loop search's (goldens:
        # tests/golden "mcts_closed_loop" and golden_mcts_stochastic.json, produced by the reference with
        # closed_loop=True).  The reference's get_plan interleaves the observation keys with the actions; here the
        # plan lists actions.

    @classmethod
    def default_config(cls):
        cfg = super(MCTS, cls).default_config()
        cfg.update({"temperature": 2 / (1 - cfg["gamma"]), "closed_loop": False})    # mcts.py:120-127
        return cfg

    def _engine_for(self, d, replicas, episodes):
        from rl_agents_b200.engine.mcts import MCTSEngine
        key = (d.kind, d.n_actions, replicas, episodes, self.config["horizon"], self.config["gamma"],
               self.config["temperature"], repr(self.rollout_policy), repr(self.prior_policy), mdp_fingerprint(d.mdp))

        def make():
            capacity = None
            if self.config["step_strategy"] == "subtree":
                capacity = subtree_capacity(episodes, self.config["horizon"], d.n_actions)
            engine = MCTSEngine(d.kind, replicas, d.n_actions, episodes, self.config["horizon"],
                                self.config["gamma"], self.config["temperature"], mdp=d.mdp,
                                rollout_policy=self.rollout_policy, prior_policy=self.prior_policy,
                                capacity=capacity)
            self._resume = 0
            return engine
        return self.cached_engine(key, make)

    def reset(self):
        super(MCTS, self).reset()
        self._resume = 0

    def step_tree(self, actions):
        """abstract.py:172-187: "reset" (default) or "subtree" (works for MCTS in the reference); "prior" is
        unreachable in the reference (mcts.py:186-190 is never called) and resets with a warning there too."""
        if self.config["step_strategy"] == "subtree":
            if actions and self.engine is not None and int(self.config.get("root_parallel", 1) or 1) <= 1 \
                    and self.last_tree is self.engine:
                self._resume = int(self.engine.reroot([actions[0]])[0])   # step_by_subtree (:195-206)
                if self._resume <= 0:
                    self.step_by_reset()
            else:
                self.step_by_reset()
        else:
            super(MCTS, self).step_tree(actions)

    def plan(self, state, observation):
        import torch
        from rl_agents_b200.engine.mcts import pcg64_words
        d = describe(state, env_words=True)
        replicas = int(self.config.get("root_parallel", 1) or 1)
        root = torch.from_numpy(d.root.reshape(1, -1) if d.root.size > 1 else d.root)
        width = int(self.config.get("wavefront", 0) or 0)
        if width > 0:
            # extension ("wavefront": W): the ONE decision searched by the whole GPU in waves of W episodes
            # (b2_mcts_plan_wave; specification oracle/planners.py::mcts_plan_wavefront).  The counter-based
            # generator is seeded from the planner's stream, so agent.seed() still fixes the result.
            from rl_agents_b200.engine.mcts import MCTSWaveEngine
            if self.rollout_policy != "random_available" or self.prior_policy != "random_available":
                raise NotImplementedError("wavefront MCTS implements the random_available policies")
            key = ("wave", d.kind, d.n_actions, self.config["episodes"], self.config["horizon"], self.config["gamma"],
                   self.config["temperature"], width, mdp_fingerprint(d.mdp))
            eng = self.cached_engine(key, lambda: MCTSWaveEngine(d.kind, d.n_actions, self.config["episodes"],
                                                                 self.config["horizon"], self.config["gamma"],
                                                                 self.config["temperature"], width, mdp=d.mdp))
            seed = int(self.np_random.integers(0, 2 ** 63 - 1))
            eng.plan(root.reshape(-1).to(eng.device).contiguous(), seed, d.env_words)
            plan, _ = eng.finish()
            self.last_tree = eng
            counts, values = eng.root_statistics()
            self.root_statistics = {"counts": counts, "values": values}
            return plan
        if replicas <= 1:
            # the reference's semantics: one tree, strict episode order, the planner's own RNG stream
            eng = self._engine_for(d, 1, self.config["episodes"])
            resume = [self._resume] if getattr(self, "_resume", 0) > 0 else None
            plan, _ = self.search_one_tree(eng, d, resume, d.env_words)
            self._resume = 0
            return plan
        # extension ("root_parallel": R): R independent trees of episodes/R episodes from the same root,
        # each on its own spawned stream; root statistics merged as in rl_agents_b200.distributed
        from rl_agents_b200.distributed import recommend
        episodes = -(-int(self.config["episodes"]) // replicas)
        eng = self._engine_for(d, replicas, episodes)
        gens = self.np_random.spawn(replicas)
        roots = root.repeat(replicas, 1) if d.root.size > 1 else root.repeat(replicas)
        # every replica copies the same env, so every replica's env copies start from the same generator words
        eng.plan(roots.to(eng.device).contiguous(), np.stack([pcg64_words(g) for g in gens]), None, d.env_words)
        plans, res, _ = eng.finish()
        self.last_tree = eng
        fc = eng.first_child[:, 0].cpu().numpy()
        counts = np.zeros(d.n_actions)
        sums = np.zeros(d.n_actions)
        per_replica = []
        for t in range(replicas):
            n = int((eng.meta[t, 0].item() >> 8) & 0xff)
            acts = (eng.meta[t, fc[t]:fc[t] + n].cpu().numpy() & 0xff).astype(int)
            c = eng.count[t, fc[t]:fc[t] + n].cpu().numpy().astype(float)
            v = eng.value[t, fc[t]:fc[t] + n].cpu().numpy()
            counts[acts] += c
            sums[acts] += c * v
            per_replica.append(dict(zip(acts.tolist(), c.tolist())))
        values = np.where(counts > 0, sums / np.maximum(counts, 1), 0.0)
        best = recommend(counts, values)
        donor = max(range(replicas), key=lambda t: per_replica[t].get(best, 0.0))
        tail = plans[donor][1:] if plans[donor] and plans[donor][0] == best else []
        self.root_statistics = {"counts": counts, "values": values}
        return [best] + tail


@register_with_reference
class MCTSAgent(AbstractTreeSearchAgent):
    """An agent that uses Monte Carlo Tree Search to plan a sequence of actions in an MDP."""

    def make_planner(self):
        return MCTS(self.env, MCTSAgent.policy_factory(self.config["prior_policy"]),
                    MCTSAgent.policy_factory(self.config["rollout_policy"]), self.config)

    @classmethod
    def default_config(cls):
        config = super(MCTSAgent, cls).default_config()
        config.update({"budget": 100, "horizon": None,
                       "prior_policy": {"type": "random_available"},
                       "rollout_policy": {"type": "random_available"},
                       "env_preprocessors": []})
        return config

    @staticmethod
    def policy_factory(policy_config):
        """mcts.py:34-44 -> the policy id the kernel implements."""
        kind = policy_config["type"]
        if kind in ("random", "random_available"):
            return kind
        if kind == "preference":                         # mcts.py:39-42: both keys are required there too
            return ("preference", policy_config["action"], policy_config["ratio"])
        raise ValueError("Unknown policy type")
