"""Flat CPU restatement of PlaTyPOOS -- TEST INFRASTRUCTURE.

rl_agents/agents/tree_search/platypoos.py (PlaTyPOOS, PlaTyPOOSNode) over struct-of-arrays lists (node id = creation
order).  Pinned against tests/golden/golden_platypoos.json, which tests/golden/make_golden_platypoos.py records from the
UNMODIFIED reference (tests/test_platypoos_oracle.py).

This restatement steps the env on EVERY sample, as the reference does: a deep copy of the node's state, `seed(
np_random.integers(2**30))`, `step(action)`.  The device kernel steps once per created child (the reward and `done` of a
step depend only on the node's state and the action on every model here), so the oracle is an independent check of that
shortcut.  The root's value is 0.0 (the reference's root has no `value` attribute; see agents/tree_search/platypoos.py).

plan: the root expanded h_max times per available action; explore(h) for h = 1 .. h_max - 1 (stable descending sort of
the layer by value, selection for p = p_top(h) .. 0, expansion in selection order, candidates[p] kept by a strict
`>`); cross-validation of every candidate in dict order up to and including the root; the actions from the root to the
first candidate of highest value.
"""
import copy

import numpy as np

from oracle import envs

INT_FIELDS = ("parent", "action", "depth", "count", "done", "to_expand")
FLOAT_FIELDS = ("cumulative_reward", "value")
EMPTY_CANDIDATES_MESSAGE = "max() iterable argument is empty"


def horizon_of(budget, n_actions):
    """The reference's h_max (platypoos.py:22-25) when the config has no "horizon"."""
    expansion_budget = budget / n_actions
    return int(np.floor(expansion_budget / (2 * (np.log2(expansion_budget) + 1) ** 2)))


def p_top(h, h_max, gamma):
    return max(int(np.floor(np.log2(h_max / np.ceil(h ** 2 * gamma ** (2 * h))))), 0)


def layer_quotas(h, p, h_max, gamma):
    """(nodes_count, evaluations, min_visits) of explore(h) at p (platypoos.py:44-46)."""
    nodes_count = int(np.floor(h_max / h * np.ceil(h * 2 ** p * gamma ** (2 * h))))
    evaluations = int(np.ceil(h * 2 ** p * gamma ** (2 * h)))
    min_visits = int(np.ceil((h - 1) * 2 ** p * gamma ** (2 * (h - 1))))
    return nodes_count, evaluations, min_visits


def cross_validation_count(depth, h_max, gamma):
    """The evaluations of cross_validate at a node of depth `depth` (platypoos.py:75-76)."""
    return int(np.floor((depth + 1) * 5 * h_max * gamma ** (2 * depth) * (1 - gamma ** 2) ** 2))


class PTree(object):
    """SoA dump in creation order; children[i] maps action -> node id in insertion order; state[i] the env copy the
    node was created with (the root's is the planning env)."""

    def __init__(self, root_state):
        self.parent, self.action, self.depth, self.count = [-1], [-1], [0], [0]
        self.cumulative_reward, self.value, self.done, self.to_expand = [0.0], [0.0], [0], [0]
        self.children, self.state = [{}], [root_state]

    def new_node(self, parent, action, state):
        i = len(self.parent)
        self.parent.append(parent)
        self.action.append(action)
        self.depth.append(self.depth[parent] + 1)
        self.count.append(0)
        self.cumulative_reward.append(0)
        self.value.append(0.0)
        self.done.append(0)
        self.to_expand.append(0)
        self.children.append({})
        self.state.append(state)
        self.children[parent][action] = i
        return i

    def __len__(self):
        return len(self.parent)


def tree_dict(t):
    out = {f: [int(x) for x in getattr(t, f)] for f in INT_FIELDS}
    for f in FLOAT_FIELDS:
        out[f] = [float(x) for x in getattr(t, f)]
    return out


def check_config(config):
    if config["step_strategy"] == "subtree":
        raise NotImplementedError("PlaTyPOOS supports step_strategy 'reset' only")


def platypoos_plan(env, config, np_random):
    """PlaTyPOOS.plan from a fresh root.  env: a FiniteMDPLite or HighwayLite (optionally wrapped in LegacyStepEnv);
    config: the planner's completed config (its "horizon" set).  Returns (plan, tree, openings, candidates), the
    candidates as [(p, node id)] in dict order."""
    check_config(config)
    u = env.unwrapped
    highway = isinstance(u, envs.HighwayLite)
    n_actions = u.action_space.n
    h_max, gamma = config["horizon"], config["gamma"]
    t = PTree(u)
    stats = {"openings": 0}

    def actions_of(state):
        return envs.highway_available_actions(state.state) if highway else range(1, n_actions)

    def expand(node, next_layer, count):
        stats["openings"] += count
        if t.done[node]:
            return
        actions = actions_of(t.state[node])
        for _ in range(count):
            for a in actions:
                state = copy.deepcopy(t.state[node])
                state.seed(int(np_random.integers(2 ** 30)))
                _, reward, done, _, _ = state.step(a)
                child = t.children[node].get(a)
                if child is None:
                    child = t.new_node(node, a, state)
                    next_layer.append(child)
                t.cumulative_reward[child] += reward
                t.count[child] += 1
                t.value[child] = t.value[node] + gamma ** (t.depth[child] - 1) * (
                    t.cumulative_reward[child] / t.count[child])
                t.done[child] = int(bool(done))

    candidates = {}
    layer = []
    expand(0, layer, h_max)
    for h in range(1, h_max):
        ordered = sorted(layer, key=lambda n: t.value[n], reverse=True)
        to_expand = []
        for p in range(p_top(h, h_max, gamma), -1, -1):
            nodes_count, evaluations, min_visits = layer_quotas(h, p, h_max, gamma)
            for n in ordered:
                if t.count[n] > min_visits and not t.to_expand[n]:
                    t.to_expand[n] = 1
                    to_expand.append((n, evaluations, p))
                if len(to_expand) >= nodes_count:
                    break
        layer = []
        for n, evaluations, p in to_expand:
            expand(n, layer, evaluations)
            if p not in candidates or t.value[n] > t.value[candidates[p]]:
                candidates[p] = n
    for n in candidates.values():
        while n >= 0:
            expand(n, [], cross_validation_count(t.depth[n], h_max, gamma))
            n = t.parent[n]
    if not candidates:
        raise ValueError(EMPTY_CANDIDATES_MESSAGE)
    best = max(candidates.values(), key=lambda n: t.value[n])
    plan = []
    while t.parent[best] >= 0:
        plan.insert(0, t.action[best])
        best = t.parent[best]
    return plan, t, stats["openings"], list(candidates.items())
