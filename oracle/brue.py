"""Flat CPU restatement of BRUE -- TEST INFRASTRUCTURE.

rl_agents/agents/tree_search/brue.py (BRUE, DecisionNode, ChanceNode), with the parts of olop.py and abstract.py it
calls, over struct-of-arrays lists (node id = creation order).  Pinned against tests/golden/golden_brue.json, which
tests/golden/make_golden_brue.py records from the UNMODIFIED reference (tests/test_brue_oracle.py).

BRUE's statistics are incremental means, gamma**d products and arg-maxes, so every float here equals the
reference's bit for bit; the digest therefore also hashes the float64 bytes of `value`.
"""
import copy
import hashlib
import math

import numpy as np

from oracle.planners import olop_allocation

DECISION, CHANCE = 0, 1
INT_FIELDS = ("parent", "action", "kind", "depth", "count")
FLOAT_FIELDS = ("value",)
HEAD = 64
# np.amax of the root's empty value list when no rollout ran (budget <= 0, brue.py:68-75, abstract.py:301)
EMPTY_ROOT_MESSAGE = "zero-size array to reduction operation maximum which has no identity"


def tree_digest(tree):
    """Compact form of a creation-order tree dump (dict of per-node lists): a SHA-256 of the integer fields, a
    SHA-256 of the float64 bytes of `value`, its exact (math.fsum) sum, and the first HEAD nodes in full.  A decision
    node's children are in creation order (dict insertion order), so the integer fields fix the child order."""
    h = hashlib.sha256(np.array([[int(x) for x in tree[f]] for f in INT_FIELDS], dtype=np.int64).tobytes())
    value = np.array([float(x) for x in tree["value"]], dtype=np.float64)
    out = {"n_nodes": len(tree["parent"]), "structure_sha256": h.hexdigest(),
           "value_sha256": hashlib.sha256(value.tobytes()).hexdigest(), "sum_value": math.fsum(value.tolist())}
    for f in INT_FIELDS:
        out[f] = [int(x) for x in tree[f][:HEAD]]
    out["value"] = value[:HEAD].tolist()
    return out


class BRUETree(object):
    """SoA dump: kind (DECISION / CHANCE), action (a chance node's action, -1 for decision nodes), depth, count,
    value (a chance node's value, a decision node's mean reward); children[i] in creation order."""

    def __init__(self):
        self.parent, self.action, self.kind, self.depth, self.count, self.value = [], [], [], [], [], []
        self.children, self.keys = [], []

    def new_node(self, parent, action, kind, depth):
        i = len(self.parent)
        self.parent.append(parent)
        self.action.append(action)
        self.kind.append(kind)
        self.depth.append(depth)
        self.count.append(0)
        self.value.append(0)
        self.children.append([])
        self.keys.append({})
        if parent >= 0:
            self.children[parent].append(i)
        return i

    def child(self, node, key, kind, action, depth):
        """DecisionNode.get_child / ChanceNode.get_child: the child under `key`, created on the first visit."""
        c = self.keys[node].get(key)
        if c is None:
            c = self.keys[node][key] = self.new_node(node, action, kind, depth)
        return c

    def __len__(self):
        return len(self.parent)


def tree_dict(t):
    """The dump of a tree returned by brue_plan, in the form tree_digest reads."""
    return {f: list(getattr(t, f)) for f in INT_FIELDS + FLOAT_FIELDS}


def brue_horizon(config, n_actions):
    """BRUE.reset (brue.py:19-22): the configured horizon, else OLOP.allocate_budget's (olop.py:46-48)."""
    if "horizon" in config:
        return config["horizon"]
    return olop_allocation(max(n_actions, config["budget"]), config["gamma"])[1]


def brue_plan(env, config, np_random):
    """BRUE.plan (brue.py:66-71) from a fresh root.  `config` is the planner's completed config; `env.step` follows
    the legacy 4-tuple API brue.py:28 expects.

    Returns (plan, tree, rollouts); tree.budget_left is `available_budget` afterwards (<= 0: the last rollout runs
    to its end whatever budget is left)."""
    gamma = config["gamma"]
    n_actions = env.action_space.n
    horizon = brue_horizon(config, n_actions)
    if horizon < 1:
        raise ValueError("BRUE needs horizon >= 1 (the reference's rollout loop never ends otherwise)")
    t = BRUETree()

    def update(node, x):                                             # DecisionNode / ChanceNode.update (:84-86, :106-108)
        t.count[node] += 1
        c = t.count[node]
        t.value[node] = (c - 1) / c * t.value[node] + x / c

    def estimate(node):                                              # :52-64
        return_ = 0
        for d in range(horizon - t.depth[node]):
            if not t.children[node]:
                break
            chance = max(t.children[node], key=lambda c: t.value[c])
            next_states = t.children[chance]
            counts = np.array([t.count[s] for s in next_states])
            node = next_states[np_random.choice(len(next_states), p=counts / counts.sum())]
            return_ += gamma ** d * t.value[node]
        return return_

    root = t.new_node(-1, -1, DECISION, 0)
    available_budget = config["budget"]
    rollouts = 0
    while available_budget > 0:
        state = copy.deepcopy(env)                                   # safe_deepcopy_env, :69
        state.seed(np_random.randint(2 ** 30))                       # rollout (:24-33)
        node, path = root, []
        for _ in range(horizon):
            action = np_random.randint(n_actions)
            obs, reward, done = state.step(action)[:3]
            chance = t.child(node, action, CHANCE, int(action), t.depth[node])
            nxt = t.child(chance, str(obs), DECISION, -1, t.depth[node] + 1)
            path.append((chance, reward, nxt))
            node = nxt
            available_budget -= 1
            if done:
                break
        rollouts += 1
        for chance, reward, nxt in reversed(path):                  # update (:35-50)
            update(nxt, reward)
            update(chance, reward + gamma * estimate(nxt))
    t.horizon, t.budget_left = horizon, available_budget
    values = [t.value[c] for c in t.children[root]]                  # get_plan: root.selection_rule (:73-91)
    if not values:
        raise ValueError(EMPTY_ROOT_MESSAGE)
    indices = np.nonzero(np.array(values) == np.amax(values))[0]
    return [t.action[t.children[root][np_random.choice(indices)]]], t, rollouts
