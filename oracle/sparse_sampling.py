"""Flat CPU restatement of sparse sampling -- TEST INFRASTRUCTURE.

rl_agents/agents/tree_search/sparse_sampling.py (SparseSampling, DecisionNode, ChanceNode), with the random_argmax of
abstract.py it calls, over struct-of-arrays lists (node id = creation order).  Pinned against
tests/golden/golden_sparse_sampling.json, which tests/golden/make_golden_sparse_sampling.py records from the UNMODIFIED
reference (tests/test_sparse_sampling_oracle.py).

A finite-MDP sample is the env's own step: `default_rng(seed).choice(p.size, p=p)` on the row (what FiniteMDPLite.step
draws after `seed`).  HighwayLite is deterministic, so each (node, available action) is stepped once and the child gets
count C, after the C seed draws -- the reference's C identical samples.  The values are the reference's operations in
its order, so the digest also hashes the float64 bytes of `value`.
"""
import hashlib
import math

import numpy as np

from oracle import envs

DECISION, CHANCE = 0, 1
INT_FIELDS = ("parent", "kind", "key", "depth", "count")
FLOAT_FIELDS = ("value",)
HEAD = 64
# horizon 0: the root has no children and selection_rule's np.amax of its empty value list raises (:45-46, :53-56)
EMPTY_ROOT_MESSAGE = "zero-size array to reduction operation maximum which has no identity"


def tree_digest(tree):
    """Compact form of a creation-order dump (dict of per-node lists): a SHA-256 of the integer fields, a SHA-256 of
    the float64 bytes of `value`, its exact (math.fsum) sum, and the first HEAD nodes in full."""
    h = hashlib.sha256(np.array([[int(x) for x in tree[f]] for f in INT_FIELDS], dtype=np.int64).tobytes())
    value = np.array([float(x) for x in tree["value"]], dtype=np.float64)
    out = {"n_nodes": len(tree["parent"]), "structure_sha256": h.hexdigest(),
           "value_sha256": hashlib.sha256(value.tobytes()).hexdigest(), "sum_value": math.fsum(value.tolist())}
    for f in INT_FIELDS:
        out[f] = [int(x) for x in tree[f][:HEAD]]
    out["value"] = value[:HEAD].tolist()
    return out


class SSTree(object):
    """SoA dump: kind (DECISION / CHANCE), key (a chance node's action; a decision node's next state on a finite MDP,
    -1 on HighwayLite and at the root), depth, count (samples that reached a decision node, 0 on chance nodes),
    value."""

    def __init__(self):
        self.parent, self.kind, self.key, self.depth, self.count, self.value = [], [], [], [], [], []

    def new_node(self, parent, kind, key, depth):
        self.parent.append(parent)
        self.kind.append(kind)
        self.key.append(key)
        self.depth.append(depth)
        self.count.append(0)
        self.value.append(0)
        return len(self.parent) - 1

    def __len__(self):
        return len(self.parent)


def tree_dict(t):
    return {f: list(getattr(t, f)) for f in INT_FIELDS + FLOAT_FIELDS}


def check_config(config):
    """The reference's own failures on a bad config, or a ValueError where it would fail obscurely: KeyError for a
    missing horizon (read first, :45) or C (read once a chance node samples, :76), ValueError for horizon 0,
    horizon < 0 (RecursionError in the reference) and C < 1 (UnboundLocalError)."""
    horizon = config["horizon"]
    if horizon == 0:
        raise ValueError(EMPTY_ROOT_MESSAGE)
    C = config["C"]
    if horizon < 0 or C < 1:
        raise ValueError("sparse sampling needs horizon >= 1 and C >= 1 (got %r, %r)" % (horizon, C))
    return horizon, C


def sparse_sampling_plan(env, config, np_random):
    """SparseSampling.plan (:21-28) from a fresh root.  env: a FiniteMDPLite or HighwayLite (optionally wrapped in
    LegacyStepEnv); `config` the planner's completed config.  Returns (plan, tree, root chance values by action)."""
    horizon, C = check_config(config)
    gamma = config["gamma"]
    u = env.unwrapped
    highway = isinstance(u, envs.HighwayLite)
    n_actions = u.action_space.n
    t = SSTree()

    def actions_of(state):
        return envs.highway_available_actions(state) if highway else range(n_actions)

    def sample(state, action):
        """One finite-MDP sample of ChanceNode.estimateQ (:77-81): the seed draw, then the seeded env's step."""
        seed = np_random.integers(2 ** 30)
        m = u.mdp
        if m.mode == "deterministic":
            return int(m.transition[state, action])
        p = m.transition[state, action]
        k = int(np.random.default_rng(seed).choice(p.size, p=p))
        return k if m.mode == "stochastic" else int(m.next[state, action, k])

    def estimate_v(node, state):                                     # DecisionNode.estimateV (:38-51)
        depth = t.depth[node]
        if depth == horizon:
            return
        values = []
        for action in actions_of(state):
            c = t.new_node(node, CHANCE, int(action), depth)
            kids, kid_state = {}, {}
            if highway:
                for _ in range(C):
                    np_random.integers(2 ** 30)
                nxt = state.copy()
                reward = float(envs.highway_step(nxt, int(action))[0])
                k = t.new_node(c, DECISION, -1, depth + 1)
                t.count[k] = C
                kids[0], kid_state[k] = k, nxt
            else:
                reward = float(u.mdp.reward[state, action])
                for _ in range(C):
                    s2 = sample(state, action)
                    k = kids.get(str(s2))
                    if k is None:                                    # ChanceNode.get_child (:93-96)
                        k = kids[str(s2)] = t.new_node(c, DECISION, s2, depth + 1)
                        kid_state[k] = s2
                    t.count[k] += 1
            for k in kids.values():
                estimate_v(k, kid_state[k])
            t.value[c] = reward + gamma * sum(t.value[k] * t.count[k] for k in kids.values()) / C
            values.append(t.value[c])
        t.value[node] = np.amax(values)

    root = t.new_node(-1, DECISION, -1, 0)
    root_state = u.state.copy() if highway else u.mdp.state
    estimate_v(root, root_state)
    actions = [t.key[c] for c in range(len(t)) if t.parent[c] == root]
    values = [t.value[c] for c in range(len(t)) if t.parent[c] == root]
    indices = np.nonzero(np.array(values) == np.amax(values))[0]      # random_argmax (abstract.py:304-311)
    root_q = np.full(n_actions, np.nan)
    root_q[actions] = values
    return [actions[np_random.choice(indices)]], t, root_q
