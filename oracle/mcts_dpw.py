"""Flat CPU restatement of MCTS with double progressive widening -- TEST INFRASTRUCTURE.

rl_agents/agents/tree_search/mcts_dpw.py (MCTSDPW, DecisionNode, ChanceNode), with the parts of mcts.py (MCTS.evaluate,
MCTSNode.update / selection_rule) and abstract.py (random_argmax) it calls, over struct-of-arrays lists (node id =
creation order).  Pinned against tests/golden/golden_mcts_dpw.json, which tests/golden/make_golden_mcts_dpw.py records
from the UNMODIFIED reference (tests/test_mcts_dpw_oracle.py).

One run (MCTSDPW.run, :59-90): seed the env copy with randint(2**30) of the planner's stream; descend while depth <
horizon, the last step was not terminal and the decision node has been visited (or is the root).  A decision node adds
a chance child for a new action, drawn with choice() from the unexplored actions in ascending id order, while
`k_action * N**alpha_action < len(children)` is false and not every available action has one; otherwise it picks the
first-maximum UCB index `value + temperature * sqrt(log(N / n))` with random_argmax.  After the step, the chance node
keys its child on sha1(str(obs))[:5] (closed loop) or on sha1("None")[:5] (open loop); an unseen key becomes a new
child while `k_state * N**alpha_state < len(children)` is false, otherwise choice() picks an existing child and the env
keeps the state it sampled.  A non-terminal run ends in MCTS.evaluate's rollout, and the return is backed up from the
last decision node to the root (count += 1; value += 1.0 / count * (total - value)).

The env's own generator (a FiniteMDPLite step draws `choice(p.size, p=p)` from it) is seeded once per run.  Values are
the reference's fp64 operations in its order, so the digest also hashes the float64 bytes of `value`.
"""
import copy
import hashlib
import math

import numpy as np

from oracle import envs
from oracle.planners import _policy

DECISION, CHANCE = 0, 1
INT_FIELDS = ("parent", "kind", "key", "count")
FLOAT_FIELDS = ("value",)
HEAD = 64


def obs_key(observation):
    """ChanceNode.get_child's key (:173): the first 5 hex digits of sha1(str(observation)), as a 20-bit integer."""
    return int(hashlib.sha1(str(observation).encode("UTF-8")).hexdigest()[:5], 16)


OPEN_LOOP_KEY = obs_key(None)       # closed_loop False: every observation is keyed as None (:79)


def tree_digest(tree):
    """Compact form of a creation-order dump (dict of per-node lists): a SHA-256 of the integer fields, a SHA-256 of
    the float64 bytes of `value`, its exact (math.fsum) sum, and the first HEAD nodes in full.  Every node's children
    are in creation order (dict insertion order), so the integer fields fix the child order."""
    h = hashlib.sha256(np.array([[int(x) for x in tree[f]] for f in INT_FIELDS], dtype=np.int64).tobytes())
    value = np.array([float(x) for x in tree["value"]], dtype=np.float64)
    out = {"n_nodes": len(tree["parent"]), "structure_sha256": h.hexdigest(),
           "value_sha256": hashlib.sha256(value.tobytes()).hexdigest(), "sum_value": math.fsum(value.tolist())}
    for f in INT_FIELDS:
        out[f] = [int(x) for x in tree[f][:HEAD]]
    out["value"] = value[:HEAD].tolist()
    return out


class DPWTree(object):
    """SoA dump: kind (DECISION / CHANCE), key (a chance node's action; a decision node's 20-bit observation key, -1
    at the root), count, value; children[i] in creation order, keyed[i] a chance node's children by key.  state_draws:
    how often state widening blocked a new state and choice() picked an existing child."""

    def __init__(self):
        self.parent, self.kind, self.key, self.count, self.value = [], [], [], [], []
        self.children, self.keyed = [], []
        self.state_draws = 0

    def new_node(self, parent, kind, key):
        i = len(self.parent)
        self.parent.append(parent)
        self.kind.append(kind)
        self.key.append(key)
        self.count.append(0)
        self.value.append(0)
        self.children.append([])
        self.keyed.append({})
        if parent >= 0:
            self.children[parent].append(i)
            self.keyed[parent][key] = i
        return i

    def __len__(self):
        return len(self.parent)


def tree_dict(t):
    return {f: list(getattr(t, f)) for f in INT_FIELDS + FLOAT_FIELDS}


def check_config(config):
    """What the device refuses up front: horizon < 1 (the root stays childless and get_plan returns None) and
    step_strategy "subtree" (it re-roots on a chance node, and the next run fails there)."""
    if config["step_strategy"] == "subtree":
        raise NotImplementedError("MCTS-DPW supports step_strategy 'reset' only")
    if config["horizon"] < 1:
        raise ValueError("MCTS-DPW needs horizon >= 1 (got %r): the root would stay childless" % config["horizon"])


def mcts_dpw_plan(env, config, np_random):
    """MCTSDPW.plan (mcts.py:179-184 with mcts_dpw.py:59-94) from a fresh root.  env: a FiniteMDPLite or HighwayLite
    (optionally wrapped in LegacyStepEnv); `config` the planner's completed config.  Returns (action, tree, env steps)."""
    check_config(config)
    u = env.unwrapped
    highway = isinstance(u, envs.HighwayLite)
    n_actions = u.action_space.n
    episodes, horizon, gamma = config["episodes"], config["horizon"], config["gamma"]
    temperature, closed_loop = config["temperature"], config["closed_loop"]
    k_a, a_a, k_s, a_s = config["k_action"], config["alpha_action"], config["k_state"], config["alpha_state"]
    t = DPWTree()
    root = t.new_node(-1, DECISION, -1)
    steps = 0
    for _ in range(episodes):
        state = copy.deepcopy(u)                                     # safe_deepcopy_env, mcts.py:183
        state.seed(np_random.integers(2 ** 30))                      # :69
        node, total, depth, terminal = root, 0, 0, False
        while depth < horizon and not terminal and (t.count[node] != 0 or node == root):
            kids, N = t.children[node], t.count[node]
            available = envs.highway_available_actions(state.state) if highway else list(range(n_actions))
            if len(kids) == len(available) or k_a * N ** a_a < len(kids):          # get_child, :120-127
                x = [t.value[c] + temperature * np.sqrt(np.log(N / t.count[c])) for c in kids]
                indices = np.nonzero(x == np.amax(x))[0]             # random_argmax (abstract.py:304-311)
                chance = kids[np_random.choice(indices)]
            else:
                # expand (:115-118): list() of a set of ints below 8 iterates in ascending order
                unexplored = sorted(set(t.key[c] for c in kids).symmetric_difference(available))
                chance = t.new_node(node, CHANCE, int(np_random.choice(unexplored)))
            obs, reward, terminal, _, _ = state.step(t.key[chance])  # truncation dropped (:76)
            steps += 1
            key = obs_key(obs) if closed_loop else OPEN_LOOP_KEY
            node = t.keyed[chance].get(key)                          # ChanceNode.get_child (:171-182)
            if node is None:
                if k_s * t.count[chance] ** a_s < len(t.children[chance]):
                    node = t.keyed[chance][np_random.choice(list(t.keyed[chance]))]
                    t.state_draws += 1
                else:
                    node = t.new_node(chance, DECISION, key)
            total += gamma ** depth * reward
            depth += 1
        if not terminal:                                             # MCTS.evaluate (mcts.py:160-177)
            for h in range(depth, horizon):
                actions, probs = _policy(config["rollout_policy"], state)
                a = np_random.choice(actions, 1, p=np.array(probs))[0]
                _, reward, term, trunc, _ = state.step(a)
                steps += 1
                total += gamma ** h * reward
                if term or trunc:
                    break
        while node >= 0:                                             # backup_to_root, update (mcts.py:248-255)
            t.count[node] += 1
            t.value[node] += 1.0 / t.count[node] * (total - t.value[node])
            node = t.parent[node]
    kids = t.children[root]                                          # get_plan: root.selection_rule (mcts.py:212-218)
    counts = np.array([t.count[c] for c in kids])
    ties = np.nonzero(counts == np.amax(counts))[0]
    best = max(ties, key=lambda i: t.value[kids[i]])
    return t.key[kids[best]], t, steps
