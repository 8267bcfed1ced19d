"""Flat CPU restatement of MDP-GapE -- TEST INFRASTRUCTURE.

rl_agents/agents/tree_search/mdp_gape.py (MDPGapE, DecisionNode, ChanceNode), with the parts of olop.py and
rl_agents/utils.py it calls, over struct-of-arrays lists (node id = creation order).  Pinned against
tests/golden/golden_mdp_gape.json, which tests/golden/make_golden_mdp_gape.py records from the UNMODIFIED
reference (tests/test_mdp_gape_oracle.py).

Kept in its own module so that oracle/planners.py stays as the other goldens pinned it; it reuses that module's
helpers (allocation, Bernoulli KL, tree record).
"""
import copy
import hashlib
import json
import math

import numpy as np

from oracle.planners import Tree, _available_actions, bernoulli_kl, olop_allocation

DECISION, CHANCE = 0, 1
INT_FIELDS = ("parent", "action", "kind", "depth", "count", "done")
FLOAT_FIELDS = ("cumulative_reward", "mu_ucb", "mu_lcb", "upper", "lower")
HEAD = 64


def tree_digest(tree):
    """Compact form of a creation-order tree dump (dict of per-node lists + `order`, the chance nodes' child order):
    a SHA-256 of the integer fields and the child orders, the exact (math.fsum) sum of every float field over the
    nodes that carry it, and the first HEAD nodes in full."""
    h = hashlib.sha256(np.array([[int(x) for x in tree[f]] for f in INT_FIELDS], dtype=np.int64).tobytes())
    h.update(json.dumps({str(c): [int(x) for x in o] for c, o in tree["order"].items()}, sort_keys=True).encode())
    out = {"n_nodes": len(tree["parent"]), "structure_sha256": h.hexdigest()}
    for f in FLOAT_FIELDS:
        out["sum_" + f] = math.fsum(float(x) for x in tree[f] if x is not None)
    for f in INT_FIELDS + FLOAT_FIELDS:
        out[f] = [None if x is None else (int(x) if f in INT_FIELDS else float(x)) for x in tree[f][:HEAD]]
    return out


def tree_dict(t):
    """The dump of a tree returned by mdp_gape_plan, in the form tree_digest reads."""
    out = {f: list(getattr(t, f)) for f in INT_FIELDS + FLOAT_FIELDS}
    out["order"] = t.order
    return out


def kl_bound(_sum, count, threshold=1, eps=1e-2, lower=False):
    """kl_upper_bound (utils.py:123-147) through newton_iteration (:150-203), upper or lower bound:
    the root of KL(mu, q) = threshold / count on [mu, 1] (upper) or [0, mu] (lower)."""
    if count == 0:
        return 0 if lower else 1
    mu = _sum / count
    max_div = threshold / count
    a, b = (0, mu) if lower else (mu, 1)
    x = math.inf
    x_next = (a + b) / 2
    if a == b:
        return a
    iterations = 0
    while abs(x - x_next) > eps and iterations < 100:
        iterations += 1
        x = x_next
        f_x = bernoulli_kl(mu, x) - max_div
        try:
            df_x = (1 - mu) / (1 - x) - mu / x
        except ZeroDivisionError:
            df_x = (f_x - (bernoulli_kl(mu, x - eps) - max_div)) / eps
        if df_x != 0:
            x_next = x - f_x / df_x
        if x_next < a:
            x_next = 0.9 * a + (1 - 0.9) * x
        elif x_next > b:
            x_next = 0.9 * b + (1 - 0.9) * x
    if x_next < a:
        x_next = a
    if x_next > b:
        x_next = b
    return x_next


def max_expectation_one_positive(f, q, c):
    """max_expectation_under_constraint (utils.py:292-342) for a distribution q with exactly ONE positive
    element -- the only case a chance node of a deterministic env produces (one observed next state, the other
    max_next_states_count - 1 children are unobserved placeholders).  Then no Newton solve happens: either the
    mass z = 1 - exp(theta(f*)) moves to the best unobserved entries (theta_func, utils.py:279-282, evaluated
    with the C library's log like the numba-compiled reference), or q itself is returned.  The operations and
    their order are the reference's."""
    x_plus = np.where(q > 0)
    x_zero = np.where(q == 0)
    if x_plus[0].size != 1:
        raise NotImplementedError("only one observed next state per chance node is restated")
    p_star = np.zeros(q.shape)
    lambda_, z = None, 0
    q_p = q[x_plus]
    f_p = f[x_plus]
    f_star = np.amax(f)
    if f_star > np.amax(f_p):
        d = float(f_star - f_p[0])
        w = float(q_p[0])
        theta_star = w * math.log(d) + math.log(w * (1 / d)) - c
        if theta_star < 0:
            lambda_ = f_star
            z = 1 - np.exp(theta_star)
            p_star[x_zero] = 1.0 * (f[x_zero] == np.amax(f[x_zero]))
            p_star[x_zero] *= z / p_star[x_zero].sum()
    if lambda_ is None:
        return q
    beta = (1 - z) / (q_p @ (1 / (lambda_ - f_p)))
    if beta != 0:
        p_star[x_plus] = beta * q_p / (lambda_ - f_p)
    return p_star


def mdp_gape_allocation(config, n_actions):
    """MDPGapE.reset / allocate_budget (mdp_gape.py:42-58): -> (episodes, horizon)."""
    if "horizon" in config:
        return config["episodes"], config["horizon"]
    if config.get("horizon_from_accuracy", False):
        gamma = config["gamma"]
        horizon = int(np.ceil(np.log(config["accuracy"] * (1 - gamma) / 2) / np.log(gamma)))
        episodes = config["budget"] // horizon
        assert episodes > 1
        return episodes, horizon
    return olop_allocation(max(n_actions, config["budget"]), config["gamma"])


def mdp_gape_plan(env, config, np_random):
    """MDPGapE.plan (mdp_gape.py:94-110) from a fresh root (:42-45).  `config` is the planner's completed
    config; `env.step` follows the legacy 4-tuple API mdp_gape.py:82 expects.

    Returns (plan, tree, episodes_run).  Tree fields per node: kind (DECISION / CHANCE), action (the action of a
    chance node; the placeholder index of a decision node below a chance node; -1 at the root), depth, count,
    done, value_upper / value_lower as `upper` / `lower`; decision nodes also carry cumulative_reward, mu_ucb,
    mu_lcb (None on chance nodes, which have no such attributes).  `t.order[c]` lists the children of chance
    node c in the reference's dict order (observed placeholders moved to the end, :272-286)."""
    gamma = config["gamma"]
    n_actions = env.action_space.n
    episodes, horizon = mdp_gape_allocation(config, n_actions)
    ub = config["upper_bound"]
    if ub["type"] != "kullback-leibler":
        raise NotImplementedError("MDP-GapE is restated for the kullback-leibler upper bound only")
    uniform = config["continuation_type"] == "uniform"
    n_next = config["max_next_states_count"]
    scope = {"np": np, "horizon": horizon, "actions": n_actions, "confidence": config["confidence"],
             "time": episodes}

    def threshold(expr, count):
        return eval(expr, dict(scope, count=count))

    t = Tree()
    t.kind, t.cumulative_reward, t.mu_ucb, t.mu_lcb, t.upper, t.lower, t.done = [], [], [], [], [], [], []
    t.order, t.keys = {}, {}

    def new_node(parent, action, kind, depth):
        t.parent.append(parent)
        t.action.append(action)
        t.kind.append(kind)
        t.depth.append(depth)
        t.count.append(0)
        t.first_child.append(-1)
        t.n_children.append(0)
        t.upper.append((1 - gamma ** (horizon - depth)) / (1 - gamma))        # :145-147, :257-258
        t.lower.append(0)
        t.done.append(False)
        decision = kind == DECISION
        t.cumulative_reward.append(0 if decision else None)
        t.mu_ucb.append(1 if decision else None)
        t.mu_lcb.append(0 if decision else None)
        return len(t.parent) - 1

    def expand_decision(node, state):                                           # :162-170
        actions = _available_actions(state)
        t.first_child[node], t.n_children[node] = len(t.parent), len(actions)
        for a in actions:
            new_node(node, int(a), CHANCE, t.depth[node])

    def children(node):
        return list(t.children(node))

    def bai(node):                                                              # :228-249
        kids = children(node)
        gap = {}
        for c in kids:
            g = -np.inf
            for o in kids:
                if o != c:
                    g = max(g, t.upper[o] - t.lower[c])
            gap[c] = g
        best = min(kids, key=lambda c: gap[c])
        challenger = max([c for c in kids if c != best], key=lambda c: t.upper[c])
        return max([best, challenger], key=lambda c: t.upper[c] - t.lower[c]), best, challenger

    root = new_node(-1, -1, DECISION, 0)
    episode, done = 0, False
    while not done:
        state = copy.deepcopy(env)                                              # safe_deepcopy_env, :98
        state.seed(np_random.randint(2 ** 30))                                  # :67
        if t.n_children[root] == 0:
            expand_decision(root, state)                                        # :69-73
        node = root
        for _ in range(horizon):
            if node == root:                                                    # sampling_rule (:183-198)
                selected, _, _ = bai(root)
                action = t.action[selected]
            elif t.n_children[node]:
                kids = children(node)
                x = np.array([t.upper[c] for c in kids])
                action = t.action[kids[np_random.choice(np.nonzero(x == np.amax(x))[0])]]
            else:
                action = np_random.randint(n_actions) if uniform else 0
            if t.n_children[node] == 0:                                         # get_child (:155-160)
                expand_decision(node, state)
            kids = children(node)
            chance = next((c for c in kids if t.action[c] == action), kids[0])
            obs, reward, terminal = state.step(t.action[chance])[:3]
            if t.n_children[chance] == 0:                                       # ChanceNode.expand (:267-270)
                t.first_child[chance], t.n_children[chance] = len(t.parent), n_next
                for i in range(n_next):
                    new_node(chance, i, DECISION, t.depth[chance] + 1)
                t.order[chance] = children(chance)
                t.keys[chance] = ["placeholder_%d" % i for i in range(n_next)]
            key = str(obs)                                                      # ChanceNode.get_child (:272-286)
            keys, order = t.keys[chance], t.order[chance]
            if key not in keys:
                for i in range(n_next):
                    if "placeholder_%d" % i in keys:
                        j = keys.index("placeholder_%d" % i)
                        keys.append(key)
                        keys.pop(j)
                        order.append(order.pop(j))
                        break
                else:
                    raise ValueError("No more placeholder nodes available, we observed more next states than "
                                     "the 'max_next_states_count' config")
            node = order[keys.index(key)]
            t.count[chance] += 1                                                # ChanceNode.update (:264-265)
            if not 0 <= reward <= 1:                                            # OLOPNode.update (olop.py:132-142)
                raise ValueError("This planner assumes that all rewards are normalized in [0, 1]")
            if terminal:
                t.done[node] = True
            if t.done[node]:
                reward = 0
            t.cumulative_reward[node] += reward
            t.count[node] += 1
            thr = threshold(ub["threshold"], t.count[node])                     # compute_reward_ucb (:200-212)
            t.mu_ucb[node] = kl_bound(t.cumulative_reward[node], t.count[node], thr)
            t.mu_lcb[node] = kl_bound(t.cumulative_reward[node], t.count[node], thr, lower=True)
        n = node                                                                # backup_to_root
        while n >= 0:
            if t.kind[n] == DECISION:                                           # :214-226
                if t.n_children[n]:
                    t.upper[n] = np.amax([t.upper[c] for c in children(n)])
                    t.lower[n] = np.amax([t.lower[c] for c in children(n)])
                else:
                    assert t.depth[n] == horizon
                    t.upper[n], t.lower[n] = 0, 0
            else:                                                               # :288-305
                kids = t.order[n]
                u_next = np.array([t.mu_ucb[c] + gamma * t.upper[c] for c in kids])
                l_next = np.array([t.mu_lcb[c] + gamma * t.lower[c] for c in kids])
                p_hat = np.array([t.count[c] for c in kids]) / t.count[n]
                c_thr = threshold(ub["transition_threshold"], t.count[n]) / t.count[n]
                p_plus = max_expectation_one_positive(u_next, p_hat, c_thr)
                p_minus = max_expectation_one_positive(-l_next, p_hat, c_thr)
                t.upper[n] = p_plus @ u_next
                t.lower[n] = p_minus @ l_next
            n = t.parent[n]
        _, best, challenger = bai(root)
        done = t.upper[challenger] - t.lower[best] < config["accuracy"]         # stopping rule (:100-102)
        done = done or episode > episodes
        episode += 1
    t.episodes, t.horizon, t.best, t.challenger = episodes, horizon, best, challenger
    _, best, _ = bai(root)                                                      # get_plan (:129-131, :172-176)
    return [t.action[best]], t, episode
