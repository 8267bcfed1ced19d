"""Flat CPU restatement of MDP-GapE on stochastic finite MDPs -- TEST INFRASTRUCTURE.

oracle/mdp_gape.py restates the deterministic case, where a chance node observes one next state and
max_expectation_under_constraint (rl_agents/utils.py:292-342) needs no Newton solve.  This module restates the
general case: a chance node observes up to max_next_states_count next states, and its backup runs
max_expectation_under_constraint in full, theta_func / d_theta_dl_func and newton_iteration included.  Pinned against
tests/golden/golden_mdp_gape_stochastic.json, which tests/golden/make_golden_mdp_gape_stochastic.py records from the
UNMODIFIED reference (tests/test_mdp_gape_stochastic_oracle.py).

Arithmetic, as the reference runs it on the host the goldens were recorded on:
- its 1-D float64 dot products (numpy's `@` and numba's `@`, lengths up to 15) are sequential fused multiply-add chains
  from 0.0; dot_fma() writes them so, rounded exactly once per step through fractions.Fraction, so that the oracle does
  not depend on the host's BLAS;
- theta_func and d_theta_dl_func are numba code, whose np.log is the C library's log: math.log here;
- np.exp, np.isclose and the elementwise divisions are numpy's.
With one positive entry of p_hat, max_expectation_under_constraint takes the same operations as
oracle.mdp_gape.max_expectation_one_positive.  Kept in its own module so that oracle/mdp_gape.py, and the arithmetic of
its goldens, stay as they were pinned; mdp_gape_plan runs that module's episode loop with the general backup.
"""
import math
from fractions import Fraction

import numpy as np

from oracle import mdp_gape as gape


def fma(a, b, c):
    """a * b + c rounded once (IEEE fused multiply-add); non-finite operands take the unfused IEEE result."""
    a, b, c = float(a), float(b), float(c)
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        return a * b + c
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def dot_fma(x, y):
    """x @ y for 1-D float64 vectors as the reference's host computes it: acc = fma(x[i], y[i], acc) from 0.0."""
    acc = 0.0
    for a, b in zip(x, y):
        acc = fma(a, b, acc)
    return acc


def theta_func(l, q_p, f_p, c):
    """utils.py:279-282 (numba): q_p @ log(l - f_p) + log(q_p @ (1 / (l - f_p))) - c."""
    l_m_f_p = l - f_p
    with np.errstate(all="ignore"):
        logs = [math.log(x) if x > 0 else (-math.inf if x == 0 else math.nan) for x in l_m_f_p]
        inv = 1 / l_m_f_p
    s2 = dot_fma(q_p, inv)
    return dot_fma(q_p, logs) + (math.log(s2) if s2 > 0 else (-math.inf if s2 == 0 else math.nan)) - c


def d_theta_dl_func(l, q_p, f_p):
    """utils.py:285-289 (numba): 1 / (l - f_p) = inv; q_p @ inv - (q_p @ inv**2) / (q_p @ inv).  A zero divisor
    raises ZeroDivisionError, as numba's scalar division does."""
    with np.errstate(all="ignore"):
        inv = 1 / (l - f_p)
    q_inv = dot_fma(q_p, inv)
    if q_inv == 0:
        raise ZeroDivisionError("division by zero")
    return q_inv - dot_fma(q_p, inv * inv) / q_inv


def newton_iteration(f, df, eps, x0, a, weight=0.9, max_iterations=100):
    """utils.py:150-203 with a lower bound `a` only (b is None), as max_expectation_under_constraint calls it."""
    x = np.inf
    x_next = x0
    iterations = 0
    while abs(x - x_next) > eps and iterations < max_iterations:
        iterations += 1
        x = x_next
        f_x = f(x)
        try:
            df_x = df(x)
        except ZeroDivisionError:
            df_x = (f_x - f(x - eps)) / eps
        if df_x != 0:
            x_next = x - f_x / df_x
        if x_next < a:
            x_next = weight * a + (1 - weight) * x
    if x_next < a:
        x_next = a
    return x_next


def max_expectation_under_constraint(f, q, c, eps=1e-2):
    """utils.py:292-342: argmax_p E_p[f] s.t. KL(q || p) <= c, the reference's operations in its order."""
    f = np.asarray(f, dtype=np.float64)
    q = np.asarray(q, dtype=np.float64)
    if np.all(q == 0):
        q = np.ones(q.size) / q.size
    x_plus = np.where(q > 0)
    x_zero = np.where(q == 0)
    p_star = np.zeros(q.shape)
    lambda_, z = None, 0
    q_p = q[x_plus]
    f_p = f[x_plus]
    f_star = np.amax(f)
    if f_star > np.amax(f_p):
        theta_star = theta_func(f_star, q_p, f_p, c)
        if theta_star < 0:
            lambda_ = f_star
            z = 1 - np.exp(theta_star)
            p_star[x_zero] = 1.0 * (f[x_zero] == np.amax(f[x_zero]))
            p_star[x_zero] *= z / p_star[x_zero].sum()
    if lambda_ is None:
        if np.isclose(f_p, f_p[0]).all():
            return q
        lambda_ = newton_iteration(lambda x: theta_func(x, q_p, f_p, c), lambda x: d_theta_dl_func(x, q_p, f_p), eps,
                                   x0=f_star + 1, a=f_star)
    with np.errstate(divide="ignore"):
        beta = (1 - z) / dot_fma(q_p, 1 / (lambda_ - f_p))
    if beta == 0:
        x_uni = np.where((q > 0) & (f == f_star))
        if np.size(x_uni) > 0:
            p_star[x_uni] = (1 - z) / np.size(x_uni)
    else:
        p_star[x_plus] = beta * q_p / (lambda_ - f_p)
    return p_star


class _FmaVector(np.ndarray):
    """A p_plus / p_minus whose `p @ next` is the host's fma chain (dot_fma), as in ChanceNode.backup_to_root."""

    def __matmul__(self, other):
        return dot_fma(np.asarray(self), other)


def _general_expectation(f, q, c):
    return np.asarray(max_expectation_under_constraint(f, q, c)).view(_FmaVector)


class _Capped(Exception):
    pass


def mdp_gape_plan(env, config, np_random, last_episode=None):
    """MDPGapE.plan (mdp_gape.py:94-110) from a fresh root, on any env whose legacy 4-tuple `step` may be stochastic
    (oracle.envs.LegacyStepEnv(FiniteMDPLite(mode="stochastic" | "sparse"))).  Each episode seeds the env copy with
    np_random.randint(2**30) (:67); the env draws its next states itself.

    This is oracle.mdp_gape.mdp_gape_plan -- its episode loop, UGapE selection, chance-node keying by str(observation)
    and statistics updates -- run with the chance-node backup of the general case: max_expectation_under_constraint
    above in place of the one-positive restatement, and `p @ next` as an fma chain.  Returns (plan, tree,
    episodes_run) as that function does, plus `t.key[node]`: the int(observation) a decision node was observed under,
    -1 on unobserved placeholders, the root and chance nodes.

    last_episode: stop after the episode of that index, before the next one draws its seed (episodes and thresholds
    stay the config's); the plan is then None, and the tree has no best / challenger."""
    trees = []

    class Tree(gape.Tree):
        def __init__(self):
            super(Tree, self).__init__()
            trees.append(self)

    rng = np_random
    if last_episode is not None:
        class Capped(object):
            seeds = 0

            def __getattr__(self, name):
                return getattr(np_random, name)

            def randint(self, n, *args, **kwargs):
                if n == 2 ** 30:
                    Capped.seeds += 1
                    if Capped.seeds > last_episode + 1:
                        raise _Capped()
                return np_random.randint(n, *args, **kwargs)
        rng = Capped()
    saved = gape.max_expectation_one_positive, gape.Tree
    gape.max_expectation_one_positive, gape.Tree = _general_expectation, Tree
    try:
        plan, t, episodes_run = gape.mdp_gape_plan(env, config, rng)
    except _Capped:
        plan, t, episodes_run = None, trees[0], last_episode + 1
    finally:
        gape.max_expectation_one_positive, gape.Tree = saved
    t.key = [-1] * len(t.parent)
    for chance, keys in t.keys.items():
        for key, node in zip(keys, t.order[chance]):
            if not key.startswith("placeholder_"):
                t.key[node] = int(key)
    return plan, t, episodes_run
