"""Finite MDPs with infinite rewards, shared by the value-iteration tests on the device (tests/test_gpu_vi_paths.py) and
by the check of the numpy comparator against the reference agents (tests/test_vi_nonfinite_oracle.py).

An infinite reward is how a user forbids (-inf) or forces (+inf) an action.  Within a few sweeps it turns into NaN:
-inf + gamma * inf where a forbidden action leads to a forced state, 0 * inf where a zero probability (sparse, dense)
or gamma = 0 meets an infinite value.  numpy's max over actions and min over models propagate that NaN whatever the
action or model holding it."""
import numpy as np

from oracle import envs as oenvs

# Deterministic, 3 states x 2 actions.  At gamma = 0.9 the second action of state 0 is -inf + 0.9 * inf = NaN from the
# second sweep on, while its first action is finite: a max that skips a NaN after the first action keeps rows 0 and 1
# finite, numpy makes them NaN.
THREE_STATE = dict(transition=np.array([[1, 2], [0, 0], [2, 2]]),
                   reward=np.array([[0.5, -np.inf], [0.25, 0.0], [np.inf, np.inf]]),
                   terminal=np.zeros(3, bool))


def garnet_mdp(mode, S, A, B, seed, terminal_rate=0.05):
    """(transition, reward, terminal, nxt) of a seeded sparse or deterministic garnet."""
    terminal = np.random.default_rng(seed).uniform(size=S) < terminal_rate
    if mode == "sparse":
        P, N, R = oenvs.garnet(S, A, B, seed=seed)
        return P, R, terminal, N
    T, R = oenvs.garnet(S, A, 1, seed=seed, deterministic=True)
    return T, R, terminal, None


def forced_and_forbidden(mode, S, A, B, seed, nan):
    """A garnet_mdp that converges early at gamma = 0.5, in which no state leads to states 0-7.  States 1-7 force their
    first action at +inf: Q(s, 0) stays +inf there, sweep after sweep, and np.isclose(inf, inf) holds.  With nan, state 0
    loops on itself with a +inf and a -inf action: -inf + 0.5 * inf = NaN from the second sweep on, for good, and
    np.isclose(nan, nan) never holds."""
    T, R, term, N = garnet_mdp(mode, S, A, B, seed=seed, terminal_rate=0.02)
    succ = N if mode == "sparse" else T
    succ[succ < 8] += 8
    succ[0] = 0
    R[1:8, 0] = np.inf
    R[0] = 0.0
    if nan:
        R[0, 0], R[0, 1] = np.inf, -np.inf
    term[:8] = False
    return T, R, term, N


def nonfinite_mdp(mode, S, A, B, seed):
    """(transition, reward, terminal, nxt) of a seeded garnet (dense: uniform rows) with about 1 % +inf and 1.5 % -inf
    rewards at any action, 5 % terminal states (some of them with infinite rewards) and, in the sparse and dense modes,
    zero probabilities: about 10 % of the sparse successors (never the first), 30 % of a dense row.  States 0 and 1 are
    fixed: state 1 loops on itself at +inf, every action of state 0 leads to state 1 only (sparse: with equal
    probabilities; dense: a uniform row), and the last action of state 0 is -inf.  So from the second sweep on at
    gamma > 0, Q(0, 0) is +inf and Q(0, A - 1) is -inf + gamma * inf = NaN."""
    rng = np.random.default_rng(seed)
    nxt = None
    if mode == "deterministic":
        transition, reward = oenvs.garnet(S, A, 1, seed=seed, deterministic=True)
        transition[:2] = 1
    elif mode == "sparse":
        transition, nxt, reward = oenvs.garnet(S, A, B, seed=seed)
        zero = rng.uniform(size=transition.shape) < 0.1
        zero[..., 0] = False
        transition[zero] = 0.0
        transition[:2] = 1.0
        transition /= transition.sum(axis=-1, keepdims=True)
        nxt[:2] = 1
    elif mode == "stochastic":
        transition = rng.uniform(size=(S, A, S))
        transition[rng.uniform(size=transition.shape) < 0.3] = 0.0
        transition[..., 0] += transition.sum(axis=-1) == 0
        transition[0] = 1.0
        transition[1] = 0.0
        transition[1, :, 1] = 1.0
        transition /= transition.sum(axis=-1, keepdims=True)
        reward = rng.uniform(size=(S, A))
    else:
        raise ValueError(mode)
    u = rng.uniform(size=(S, A))
    reward[u < 0.01] = np.inf
    reward[(u >= 0.01) & (u < 0.025)] = -np.inf
    reward[0] = 0.5
    reward[0, -1] = -np.inf
    reward[1] = np.inf
    terminal = rng.uniform(size=S) < 0.05
    terminal[:2] = False
    return transition, reward, terminal, nxt


def nonfinite_models(mode, M, S, A, seed):
    """(transitions [M, S, A(, S)], rewards [M, S, A]) of M models from nonfinite_mdp (terminal states dropped: robust
    value iteration has none), with every action of state 0 at -inf: from the second sweep on Q(0, a) is NaN in all M
    models at once."""
    T, R = [], []
    for m in range(M):
        t, r, _, _ = nonfinite_mdp(mode, S, A, 1, seed + m)
        r[0] = -np.inf
        T.append(t)
        R.append(r)
    return np.array(T), np.array(R)


def nan_after_a_number(q):
    """True when a row of Q holds a NaN at some action after a first action that is not NaN: the max over actions
    that skipped such a NaN returned a number there."""
    nan = np.isnan(q)
    return bool((~nan[:, :1] & nan[:, 1:]).any())


def nan_in_some_models(qm):
    """(some, all) for model-wise values qm [M, S, A]: a NaN in some but not all models of an (s, a) pair, and in all."""
    nan = np.isnan(qm)
    return bool((nan.any(axis=0) & ~nan.all(axis=0)).any()), bool(nan.all(axis=0).any())
