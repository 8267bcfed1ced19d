"""Host-computed tables the kernels read so that their floating point matches
the reference's Python float arithmetic bit for bit."""
import numpy as np


def gamma_tables(gamma, n):
    """gamma**d and gamma**d/(1-gamma) with Python float `**` (deterministic.py:52-53)."""
    gamma = float(gamma)
    gp = np.array([gamma ** d for d in range(n)], dtype=np.float64)
    with np.errstate(divide="ignore"):
        gd = np.array([(gamma ** d) / (1 - gamma) if gamma != 1 else np.inf for d in range(n)], dtype=np.float64)
    return gp, gd


def terminal_bonus_table(terminal_reward, gamma, n):
    """(terminal_reward * gamma**d) / (1 - gamma), the reference's association (deterministic.py:60-63)."""
    gamma, tr = float(gamma), float(terminal_reward)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.array([(tr * gamma ** d) / (1 - gamma) if gamma != 1 else np.inf * tr for d in range(n)],
                        dtype=np.float64)


def uniform_cdf_table(n_actions):
    """Row n: cumsum(ones(n)/n)/cumsum[-1] -- the cdf Generator.choice(a, 1, p=p)
    searches for a uniform p over n actions (mcts.py:60-72,172)."""
    t = np.ones((n_actions + 1, n_actions), dtype=np.float64)
    for n in range(1, n_actions + 1):
        cdf = (np.ones(n) / n).cumsum()
        cdf /= cdf[-1]
        t[n, :n] = cdf
    return t


def preference_tables(n_actions, ratio):
    """MCTSAgent.preference_policy (mcts.py:76-97) for every (number of available actions n, position k-1 of
    the preferred action among them; k = 0: not available -> uniform): the probabilities exactly as numpy
    computes them there, and the cdf Generator.choice(actions, 1, p=p) searches.  Shape [(A+1), (A+1), A]."""
    A = int(n_actions)
    prior = np.ones((A + 1, A + 1, A), dtype=np.float64)
    cdf = np.ones((A + 1, A + 1, A), dtype=np.float64)
    for n in range(1, A + 1):
        for k in range(0, n + 1):
            if k == 0:
                p = np.ones(n) / n
            else:
                p = np.ones(n) / (n - 1 + ratio)
                p[k - 1] *= ratio
            c = p.cumsum()
            c /= c[-1]
            prior[n, k, :n] = p
            cdf[n, k, :n] = c
    return prior, cdf


def choice_rows_ok(p):
    """Per row of p [..., B]: whether Generator.choice(B, p=row) accepts it -- its Kahan sum is not NaN, no entry is
    negative, and the sum is within sqrt(eps) of 1."""
    p = np.asarray(p, dtype=np.float64)
    total, comp = p[..., 0].copy(), np.zeros(p.shape[:-1])
    with np.errstate(invalid="ignore", over="ignore"):
        for i in range(1, p.shape[-1]):          # numpy's kahan_sum, row by row
            y = p[..., i] - comp
            t = total + y
            comp = (t - total) - y
            total = t
        bad = np.isnan(total) | (p < 0).any(axis=-1) | (np.abs(total - 1.0) > np.sqrt(np.finfo(np.float64).eps))
    return ~bad


def sampled_mdp_tables(mdp):
    """A finite MDP as its env steps it (FiniteMDPEnv.step): r = reward[s, a]; k = Generator.choice(B, p=p[s, a]) of
    the env's freshly seeded generator, i.e. searchsorted(cdf, random(), "right") with the cdf numpy builds
    (p.cumsum(); cdf /= cdf[-1]); s' = next[s, a, k].  "deterministic": B = 1, next = transition; "stochastic":
    B = S, next[s, a, k] = k; "sparse": the given next.  -> dict(cdf, next, reward, row_ok)."""
    reward = np.ascontiguousarray(mdp.reward, dtype=np.float64)
    S, A = reward.shape
    if mdp.mode == "deterministic":
        nxt = np.asarray(mdp.transition).reshape(S, A, 1)
        cdf = np.ones((S, A, 1))
        ok = np.ones((S, A), dtype=bool)
    elif mdp.mode in ("stochastic", "sparse"):
        p = np.asarray(mdp.transition, dtype=np.float64)
        if mdp.mode == "stochastic":
            nxt = np.broadcast_to(np.arange(p.shape[-1]), p.shape)
        else:
            nxt = np.asarray(mdp.next)
        with np.errstate(invalid="ignore", divide="ignore"):
            cdf = p.cumsum(axis=-1)
            cdf /= cdf[..., -1:]
        ok = choice_rows_ok(p)
    else:
        raise ValueError("Unknown mode %r" % (mdp.mode,))
    if nxt.shape != cdf.shape or (nxt.size and (nxt.min() < 0 or nxt.max() >= S)):
        raise ValueError("next states must be an [S, A, B] table of state ids")
    return {"cdf": np.ascontiguousarray(cdf), "next": np.ascontiguousarray(nxt, dtype=np.int32), "reward": reward,
            "row_ok": np.ascontiguousarray(ok, dtype=np.uint8)}


class SampledFiniteTables(object):
    """Device copy of a finite MDP in any mode, stepped as FiniteMDPEnv.step by the planners that sample transitions
    (OLOP, MDP-GapE, MCTS-DPW, PlaTyPOOS, sparse sampling): the b2_finite_mdp_sampled tables, terminal (uint8 [S],
    done = terminal[state before the step]) and env_draws (1 when a step draws from the env's generator)."""

    def __init__(self, mdp, device):
        import torch
        self.mode = mdp.mode
        t = sampled_mdp_tables(mdp)
        self.p = None if mdp.mode == "deterministic" else np.asarray(mdp.transition, dtype=np.float64)
        self.n_states, self.n_actions, self.n_next = t["cdf"].shape
        for k, v in t.items():
            setattr(self, k, torch.as_tensor(v, device=device))
        self.terminal = torch.as_tensor(np.ascontiguousarray(mdp.terminal, dtype=np.uint8), device=device)
        self.env_draws = int(mdp.mode != "deterministic")

    def raise_rejected_row(self, row):
        """Raise what Generator.choice raises on the probability row s * A + a that a kernel flagged (numpy's own
        ValueError, as the reference's env step does), or AssertionError if numpy accepts it."""
        p = self.p.reshape(-1, self.p.shape[-1])[row]
        np.random.default_rng(0).choice(p.size, p=p)
        raise AssertionError("row %d was flagged but Generator.choice accepts it" % row)

    def struct(self):
        from rl_agents_b200 import _lib
        return _lib.FiniteMDPSampled(self.n_states, self.n_actions, self.n_next, 0, self.cdf.data_ptr(),
                                     self.next.data_ptr(), self.reward.data_ptr(), self.row_ok.data_ptr())


def finite_model(env_kind, mdp, device):
    """-> (sampled, tables, the b2_finite_mdp a planner config carries) of an engine on env_kind: a finite MDP in
    mode "deterministic" gets FiniteTables, whose struct the config carries; in any other mode SampledFiniteTables,
    passed to the *_sampled entry point, and the config carries an empty struct, as on the other env kinds, which get no
    tables."""
    from rl_agents_b200 import _lib
    if env_kind != _lib.ENV_FINITE:
        return False, None, _lib.FiniteMDP()
    if mdp.mode == "deterministic":
        tables = FiniteTables(mdp, device)
        return False, tables, tables.struct()
    return True, SampledFiniteTables(mdp, device), _lib.FiniteMDP()


class FiniteTables(object):
    """Device copy of a deterministic finite MDP (int32 transitions)."""

    def __init__(self, mdp, device):
        import torch
        if mdp.mode != "deterministic":
            raise ValueError("tree search on a finite MDP needs mode == 'deterministic' (got %r)" % mdp.mode)
        self.n_states, self.n_actions = mdp.reward.shape
        self.transition = torch.as_tensor(np.ascontiguousarray(mdp.transition, dtype=np.int32), device=device)
        self.reward = torch.as_tensor(np.ascontiguousarray(mdp.reward, dtype=np.float64), device=device)
        self.terminal = torch.as_tensor(np.ascontiguousarray(mdp.terminal, dtype=np.uint8), device=device)

    def struct(self):
        from rl_agents_b200 import _lib
        return _lib.FiniteMDP(self.n_states, self.n_actions, self.transition.data_ptr(),
                              self.reward.data_ptr(), self.terminal.data_ptr())
