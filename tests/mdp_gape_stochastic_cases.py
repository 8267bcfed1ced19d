"""The finite MDPs of the stochastic MDP-GapE goldens (tests/golden/make_golden_mdp_gape_stochastic.py), rebuilt from
seeds so that the generator, the oracle tests and the GPU tests plan on the same tables."""
import numpy as np

from oracle import envs


def _garnet(S, A, B, seed):
    p, nxt, r = envs.garnet(S, A, B, seed=seed)
    return {"mode": "sparse", "transition": p, "next": nxt, "reward": r, "terminal": np.zeros(S, bool)}


def case_mdps():
    """name -> {mode, transition, next, reward, terminal}."""
    out = {"garnet50": _garnet(50, 4, 3, 0), "garnet30_b2": _garnet(30, 3, 2, 1)}
    # a small dense "stochastic" MDP: every row reaches all 6 states, some with probability 0
    rng = np.random.default_rng(7)
    p = rng.uniform(0.0, 1.0, size=(6, 3, 6)) * (rng.uniform(size=(6, 3, 6)) > 0.25)
    p[:, :, 0] += 0.05
    p /= p.sum(axis=-1, keepdims=True)
    out["dense6"] = {"mode": "stochastic", "transition": p, "next": None,
                     "reward": rng.uniform(0.0, 1.0, size=(6, 3)), "terminal": np.zeros(6, bool)}
    # successor ids repeated within a row: one child per distinct id
    dup = _garnet(20, 3, 4, 2)
    dup["next"][:, :, 1] = dup["next"][:, :, 0]
    dup["next"][::2, :, 3] = dup["next"][::2, :, 2]
    out["dup20"] = dup
    # terminal states
    term = _garnet(40, 3, 3, 3)
    term["terminal"][::5] = True
    out["term40"] = term
    # a NaN row at the root (reached) and one at a state no row leads to (never reached)
    bad = _garnet(20, 3, 3, 4)
    bad["next"][bad["next"] == 19] = 18
    bad["transition"][0, 1] = np.nan
    bad["transition"][19, 0] = np.nan
    out["bad20"] = bad
    unreached = _garnet(20, 3, 3, 4)
    unreached["next"][unreached["next"] == 19] = 18
    unreached["transition"][19, 0] = np.nan
    out["unreached_bad20"] = unreached
    # rewards outside [0, 1]
    wide = _garnet(20, 3, 3, 5)
    wide["reward"] = 2 * wide["reward"] - 0.5
    out["wide20"] = wide
    return out


MDPS = case_mdps()


def oracle_env(name, state=0):
    m = MDPS[name]
    return envs.FiniteMDPLite(m["transition"], m["reward"], m["terminal"], mode=m["mode"], nxt=m["next"], state=state)


def product_env(name, state=0):
    from rl_agents_b200.envs import FiniteMDPEnv
    m = MDPS[name]
    return FiniteMDPEnv(m["transition"], m["reward"], m["terminal"], mode=m["mode"], nxt=m["next"], state=state)
