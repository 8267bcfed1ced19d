"""The one place the planners touch an env's object model (SURVEY 8b, "env
hand-off"): turn the (pre-processed) env object `agent.plan` receives into the
arrays the kernels read."""
import numpy as np

from rl_agents_b200 import _lib


class EnvDescription(object):
    __slots__ = ("kind", "n_actions", "mdp", "root", "env_words")


def describe(env, env_words=False):
    """-> EnvDescription(kind, action_space.n, finite MDP tables or None, root state int32 array, env_words).
    env_words: with env_words set (the planners that step deep copies of the env without reseeding them: MCTS), for a
    finite MDP in mode "stochastic" or "sparse", the uint64 [6] words (pcg64_words) of the env's own generator, which
    such a copy steps with -- ValueError when that generator is not a numpy Generator(PCG64); None otherwise."""
    u = getattr(env, "unwrapped", env)
    d = EnvDescription()
    d.n_actions = int(env.action_space.n)
    d.env_words = None
    kind = getattr(u, "b2_env_kind", None)
    if kind == "intersection":
        d.kind, d.mdp = _lib.ENV_INTERSECTION, None
        d.root = np.ascontiguousarray(u.words, dtype=np.int32)
        return d
    if kind == "highway" or (kind is None and hasattr(u, "words")):
        d.kind, d.mdp = _lib.ENV_HIGHWAY, None
        d.root = np.ascontiguousarray(u.words, dtype=np.int32)
        return d
    from rl_agents_b200.envs.highway_adapter import looks_like_highway_env, scene_from_highway_env
    if kind is None and looks_like_highway_env(u):
        # a live `highway_env` highway-v0 object: pack its scene; the search runs on the HighwayLite model of it
        d.kind, d.mdp = _lib.ENV_HIGHWAY, None
        d.root = scene_from_highway_env(u)
        return d
    mdp = getattr(u, "mdp", None)
    if mdp is not None and hasattr(mdp, "transition") and hasattr(mdp, "reward"):
        # rl_agents_b200.envs.FiniteMDPEnv or the `finite_mdp` package's FiniteMDPEnv
        d.kind, d.mdp = _lib.ENV_FINITE, mdp
        d.root = np.array([int(mdp.state)], dtype=np.int32)
        if env_words and getattr(mdp, "mode", "deterministic") != "deterministic":
            from rl_agents_b200.engine.mcts import pcg64_words
            gen = getattr(u, "np_random", None)
            if not isinstance(gen, np.random.Generator) or not isinstance(gen.bit_generator, np.random.PCG64):
                raise ValueError("a stochastic finite-MDP env must step with a numpy Generator(PCG64) "
                                 "(got %r)" % (type(getattr(gen, "bit_generator", gen)).__name__,))
            d.env_words = pcg64_words(gen)
        return d
    raise TypeError("rl_agents_b200 planners need a HighwayLiteEnv, a highway_env highway-v0 env or a finite-MDP env "
                    "(got %r); see INTEGRATION.md for the env hand-off" % type(u).__name__)


def mdp_fingerprint(mdp):
    """Cache key of the device copy of a finite MDP's tables: shapes, buffer addresses and a strided
    checksum -- so that a copying preprocessor (a new but identical mdp object per decision) reuses the
    device tables, and an mdp mutated in place or a different one recycled at the same id() does not."""
    if mdp is None:
        return None
    parts = [getattr(mdp, "mode", None)]
    for name in ("transition", "reward", "terminal", "next"):
        arr = getattr(mdp, name, None)
        if arr is None:
            parts.append(None)
            continue
        arr = np.asarray(arr)
        flat = arr.reshape(-1)
        stride = max(1, flat.size // 4096)
        parts.append((arr.shape, str(arr.dtype), float(np.asarray(flat[::stride], dtype=np.float64).sum()),
                      float(np.asarray(flat[-1:], dtype=np.float64).sum())))
    return tuple(parts)
