"""The cases of tests/golden/golden_mcts_stochastic.json (MCTS on stochastic finite MDPs) and the compact form in which it
keeps a tree: one SHA-256 digest of the node arrays in creation order -- parents, actions, counts, and value and prior as
float64 bytes -- which the device reproduces exactly.  A re-rooted tree ("subtree") is digested in the breadth-first
form of tests/util.py::canonical_tree, since a re-rooted tree's node ids differ between the reference and the device.

The env generator of every case is seeded (`env_seed`) and, where `advance` > 0, moved forward by that many doubles
before the decision, so the search replays a stream that does not start at the seed."""
import hashlib

import numpy as np

from tests.mdp_gape_stochastic_cases import MDPS, oracle_env, product_env
from tests.util import canonical_tree

PREFERENCE = {"prior_policy": {"type": "preference", "action": 1, "ratio": 3},
              "rollout_policy": {"type": "preference", "action": 2, "ratio": 2}}
RANDOM = {"prior_policy": {"type": "random"}, "rollout_policy": {"type": "random"}}

# name -> (MDP, root state, agent config, planner seed, env seed, env doubles drawn before the decision)
CASES = {
    "dense6_b400_g0.8": ("dense6", 0, {"budget": 400, "gamma": 0.8}, 0, 100, 0),
    "garnet50_b300_g0.8_preference": ("garnet50", 3, dict(PREFERENCE, budget=300, gamma=0.8), 1, 101, 0),
    "dup20_b300_g0.85_random": ("dup20", 0, dict(RANDOM, budget=300, gamma=0.85), 2, 102, 0),
    "term40_b600_g0.9": ("term40", 1, {"budget": 600, "gamma": 0.9}, 3, 103, 0),
    "garnet50_b2000_g0.9": ("garnet50", 20, {"budget": 2000, "gamma": 0.9}, 4, 104, 0),
    "garnet30_b2_b400_g0.8_advanced_env": ("garnet30_b2", 4, {"budget": 400, "gamma": 0.8}, 5, 105, 7),
    "dense6_b300_g0.8_advanced_env_random": ("dense6", 2, dict(RANDOM, budget=300, gamma=0.8), 6, 106, 3),
    "unreached_bad20_b300_g0.8": ("unreached_bad20", 0, {"budget": 300, "gamma": 0.8}, 7, 107, 0),
}
CLOSED_LOOP = {
    "garnet50_b400_g0.8_closed_loop": ("garnet50", 0, {"budget": 400, "gamma": 0.8, "closed_loop": True}, 8, 108, 0),
    "dense6_b300_g0.8_closed_loop_preference": ("dense6", 1, dict(PREFERENCE, budget=300, gamma=0.8,
                                                                  closed_loop=True), 9, 109, 0),
}
SUBTREE = {
    "garnet50_b300_g0.85_subtree": ("garnet50", 0, {"budget": 300, "gamma": 0.85, "step_strategy": "subtree"},
                                    10, 110, 0),
    "term40_b300_g0.8_subtree": ("term40", 2, {"budget": 300, "gamma": 0.8, "step_strategy": "subtree"}, 11, 111, 0),
}
ERRORS = {
    "bad20_reached_nan_row": ("bad20", 0, {"budget": 300, "gamma": 0.8}, 12, 112, 0),
}


def planner_rng(seed):
    """The planner's generator after agent.seed(seed) (seeding.np_random)."""
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def live_env(case, product=False):
    """The case's env: MDP, root state, seeded generator moved forward by `advance` doubles."""
    mdp, state, _, _, env_seed, advance = case
    env = (product_env if product else oracle_env)(mdp, state)
    env.seed(env_seed)
    if advance:
        env.np_random.random(advance)
    return env


def policy(config, key):
    return config.get(key, {"type": "random_available"})


def _sha256(arrays):
    h = hashlib.sha256()
    for a, dtype in arrays:
        h.update(np.ascontiguousarray(np.asarray(a).astype(dtype)).tobytes())
    return h.hexdigest()


def tree_digest(tree):
    """tree: dict of equal-length node arrays in creation order (parent, action, count, value, prior)."""
    return {"n_nodes": len(tree["parent"]),
            "sha256": _sha256([(tree["parent"], np.int64), (tree["action"], np.int64), (tree["count"], np.int64),
                               (tree["value"], np.float64), (tree["prior"], np.float64)])}


def canonical_digest(first_child, n_children, action, count, value, prior):
    """The breadth-first form (tests/util.py::canonical_tree) of a tree, digested."""
    rows = canonical_tree(first_child, n_children, [action, count, value, prior])
    cols = list(zip(*rows))
    return {"n_nodes": len(rows),
            "sha256": _sha256([(cols[0], np.int64), (cols[1], np.int64), (cols[2], np.int64), (cols[3], np.float64),
                               (cols[4], np.float64)])}


def rng_words_state(words):
    """uint64 [6] PCG64 words -> the rng_state dict of the goldens."""
    w = [int(x) for x in words]
    return {"state": str((w[0] << 64) | w[1]), "inc": str((w[2] << 64) | w[3]), "has_uint32": w[4], "uinteger": w[5]}


def rng_state(gen):
    st = gen.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]), "has_uint32": int(st["has_uint32"]),
            "uinteger": int(st["uinteger"])}


assert all(MDPS[c[0]]["mode"] in ("stochastic", "sparse") for d in (CASES, CLOSED_LOOP, SUBTREE, ERRORS)
           for c in d.values())
