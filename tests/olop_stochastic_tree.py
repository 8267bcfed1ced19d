"""The compact form in which tests/golden/golden_olop_stochastic.json keeps an OLOP tree: SHA-256 digests of its node
arrays in creation order, one over the fields the device reproduces exactly and one over the KL bounds, which CUDA's
log moves by an ulp; plus the bounds' sums, for a tolerance check."""
import hashlib

import numpy as np

EXACT_FIELDS = (("parent", np.int64), ("action", np.int64), ("count", np.int64), ("done", np.uint8),
                ("cumulative_reward", np.float64))
FLOAT_FIELDS = ("mu_ucb", "upper")


def _sha256(tree, fields):
    h = hashlib.sha256()
    for f, dtype in fields:
        h.update(np.ascontiguousarray(np.asarray(tree[f]).astype(dtype)).tobytes())
    return h.hexdigest()


def tree_digest(tree):
    """tree: dict of equal-length node arrays (parent, action, count, done, cumulative_reward, mu_ucb, upper)."""
    out = {"n_nodes": len(tree["parent"]), "exact_sha256": _sha256(tree, EXACT_FIELDS),
           "float_sha256": _sha256(tree, [(f, np.float64) for f in FLOAT_FIELDS])}
    for f in FLOAT_FIELDS:
        out["sum_" + f] = float(np.sum(np.asarray(tree[f], dtype=np.float64)))
    return out
