"""Batched sparse-sampling engine (device side of SparseSamplingAgent)."""
import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import SampledFiniteTables
from rl_agents_b200.engine.tree_engine import TreeEngine

# what the reference raises at horizon 0: the root has no children, and selection_rule's np.amax of its empty value
# list fails (sparse_sampling.py:45-46, :53-56; abstract.py:301)
EMPTY_ROOT_MESSAGE = "zero-size array to reduction operation maximum which has no identity"


def check_horizon_and_c(horizon, C):
    """The reference fails on these with errors that say little; refuse them up front."""
    if horizon == 0:
        raise ValueError(EMPTY_ROOT_MESSAGE)
    if horizon < 0:
        raise ValueError("sparse sampling needs horizon >= 1 (got %d): with a negative horizon the reference "
                         "recurses until Python raises RecursionError" % horizon)
    if C < 1:
        raise ValueError("sparse sampling needs C >= 1 (got %d): with C = 0 the reference takes no sample and "
                         "raises UnboundLocalError on the unbound `reward`" % C)


def worst_case_nodes(n_actions, horizon, C):
    """Nodes of a tree in which every sample reaches a new state: (A C)^d decision nodes and A (A C)^d chance nodes
    at depth d."""
    b = n_actions * C
    return sum(b ** d for d in range(horizon + 1)) + n_actions * sum(b ** d for d in range(horizon))


def deterministic_nodes(n_actions, horizon):
    """Nodes of a tree on a deterministic model in which every decision node has all n_actions actions: A^d decision
    and A^d chance nodes at depth d >= 1, and the root."""
    return 1 + 2 * sum(n_actions ** d for d in range(1, horizon + 1))


class SparseSamplingEngine(TreeEngine):
    """One tree per lane (finite MDPs) or per 16-lane group (HighwayLite), n_trees independent decisions per launch,
    each a depth-first search (b2_sparse_sampling_plan)."""
    WORKSPACE_BYTES = "b2_sparse_sampling_workspace_bytes"
    PLAN = "b2_sparse_sampling_plan"

    def __init__(self, env_kind, n_trees, n_actions, horizon, C, gamma, mdp=None, record_tree=False, capacity=None,
                 device="cuda"):
        """record_tree: also dump every tree in creation order (capacity: nodes per tree, by default the worst
        case).  The plan itself needs no node storage."""
        super(SparseSamplingEngine, self).__init__(n_trees, _lib.SPARSE_SAMPLING_RESULT_WORDS, device)
        torch = self.torch
        if env_kind not in (_lib.ENV_FINITE, _lib.ENV_HIGHWAY):
            raise NotImplementedError("sparse sampling runs on finite MDPs and HighwayLite")
        self.env_kind = env_kind
        self.n_actions = int(n_actions)
        self.horizon, self.C, self.gamma = int(horizon), int(C), float(gamma)
        check_horizon_and_c(self.horizon, self.C)
        self.tables = SampledFiniteTables(mdp, self.device) if env_kind == _lib.ENV_FINITE else None
        self.cfg = _lib.SparseSamplingConfig(env_kind, self.n_trees, self.n_actions, self.horizon, self.C, 0,
                                             self.gamma, self.tables.struct() if self.tables else _lib.FiniteMDPSampled())
        self._check_config()
        self.workspace = torch.empty(int(getattr(self.lib, self.WORKSPACE_BYTES)(self.cfg)), dtype=torch.uint8,
                                     device=self.device)
        self.tree = None
        if record_tree:
            self.capacity = int(capacity) if capacity is not None else self.worst_case_nodes()
            if self.capacity >= 2 ** 31:
                raise ValueError("a recorded tree of up to %d nodes does not fit int32 node ids" % self.capacity)
            self.tree = _lib.SparseSamplingTree(self.capacity, 0,
                                                *self._alloc_tree(_lib.SPARSE_SAMPLING_TREE_FIELDS, self.capacity))
        self.root_q = torch.empty((self.n_trees, self.n_actions), dtype=torch.float64, device=self.device)
        self.plan_buf = torch.empty(self.n_trees, dtype=torch.int8, device=self.device)

    def _check_config(self):
        """Refuse what this engine's kernel cannot plan (the lane kernel plans every model)."""

    def worst_case_nodes(self):
        """The default dump capacity."""
        return worst_case_nodes(self.n_actions, self.horizon, self.C)

    def plan(self, root_states, rng_words):
        """root_states: [n_trees] state ids (finite) or [n_trees, 136] words (HighwayLite), on the device."""
        self._load_rng(rng_words)
        _lib.check(getattr(self.lib, self.PLAN)(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.workspace),
                                                _lib.ptr(self.rng), _lib.ptr(self.root_q), _lib.ptr(self.plan_buf),
                                                _lib.ptr(self.result), _lib.current_stream()))

    def _check(self, res):
        """A sampled probability row that Generator.choice rejects raises its ValueError, as the reference's env step
        does."""
        bad = np.nonzero(res[:, 4] == 2)[0]
        if bad.size:
            self.tables.raise_rejected_row(int(res[bad[0], 5]))
        if (res[:, 4] != 0).any():
            raise RuntimeError("sparse-sampling tree dump exhausted its capacity of %d nodes" % self.capacity)

    def tree_dict(self, tree=0):
        """The dump of one tree in creation order: parent, kind (0 decision, 1 chance), key, depth, count, value."""
        if self.tree is None:
            raise ValueError("the engine was built without record_tree")
        n = int(self.result[tree, 0].item())
        return {k: getattr(self, k)[tree, :n].cpu().numpy() for k in _lib.SPARSE_SAMPLING_TREE_FIELDS}


def level_workspace_bytes(env_kind, n_actions, horizon, C):
    """Bytes of workspace SparseSamplingLevelEngine allocates for one decision (None: the worst-case tree does not
    fit int32 node ids)."""
    cfg = _lib.SparseSamplingConfig(env_kind, 1, int(n_actions), int(horizon), int(C), 0, 0.0, _lib.FiniteMDPSampled())
    n = int(_lib.load().b2_sparse_sampling_levels_workspace_bytes(cfg))
    return n if n > 0 else None


class SparseSamplingLevelEngine(SparseSamplingEngine):
    """ONE decision on a deterministic model (HighwayLite, or a finite MDP in mode "deterministic") searched by the
    whole GPU level by level (b2_sparse_sampling_plan_levels): the same outputs as SparseSamplingEngine bit for bit.
    Its workspace is sized for the tree in which every decision node has all actions (level_workspace_bytes)."""
    WORKSPACE_BYTES = "b2_sparse_sampling_levels_workspace_bytes"
    PLAN = "b2_sparse_sampling_plan_levels"

    def _check_config(self):
        if self.n_trees != 1:
            raise ValueError("the level-synchronous engine plans one decision (n_trees = 1, got %d)" % self.n_trees)
        if self.tables is not None and self.tables.n_next != 1:
            raise ValueError("the level-synchronous engine needs a deterministic model (finite MDP mode %r)"
                             % self.tables.mode)
        if level_workspace_bytes(self.env_kind, self.n_actions, self.horizon, self.C) is None:
            raise ValueError("a sparse-sampling tree of horizon %d over %d actions does not fit int32 node ids"
                             % (self.horizon, self.n_actions))

    def worst_case_nodes(self):
        return deterministic_nodes(self.n_actions, self.horizon)
