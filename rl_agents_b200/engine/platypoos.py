"""Batched PlaTyPOOS engine (device side of PlaTyPOOSAgent).

The host builds, once per engine and shared by every tree, every table the kernel would otherwise evaluate with log2,
ceil, floor or pow, each with the reference's own numpy expression (platypoos.py:22-25, :41-46, :75-76): h_max, p_top(h),
nodes_count / evaluations / min_visits per (h, p), gamma**d and the cross-validation evaluations per depth.  It also
bounds the arena: the widest layer and the node count of the widest tree the quotas allow."""
import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import SampledFiniteTables, gamma_tables
from rl_agents_b200.engine.tree_engine import TreeEngine

MAX_P = 32                          # p_top(h) < MAX_P: 2**31 evaluations per node would not fit the result words
INT32_MAX = 2 ** 31 - 1
# what the reference raises when get_plan finds no candidate: h_max < 2 runs no explore(), and a root without children
# (a finite MDP with one action: range(1, 1)) has nothing to select (platypoos.py:83)
EMPTY_CANDIDATES_MESSAGE = "max() iterable argument is empty"


def horizon_of(budget, n_actions):
    """h_max when the config has no "horizon" (platypoos.py:22-25).  A negative budget raises the reference's error
    (int() of NaN)."""
    expansion_budget = budget / n_actions
    return int(np.floor(expansion_budget / (2 * (np.log2(expansion_budget) + 1) ** 2)))


def p_top(h, h_max, gamma):
    return max(int(np.floor(np.log2(h_max / np.ceil(h ** 2 * gamma ** (2 * h))))), 0)


def layer_quotas(h, p, h_max, gamma):
    """(nodes_count, evaluations, min_visits) of explore(h) at p (platypoos.py:44-46)."""
    nodes_count = int(np.floor(h_max / h * np.ceil(h * 2 ** p * gamma ** (2 * h))))
    evaluations = int(np.ceil(h * 2 ** p * gamma ** (2 * h)))
    min_visits = int(np.ceil((h - 1) * 2 ** p * gamma ** (2 * (h - 1))))
    return nodes_count, evaluations, min_visits


def cross_validation_count(depth, h_max, gamma):
    return int(np.floor((depth + 1) * 5 * h_max * gamma ** (2 * depth) * (1 - gamma ** 2) ** 2))


def check_plannable(h_max, n_actions, finite):
    """Refuse up front what leaves get_plan without a candidate; the reference raises ValueError there."""
    if h_max < 2:
        raise ValueError("%s: PlaTyPOOS needs horizon >= 2 (got %d) -- explore() never runs, so there is no "
                         "candidate to plan to (raise the budget or set \"horizon\")" % (EMPTY_CANDIDATES_MESSAGE, h_max))
    if finite and n_actions < 2:
        raise ValueError("%s: a finite MDP with %d action(s) gives the root no child -- PlaTyPOOS expands actions "
                         "1..n-1 of an env without get_available_actions" % (EMPTY_CANDIDATES_MESSAGE, n_actions))


def quota_tables(h_max, gamma):
    """-> dict(p_top [H], nodes_count / evaluations / min_visits [H, MAX_P] (entry h, p), cv_count [H],
    gamma_pow [H]).  Row 0 of the explore tables is unused; quotas past int32 are clipped (no layer reaches them)."""
    H = int(h_max)
    out = {"p_top": np.zeros(H, np.int32), "cv_count": np.zeros(H, np.int32)}
    for k in ("nodes_count", "evaluations", "min_visits"):
        out[k] = np.zeros((H, MAX_P), np.int32)
    for h in range(1, H):
        pt = p_top(h, H, gamma)
        if pt >= MAX_P:
            raise ValueError("PlaTyPOOS's p_top(%d) = %d is past the supported %d" % (h, pt, MAX_P - 1))
        out["p_top"][h] = pt
        for p in range(pt + 1):
            for k, v in zip(("nodes_count", "evaluations", "min_visits"), layer_quotas(h, p, H, gamma)):
                out[k][h, p] = min(v, INT32_MAX)
    for d in range(H):
        out["cv_count"][d] = max(min(cross_validation_count(d, H, gamma), INT32_MAX), -INT32_MAX)
    out["gamma_pow"] = gamma_tables(gamma, H)[0]
    return out


def worst_case_layers(h_max, branching, tables):
    """Per depth, the most nodes a layer can hold when every expanded node has `branching` children: the root's
    children, then per explore(h) the selection bound (the list reaches nodes_count at p, or grows by the one node a
    met quota may still add) times the branching.  -> list of widths, depth 0 .. h_max."""
    W = [1, branching]
    for h in range(1, h_max):
        n = 0
        for p in range(int(tables["p_top"][h]), -1, -1):
            nc = int(tables["nodes_count"][h, p])
            n = min(W[h], n + 1 if n >= nc else nc)
        W.append(n * branching)
    return W


class PlaTyPOOSEngine(TreeEngine):
    """n_trees independent PlaTyPOOS decisions per launch, one tree per CTA, each on its own numpy PCG64 stream.  Plans
    hold several actions (result word 2), so `_plans` returns each tree's whole plan."""

    def __init__(self, env_kind, n_trees, n_actions, horizon, gamma, mdp=None, node_capacity=None,
                 layer_capacity=None, device="cuda"):
        """node_capacity / layer_capacity: per tree, by default the worst case the quotas allow
        (worst_case_layers); a tree that outgrows a smaller one sets error 1 (B2Error)."""
        if env_kind not in (_lib.ENV_FINITE, _lib.ENV_HIGHWAY):
            raise NotImplementedError("PlaTyPOOS runs on finite MDPs and HighwayLite")
        self.env_kind = env_kind
        self.n_actions, self.horizon, self.gamma = int(n_actions), int(horizon), gamma
        check_plannable(self.horizon, self.n_actions, env_kind == _lib.ENV_FINITE)
        t = quota_tables(self.horizon, gamma)
        branching = self.n_actions - 1 if env_kind == _lib.ENV_FINITE else _lib.HW_ACTIONS
        widths = worst_case_layers(self.horizon, branching, t)
        self.node_capacity = int(node_capacity) if node_capacity is not None else sum(widths)
        self.layer_capacity = int(layer_capacity) if layer_capacity is not None else max(widths)
        if not (1 <= self.node_capacity <= INT32_MAX and 1 <= self.layer_capacity <= INT32_MAX):
            raise ValueError("a PlaTyPOOS arena of %d nodes (layers of %d) does not fit int32 node ids"
                             % (self.node_capacity, self.layer_capacity))
        super(PlaTyPOOSEngine, self).__init__(n_trees, _lib.PLATYPOOS_RESULT_WORDS, device)
        torch = self.torch
        self.tables_host = t
        for k in ("p_top", "nodes_count", "evaluations", "min_visits", "cv_count", "gamma_pow"):
            setattr(self, k, torch.as_tensor(np.ascontiguousarray(t[k]), device=self.device))
        self.tables, self.terminal, env_draws, mdp_struct = None, None, 0, _lib.FiniteMDPSampled()
        if env_kind == _lib.ENV_FINITE:
            self.tables = SampledFiniteTables(mdp, self.device)
            self.terminal = self.tables.terminal
            env_draws, mdp_struct = self.tables.env_draws, self.tables.struct()
        self.cfg = _lib.PlaTyPOOSConfig(
            env_kind, self.n_trees, self.n_actions, self.horizon, self.node_capacity, self.layer_capacity, MAX_P,
            env_draws, self.p_top.data_ptr(), self.nodes_count.data_ptr(), self.evaluations.data_ptr(),
            self.min_visits.data_ptr(), self.cv_count.data_ptr(), self.gamma_pow.data_ptr(),
            self.terminal.data_ptr() if self.terminal is not None else None, mdp_struct)
        self.tree = _lib.PlaTyPOOSTree(*self._alloc_tree(_lib.PLATYPOOS_TREE_FIELDS, self.node_capacity))
        self.workspace = torch.empty(int(self.lib.b2_platypoos_workspace_bytes(self.cfg)), dtype=torch.uint8,
                                     device=self.device)
        self.plan_buf = torch.empty((self.n_trees, self.horizon), dtype=torch.int8, device=self.device)
        self.candidates = torch.empty((self.n_trees, 2 * MAX_P), dtype=torch.int32, device=self.device)

    def plan(self, root_states, rng_words):
        """root_states: [n_trees] state ids (finite) or [n_trees, 136] words (HighwayLite), on the device."""
        self._load_rng(rng_words)
        _lib.check(self.lib.b2_platypoos_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.workspace),
                                              _lib.ptr(self.rng), _lib.ptr(self.plan_buf), _lib.ptr(self.candidates),
                                              _lib.ptr(self.result), _lib.current_stream()))

    def _check(self, res):
        """A sampled probability row that Generator.choice rejects raises its ValueError, as the reference's env step
        does; the other error words raise what the reference raises or a B2Error."""
        err = res[:, 3]
        bad = np.nonzero(err == 2)[0]
        if bad.size:
            self.tables.raise_rejected_row(int(res[bad[0], 4]))
        if (err == 4).any():
            raise ValueError(EMPTY_CANDIDATES_MESSAGE)
        if (err == 3).any():
            raise _lib.B2Error("PlaTyPOOS cross-validation reached a node that explore() did not expand")
        if (err != 0).any():
            raise _lib.B2Error("PlaTyPOOS arena of %d nodes (layers of %d) exhausted"
                               % (self.node_capacity, self.layer_capacity))

    def _plans(self, res):
        plans = self.plan_buf.cpu().numpy()
        return [plans[i, :res[i, 2]].astype(int).tolist() for i in range(self.n_trees)]

    def tree_dict(self, tree=0):
        """The nodes of one tree in creation order, the fields of oracle/platypoos.py's dump: parent, action, depth,
        count, done, to_expand, cumulative_reward, value; and the candidates as [(p, node id)] in dict order."""
        n = int(self.result[tree, 0].item())
        get = {k: getattr(self, k)[tree, :n].cpu().numpy() for k in _lib.PLATYPOOS_TREE_FIELDS}
        out = {k: get[k] for k in ("parent", "action", "depth", "count")}
        out["done"] = get["flags"] & 1
        out["to_expand"] = (get["flags"] >> 1) & 1
        out["cumulative_reward"] = get["cumulative"]
        out["value"] = get["value"]
        cand = self.candidates[tree].cpu().numpy().reshape(-1, 2)
        out["candidates"] = [(int(p), int(c)) for p, c in cand[:int(self.result[tree, 6].item())]]
        return out
