"""Batched OPD engine (device side of DeterministicPlannerAgent)."""
import logging

import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import FiniteTables, gamma_tables, terminal_bonus_table
from rl_agents_b200.engine.tree_engine import decode_action

logger = logging.getLogger(__name__)


class OPDEngine(object):
    """n_trees independent OPD decisions per launch (one CTA per tree).

    The node arrays are torch tensors [n_trees, node_capacity] kept resident in
    HBM between decisions; `plan()` enqueues the search, `finish()` synchronises,
    raises the reference's errors and returns the plans."""

    def __init__(self, env_kind, n_trees, n_actions, budget, gamma, terminal_reward=0.0, mdp=None,
                 device="cuda", keys_in_smem=False, kernel=0):
        import torch
        self.torch = torch
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.env_kind = env_kind
        self.n_trees, self.n_actions = int(n_trees), int(n_actions)
        self.n_expansions = int(budget) // self.n_actions            # deterministic.py:118
        self.capacity = 1 + self.n_expansions * self.n_actions
        self.plan_capacity = self.n_expansions + 1
        gp, gd = gamma_tables(gamma, self.n_expansions + 2)
        self.gamma_pow = torch.as_tensor(gp, device=self.device)
        self.gamma_pow_div = torch.as_tensor(gd, device=self.device)
        self.terminal_bonus = torch.as_tensor(terminal_bonus_table(terminal_reward, gamma, self.n_expansions + 2),
                                              device=self.device)
        self.tables = FiniteTables(mdp, self.device) if env_kind == _lib.ENV_FINITE else None
        shape = (self.n_trees, self.capacity)
        i32, f64 = torch.int32, torch.float64
        self.parent = torch.empty(shape, dtype=i32, device=self.device)
        self.first_child = torch.empty(shape, dtype=i32, device=self.device)
        self.depth = torch.empty(shape, dtype=i32, device=self.device)
        self.count = torch.empty(shape, dtype=i32, device=self.device)
        self.meta = torch.empty(shape, dtype=i32, device=self.device)
        self.reward = torch.empty(shape, dtype=f64, device=self.device)
        self.lower = torch.empty(shape, dtype=f64, device=self.device)
        self.upper = torch.empty(shape, dtype=f64, device=self.device)
        sshape = shape if env_kind == _lib.ENV_FINITE else shape + (_lib.HW_STATE_WORDS,)
        self.state = torch.empty(sshape, dtype=i32, device=self.device)
        self.cfg = _lib.OPDConfig(env_kind, self.n_trees, self.n_actions, self.n_expansions, self.capacity,
                                  self.plan_capacity, 1 if keys_in_smem else 0, int(kernel), float(terminal_reward),
                                  self.gamma_pow.data_ptr(), self.gamma_pow_div.data_ptr(),
                                  self.tables.struct() if self.tables else _lib.FiniteMDP(),
                                  self.terminal_bonus.data_ptr())
        self.tree = _lib.OPDTree(*[t.data_ptr() for t in (self.parent, self.first_child, self.depth, self.count,
                                                          self.meta, self.reward, self.lower, self.upper, self.state)])
        ws = self.lib.b2_opd_workspace_bytes(self.cfg)
        if ws < 0:
            raise _lib.B2Error("unsupported OPD configuration")
        self.workspace = torch.empty(max(int(ws), 8), dtype=torch.uint8, device=self.device)
        self.plan_buf = torch.empty((self.n_trees, self.plan_capacity), dtype=torch.int8, device=self.device)
        self.result = torch.empty((self.n_trees, _lib.OPD_RESULT_WORDS), dtype=i32, device=self.device)

    def plan(self, root_states):
        """root_states: int32 device tensor [n_trees] (finite) or [n_trees, 136]."""
        assert root_states.dtype == self.torch.int32 and root_states.is_cuda and root_states.is_contiguous()
        _lib.check(self.lib.b2_opd_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.workspace),
                                        _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def finish(self, np_randoms=None):
        """Synchronise; returns (plans, result array).  Ties in get_plan are broken
        on the host with the planner RNG exactly as abstract.py:304-311 does."""
        res = self.result.cpu().numpy()
        if (res[:, 4] != 0).any():
            raise ValueError("This planner assumes that all rewards are normalized in [0, 1]")  # :46-47
        n_term = int(res[:, 3].sum())
        if n_term:
            logger.warning("Expanding a terminal state")                                         # :111-112
        plans_dev = self.plan_buf.cpu().numpy()
        plans = []
        for i in range(self.n_trees):
            plan = plans_dev[i, :res[i, 5]].astype(int).tolist()
            if res[i, 6] >= 0:
                rng = np_randoms[i] if np_randoms is not None else np.random.default_rng()
                plan += self._host_plan_from(i, int(res[i, 6]), rng)
            plans.append(plan)
        return plans, res

    def _host_plan_from(self, tree, node, rng):
        fc = self.first_child[tree].cpu().numpy()
        meta = self.meta[tree].cpu().numpy()
        lower = self.lower[tree].cpu().numpy()
        plan = []
        while fc[node] >= 0:
            n = (meta[node] >> 8) & 0xff
            x = lower[fc[node]:fc[node] + n]
            indices = np.nonzero(x == np.amax(x))[0]
            node = fc[node] + int(rng.choice(indices))
            plan.append(int(meta[node] & 0xff))
        return plan

    def tree_dict(self, tree=0):
        """Host copy of one tree in the layout of the oracle / golden dumps."""
        n = int(self.result[tree, 0].item())
        meta = self.meta[tree, :n].cpu().numpy()
        return {"parent": self.parent[tree, :n].cpu().numpy(), "action": decode_action(meta),
                "count": self.count[tree, :n].cpu().numpy(), "depth": self.depth[tree, :n].cpu().numpy(),
                "first_child": self.first_child[tree, :n].cpu().numpy(), "n_children": (meta >> 8) & 0xff,
                "done": ((meta >> 16) & 1).astype(bool), "reward": self.reward[tree, :n].cpu().numpy(),
                "lower": self.lower[tree, :n].cpu().numpy(), "upper": self.upper[tree, :n].cpu().numpy()}


class OPDWaveEngine(OPDEngine):
    """ONE OPD decision searched by the whole GPU in waves of `width` leaves (b2_opd_plan_wave).

    width = 1 is the reference's strict best-first order; any width is bit-identical with the specification
    oracle/planners.py::opd_plan_wavefront.  Same tensors / finish() / tree_dict() as OPDEngine with
    n_trees = 1."""

    def __init__(self, env_kind, n_actions, budget, gamma, width, terminal_reward=0.0, mdp=None, device="cuda",
                 max_ctas=0, n_models=0, model_mdps=None):
        """n_models = M >= 1: DROP (DiscreteRobustPlanner, rl_agents/agents/robust/robust.py) -- the joint env of M
        models; `model_mdps`: the M finite MDPs (env_kind FINITE), root states [M] ids or [M, 136] words."""
        first = model_mdps[0] if (model_mdps and env_kind == _lib.ENV_FINITE) else mdp
        super(OPDWaveEngine, self).__init__(env_kind, 1, n_actions, budget, gamma, terminal_reward, first, device)
        self.width = int(width)
        self.n_models = int(n_models)
        torch = self.torch
        self.model_tables = []
        if self.n_models > 0:
            if self.n_models > 8:
                raise ValueError("at most 8 models")
            if env_kind == _lib.ENV_FINITE:
                if not model_mdps or len(model_mdps) != self.n_models:
                    raise ValueError("model_mdps must list one finite MDP per model")
                self.model_tables = [FiniteTables(m, self.device) for m in model_mdps]
                self.state = torch.empty((1, self.capacity, self.n_models), dtype=torch.int32, device=self.device)
            else:
                self.state = torch.empty((1, self.capacity, self.n_models, _lib.HW_STATE_WORDS), dtype=torch.int32,
                                         device=self.device)
            self.tree = _lib.OPDTree(*[t.data_ptr() for t in (self.parent, self.first_child, self.depth, self.count,
                                                              self.meta, self.reward, self.lower, self.upper, self.state)])
        self.wcfg = _lib.OPDWaveConfig(env_kind, self.n_actions, self.n_expansions, self.capacity, self.plan_capacity,
                                       self.width, int(max_ctas), self.n_models, self.gamma_pow.data_ptr(),
                                       self.gamma_pow_div.data_ptr(), self.terminal_bonus.data_ptr(),
                                       self.tables.struct() if self.tables else _lib.FiniteMDP())
        for m, tab in enumerate(self.model_tables):
            self.wcfg.model_mdps[m] = tab.struct()
        ws = self.lib.b2_opd_wave_workspace_bytes(self.wcfg)
        if ws < 0:
            raise _lib.B2Error("unsupported wavefront OPD configuration")
        self.workspace = self.torch.empty(int(ws), dtype=self.torch.uint8, device=self.device)

    def plan(self, root_state):
        """root_state: int32 device tensor [1] (finite) or [136] / [1, 136]."""
        assert root_state.dtype == self.torch.int32 and root_state.is_cuda and root_state.is_contiguous()
        _lib.check(self.lib.b2_opd_plan_wave(self.wcfg, _lib.ptr(root_state), self.tree, _lib.ptr(self.workspace),
                                             _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    @property
    def n_waves(self):
        return int(self.result[0, 7].item())


class OPDSpeculativeEngine(OPDEngine):
    """ONE OPD decision in the reference's strict best-first order (deterministic.py:106-114), searched by the
    whole GPU (b2_opd_plan_spec): per wave the `width` best frontier leaves are simulated speculatively (once:
    results stay cached until the leaf is expanded) and the prefix the strict order would have taken is
    committed.  The tree is bit-identical with OPDEngine's; `state` is an arena (a node's scene is not at its
    index).  Trees up to 24576 nodes."""

    def __init__(self, env_kind, n_actions, budget, gamma, width=64, terminal_reward=0.0, mdp=None, device="cuda",
                 max_ctas=0):
        super(OPDSpeculativeEngine, self).__init__(env_kind, 1, n_actions, budget, gamma, terminal_reward, mdp, device)
        self.width = int(width)
        torch = self.torch
        self.wcfg = _lib.OPDWaveConfig(env_kind, self.n_actions, self.n_expansions, self.capacity, self.plan_capacity,
                                       self.width, int(max_ctas), 0, self.gamma_pow.data_ptr(),
                                       self.gamma_pow_div.data_ptr(), self.terminal_bonus.data_ptr(),
                                       self.tables.struct() if self.tables else _lib.FiniteMDP())
        ws = self.lib.b2_opd_spec_workspace_bytes(self.wcfg)
        slots = self.lib.b2_opd_spec_arena_slots(self.wcfg)
        if ws < 0 or slots < 0:
            raise _lib.B2Error("unsupported speculative OPD configuration (width <= 256, tree <= 24576 nodes)")
        sshape = (1, int(slots)) if env_kind == _lib.ENV_FINITE else (1, int(slots), _lib.HW_STATE_WORDS)
        self.state = torch.empty(sshape, dtype=torch.int32, device=self.device)
        self.tree = _lib.OPDTree(*[t.data_ptr() for t in (self.parent, self.first_child, self.depth, self.count,
                                                          self.meta, self.reward, self.lower, self.upper, self.state)])
        self.workspace = torch.empty(int(ws), dtype=torch.uint8, device=self.device)

    def plan(self, root_state):
        assert root_state.dtype == self.torch.int32 and root_state.is_cuda and root_state.is_contiguous()
        _lib.check(self.lib.b2_opd_plan_spec(self.wcfg, _lib.ptr(root_state), self.tree, _lib.ptr(self.workspace),
                                             _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    @property
    def n_waves(self):
        return int(self.result[0, 7].item())
