"""Batched OPD engine (device side of DeterministicPlannerAgent)."""
import logging

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import FiniteTables
from rl_agents_b200.engine.tree_engine import HostTieEngine, decode_action

logger = logging.getLogger(__name__)


class _OPDTrees(HostTieEngine):
    """What every OPD kernel reads besides its config, workspace and per-node `state`: the gamma and terminal-bonus
    tables, the finite tables and the node arrays, torch tensors [n_trees, node_capacity] kept resident in HBM
    between decisions; `plan()` enqueues the search, `finish()` synchronises, raises the reference's errors and
    returns the plans."""

    def __init__(self, env_kind, n_trees, n_actions, budget, gamma, terminal_reward, mdp, device):
        super(_OPDTrees, self).__init__(n_trees, n_actions, budget, gamma, terminal_reward, device, gamma_pow_div=True)
        self.env_kind = env_kind
        self.tables = FiniteTables(mdp, self.device) if env_kind == _lib.ENV_FINITE else None
        self._nodes = self._alloc_tree(_lib.OPD_TREE_FIELDS, self.capacity)

    def _alloc_state(self, *shape):
        """The per-node int32 `state` of the given leading shape (a state id, or 136 words of a scene) -> `tree`."""
        words = () if self.env_kind == _lib.ENV_FINITE else (_lib.HW_STATE_WORDS,)
        self.state = self.torch.empty(shape + words, dtype=self.torch.int32, device=self.device)
        self.tree = _lib.OPDTree(*self._nodes, self.state.data_ptr())

    def _check(self, res):
        super(_OPDTrees, self)._check(res)
        if int(res[:, 3].sum()):
            logger.warning("Expanding a terminal state")                          # deterministic.py:111-112

    def tree_dict(self, tree=0):
        """Host copy of one tree in the layout of the oracle / golden dumps."""
        n = int(self.result[tree, 0].item())
        meta = self.meta[tree, :n].cpu().numpy()
        return {"parent": self.parent[tree, :n].cpu().numpy(), "action": decode_action(meta),
                "count": self.count[tree, :n].cpu().numpy(), "depth": self.depth[tree, :n].cpu().numpy(),
                "first_child": self.first_child[tree, :n].cpu().numpy(), "n_children": (meta >> 8) & 0xff,
                "done": ((meta >> 16) & 1).astype(bool), "reward": self.reward[tree, :n].cpu().numpy(),
                "lower": self.lower[tree, :n].cpu().numpy(), "upper": self.upper[tree, :n].cpu().numpy()}


class OPDEngine(_OPDTrees):
    """n_trees independent OPD decisions per launch (one CTA per tree).  `kernel` fills b2_opd_config.reserved,
    which must be 0: plan() raises B2Error otherwise."""

    def __init__(self, env_kind, n_trees, n_actions, budget, gamma, terminal_reward=0.0, mdp=None,
                 device="cuda", keys_in_smem=False, kernel=0):
        super(OPDEngine, self).__init__(env_kind, n_trees, n_actions, budget, gamma, terminal_reward, mdp, device)
        self._alloc_state(self.n_trees, self.capacity)
        self.cfg = _lib.OPDConfig(env_kind, self.n_trees, self.n_actions, self.n_expansions, self.capacity,
                                  self.plan_capacity, 1 if keys_in_smem else 0, int(kernel), float(terminal_reward),
                                  self.gamma_pow.data_ptr(), self.gamma_pow_div.data_ptr(),
                                  self.tables.struct() if self.tables else _lib.FiniteMDP(),
                                  self.terminal_bonus.data_ptr())
        ws = self.lib.b2_opd_workspace_bytes(self.cfg)
        if ws < 0:
            raise _lib.B2Error("unsupported OPD configuration")
        self.workspace = self.torch.empty(max(int(ws), 8), dtype=self.torch.uint8, device=self.device)

    def plan(self, root_states):
        """root_states: int32 device tensor [n_trees] (finite) or [n_trees, 136]."""
        assert root_states.dtype == self.torch.int32 and root_states.is_cuda and root_states.is_contiguous()
        _lib.check(self.lib.b2_opd_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.workspace),
                                        _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))


class _OPDWholeGPU(_OPDTrees):
    """ONE OPD decision searched by the whole GPU (n_trees = 1), configured by an OPDWaveConfig."""

    def __init__(self, env_kind, n_actions, budget, gamma, width, terminal_reward, mdp, device, max_ctas, n_models=0):
        super(_OPDWholeGPU, self).__init__(env_kind, 1, n_actions, budget, gamma, terminal_reward, mdp, device)
        self.width = int(width)
        self.cfg = _lib.OPDWaveConfig(env_kind, self.n_actions, self.n_expansions, self.capacity, self.plan_capacity,
                                      self.width, int(max_ctas), int(n_models), self.gamma_pow.data_ptr(),
                                      self.gamma_pow_div.data_ptr(), self.terminal_bonus.data_ptr(),
                                      self.tables.struct() if self.tables else _lib.FiniteMDP())

    @property
    def n_waves(self):
        return int(self.result[0, 7].item())


class OPDWaveEngine(_OPDWholeGPU):
    """ONE OPD decision searched by the whole GPU in waves of `width` leaves (b2_opd_plan_wave).

    width = 1 is the reference's strict best-first order; any width is bit-identical with the specification
    oracle/planners.py::opd_plan_wavefront.  Same tensors / finish() / tree_dict() as OPDEngine with
    n_trees = 1."""

    def __init__(self, env_kind, n_actions, budget, gamma, width, terminal_reward=0.0, mdp=None, device="cuda",
                 max_ctas=0, n_models=0, model_mdps=None):
        """n_models = M >= 1: DROP (DiscreteRobustPlanner, rl_agents/agents/robust/robust.py) -- the joint env of M
        models; `model_mdps`: the M finite MDPs (env_kind FINITE), root states [M] ids or [M, 136] words (HighwayLite or
        IntersectionLite scenes, one per model)."""
        first = model_mdps[0] if (model_mdps and env_kind == _lib.ENV_FINITE) else mdp
        super(OPDWaveEngine, self).__init__(env_kind, n_actions, budget, gamma, width, terminal_reward, first, device,
                                            max_ctas, n_models)
        self.n_models = int(n_models)
        self.model_tables = []
        if self.n_models > 0:
            if self.n_models > 8:
                raise ValueError("at most 8 models")
            if env_kind == _lib.ENV_FINITE:
                if not model_mdps or len(model_mdps) != self.n_models:
                    raise ValueError("model_mdps must list one finite MDP per model")
                self.model_tables = [FiniteTables(m, self.device) for m in model_mdps]
            self._alloc_state(1, self.capacity, self.n_models)
        else:
            self._alloc_state(1, self.capacity)
        for m, tab in enumerate(self.model_tables):
            self.cfg.model_mdps[m] = tab.struct()
        ws = self.lib.b2_opd_wave_workspace_bytes(self.cfg)
        if ws < 0:
            raise _lib.B2Error("unsupported wavefront OPD configuration")
        self.workspace = self.torch.empty(int(ws), dtype=self.torch.uint8, device=self.device)

    def plan(self, root_state):
        """root_state: int32 device tensor [1] (finite) or [136] / [1, 136]."""
        assert root_state.dtype == self.torch.int32 and root_state.is_cuda and root_state.is_contiguous()
        _lib.check(self.lib.b2_opd_plan_wave(self.cfg, _lib.ptr(root_state), self.tree, _lib.ptr(self.workspace),
                                             _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))


class OPDSpeculativeEngine(_OPDWholeGPU):
    """ONE OPD decision in the reference's strict best-first order (deterministic.py:106-114), searched by the
    whole GPU (b2_opd_plan_spec): per wave the `width` best frontier leaves are simulated speculatively (once:
    results stay cached until the leaf is expanded) and the prefix the strict order would have taken is
    committed.  The tree is bit-identical with OPDEngine's; `state` is an arena (a node's scene is not at its
    index).  Trees up to 24576 nodes."""

    def __init__(self, env_kind, n_actions, budget, gamma, width=64, terminal_reward=0.0, mdp=None, device="cuda",
                 max_ctas=0):
        super(OPDSpeculativeEngine, self).__init__(env_kind, n_actions, budget, gamma, width, terminal_reward, mdp,
                                                   device, max_ctas)
        ws = self.lib.b2_opd_spec_workspace_bytes(self.cfg)
        slots = self.lib.b2_opd_spec_arena_slots(self.cfg)
        if ws < 0 or slots < 0:
            raise _lib.B2Error("unsupported speculative OPD configuration (width <= 256, tree <= 24576 nodes)")
        self._alloc_state(1, int(slots))
        self.workspace = self.torch.empty(int(ws), dtype=self.torch.uint8, device=self.device)

    def plan(self, root_state):
        assert root_state.dtype == self.torch.int32 and root_state.is_cuda and root_state.is_contiguous()
        _lib.check(self.lib.b2_opd_plan_spec(self.cfg, _lib.ptr(root_state), self.tree, _lib.ptr(self.workspace),
                                             _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))
