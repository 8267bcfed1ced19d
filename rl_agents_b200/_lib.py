"""ctypes binding of libb2planner.so (include/b2_planner.h).

The CUDA library IS the product: there is no CPU fallback.  Import of this
module never builds anything; `load()` raises if the library is missing.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2PLANNER_LIB") or os.path.join(HERE, "csrc", "libb2planner.so")   # env: kernel-variant experiments

c_void_p, c_int, c_int32, c_int64, c_double = (ctypes.c_void_p, ctypes.c_int, ctypes.c_int32,
                                               ctypes.c_int64, ctypes.c_double)

HW_STATE_WORDS = 136
HW_ACTIONS = 5
ENV_FINITE, ENV_HIGHWAY, ENV_INTERSECTION = 0, 1, 2
VI_DETERMINISTIC, VI_STOCHASTIC, VI_SPARSE = 0, 1, 2
OPD_RESULT_WORDS = 16
MCTS_RESULT_WORDS = 8
OLOP_RESULT_WORDS = 8
MDP_GAPE_RESULT_WORDS = 8
BRUE_RESULT_WORDS = 8
SPARSE_SAMPLING_RESULT_WORDS = 8
MCTS_DPW_RESULT_WORDS = 8
PLATYPOOS_RESULT_WORDS = 8
PCG64_STATE_WORDS = 6


class FiniteMDP(ctypes.Structure):
    _fields_ = [("n_states", c_int32), ("n_actions", c_int32), ("transition", c_void_p),
                ("reward", c_void_p), ("terminal", c_void_p)]


class VIProblem(ctypes.Structure):
    _fields_ = [("mode", c_int32), ("n_actions", c_int32), ("n_next", c_int32), ("reserved", c_int32),
                ("n_states", c_int64), ("row_begin", c_int64), ("row_end", c_int64),
                ("gamma", c_double), ("rtol", c_double), ("atol", c_double),
                ("transition", c_void_p), ("next", c_void_p), ("reward", c_void_p), ("terminal", c_void_p)]


MAX_PEERS = 8


class VIP2P(ctypes.Structure):
    _fields_ = [("world", c_int32), ("rank", c_int32), ("v", (c_void_p * MAX_PEERS) * 2),
                ("flags", c_void_p * MAX_PEERS), ("parts", c_void_p * MAX_PEERS),
                ("viol_local", c_void_p), ("done", c_void_p), ("status", c_void_p)]


class OPDConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_trees", c_int32), ("n_actions", c_int32),
                ("n_expansions", c_int32), ("node_capacity", c_int32), ("plan_capacity", c_int32),
                ("keys_in_smem", c_int32), ("reserved", c_int32), ("terminal_reward", c_double),
                ("gamma_pow", c_void_p), ("gamma_pow_div", c_void_p), ("mdp", FiniteMDP),
                ("terminal_bonus", c_void_p)]


class OPDWaveConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_actions", c_int32), ("n_expansions", c_int32),
                ("node_capacity", c_int32), ("plan_capacity", c_int32), ("width", c_int32),
                ("max_ctas", c_int32), ("n_models", c_int32), ("gamma_pow", c_void_p),
                ("gamma_pow_div", c_void_p), ("terminal_bonus", c_void_p), ("mdp", FiniteMDP),
                ("model_mdps", FiniteMDP * 8)]


class GBOPConfig(ctypes.Structure):
    _fields_ = [("n_trees", c_int32), ("n_actions", c_int32), ("n_expansions", c_int32), ("node_capacity", c_int32),
                ("plan_capacity", c_int32), ("queue_capacity", c_int32), ("backup_aggregated_nodes", c_int32),
                ("prune_suboptimal_leaves", c_int32), ("gamma", c_double), ("default_value", c_double),
                ("accuracy_scale", c_double), ("gamma_pow", c_void_p), ("terminal_bonus", c_void_p), ("mdp", FiniteMDP)]


class GBOPDConfig(ctypes.Structure):
    _fields_ = [("n_trees", c_int32), ("n_actions", c_int32), ("n_epochs", c_int32), ("sampling_timeout", c_int32),
                ("plan_capacity", c_int32), ("queue_capacity", c_int32), ("gamma", c_double), ("default_value", c_double),
                ("accuracy", c_double), ("mdp", FiniteMDP), ("rev_ptr", c_void_p), ("rev_idx", c_void_p)]


GBOP_TREE_FIELDS = ("parent", "first_child", "depth", "count", "meta", "reward", "lower", "obs")


class GBOPTree(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in GBOP_TREE_FIELDS]


OPD_TREE_FIELDS = ("parent", "first_child", "depth", "count", "meta", "reward", "lower", "upper")


class OPDTree(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in OPD_TREE_FIELDS + ("state",)]


class OPDHostConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_trees", c_int32), ("n_actions", c_int32), ("budget", c_int32),
                ("keys_in_smem", c_int32), ("kernel", c_int32), ("gamma", c_double), ("terminal_reward", c_double),
                ("mdp", FiniteMDP)]


class MCTSConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_trees", c_int32), ("n_actions", c_int32), ("episodes", c_int32),
                ("horizon", c_int32), ("node_capacity", c_int32), ("rollout_policy", c_int32),
                ("prior_policy", c_int32), ("temperature", c_double), ("gamma_pow", c_void_p),
                ("uniform_cdf", c_void_p), ("mdp", FiniteMDP), ("prior_pref_action", c_int32),
                ("rollout_pref_action", c_int32), ("pref_prior", c_void_p), ("pref_cdf", c_void_p),
                ("resume_nodes", c_void_p)]


class MCTSWaveConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_actions", c_int32), ("episodes", c_int32), ("horizon", c_int32),
                ("node_capacity", c_int32), ("width", c_int32), ("rollout_policy", c_int32),
                ("prior_policy", c_int32), ("temperature", c_double), ("seed", ctypes.c_uint64),
                ("gamma_pow", c_void_p), ("mdp", FiniteMDP), ("max_ctas", c_int32), ("reserved", c_int32)]


class MCTSWaveTree(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("parent", "first_child", "count", "meta", "vsum", "value")]


MCTS_TREE_FIELDS = ("parent", "first_child", "count", "meta", "value", "prior")


class MCTSTree(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in MCTS_TREE_FIELDS]


class OLOPConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_trees", c_int32), ("n_actions", c_int32), ("episodes", c_int32),
                ("horizon", c_int32), ("node_capacity", c_int32), ("kl", c_int32), ("continuation", c_int32),
                ("gamma", c_double), ("thresholds", c_void_p), ("init_upper", c_void_p), ("mdp", FiniteMDP)]


OLOP_TREE_FIELDS = ("parent", "first_child", "count", "meta", "cumulative", "mu_ucb", "upper")


class OLOPTree(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in OLOP_TREE_FIELDS]


class MDPGapEConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_trees", c_int32), ("n_actions", c_int32), ("episodes", c_int32),
                ("horizon", c_int32), ("node_capacity", c_int32), ("max_next_states", c_int32),
                ("continuation", c_int32), ("gamma", c_double), ("accuracy", c_double), ("thresholds", c_void_p),
                ("transition_thresholds", c_void_p), ("init_upper", c_void_p), ("mdp", FiniteMDP)]


MDP_GAPE_TREE_FIELDS = ("parent", "first_child", "count", "meta", "cumulative", "mu_ucb", "mu_lcb", "upper", "lower")


class MDPGapETree(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in MDP_GAPE_TREE_FIELDS]


class BRUEConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_trees", c_int32), ("n_actions", c_int32), ("budget", c_int32),
                ("horizon", c_int32), ("node_capacity", c_int32), ("gamma", c_double), ("gamma_pow", c_void_p),
                ("mdp", FiniteMDP)]


BRUE_TREE_FIELDS = ("parent", "first_child", "next_sibling", "count", "meta", "value")


class BRUETree(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in BRUE_TREE_FIELDS + ("path", "path_reward")]


class FiniteMDPSampled(ctypes.Structure):
    _fields_ = [("n_states", c_int32), ("n_actions", c_int32), ("n_next", c_int32), ("reserved", c_int32),
                ("cdf", c_void_p), ("next", c_void_p), ("reward", c_void_p), ("row_ok", c_void_p)]


class SparseSamplingConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_trees", c_int32), ("n_actions", c_int32), ("horizon", c_int32),
                ("C", c_int32), ("reserved", c_int32), ("gamma", c_double), ("mdp", FiniteMDPSampled)]


SPARSE_SAMPLING_TREE_FIELDS = ("parent", "kind", "key", "depth", "count", "value")


class SparseSamplingTree(ctypes.Structure):
    _fields_ = [("capacity", c_int32), ("reserved", c_int32)] + [(n, c_void_p) for n in SPARSE_SAMPLING_TREE_FIELDS]


class MCTSDPWConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_trees", c_int32), ("n_actions", c_int32), ("episodes", c_int32),
                ("horizon", c_int32), ("node_capacity", c_int32), ("rollout_policy", c_int32),
                ("rollout_pref_action", c_int32), ("closed_loop", c_int32), ("open_key", c_int32),
                ("env_draws", c_int32), ("reserved", c_int32), ("temperature", c_double), ("gamma_pow", c_void_p),
                ("uniform_cdf", c_void_p), ("pref_cdf", c_void_p), ("action_widen", c_void_p),
                ("state_widen", c_void_p), ("bonus", c_void_p), ("obs_keys", c_void_p), ("terminal", c_void_p),
                ("mdp", FiniteMDPSampled)]


MCTS_DPW_TREE_FIELDS = ("parent", "first_child", "next_sibling", "count", "kind", "key", "value")


class MCTSDPWTree(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in MCTS_DPW_TREE_FIELDS]


class PlaTyPOOSConfig(ctypes.Structure):
    _fields_ = [("env_kind", c_int32), ("n_trees", c_int32), ("n_actions", c_int32), ("horizon", c_int32),
                ("node_capacity", c_int32), ("layer_capacity", c_int32), ("max_p", c_int32), ("env_draws", c_int32),
                ("p_top", c_void_p), ("nodes_count", c_void_p), ("evaluations", c_void_p), ("min_visits", c_void_p),
                ("cv_count", c_void_p), ("gamma_pow", c_void_p), ("terminal", c_void_p), ("mdp", FiniteMDPSampled)]


PLATYPOOS_TREE_FIELDS = ("parent", "first_child", "action", "depth", "count", "flags", "state", "cumulative", "value",
                         "reward")


class PlaTyPOOSTree(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in PLATYPOOS_TREE_FIELDS]


EXPORTS = {
    "b2_last_error": (ctypes.c_char_p, []),
    "b2_version": (c_int, []),
    "b2_device_info": (c_int, [ctypes.POINTER(c_int)] * 3 + [ctypes.c_char_p, c_int]),
    "b2_intersection_step": (c_int, [c_void_p] * 5 + [c_int32, c_void_p]),
    "b2_selftest_const_division": (c_int, [c_void_p, c_void_p]),
    "b2_selftest_highway_step_groups": (c_int, [c_void_p] * 6 + [c_int32, c_int32, c_void_p]),
    "b2_selftest_pcg64": (c_int, [c_void_p] * 5 + [c_int32, c_int32, c_void_p]),
    "b2_selftest_kl": (c_int, [c_void_p, c_void_p, c_int32, c_void_p] + [c_void_p] * 4 + [c_int32, c_void_p, c_void_p]),
    "b2_selftest_sampled_next": (c_int, [c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_void_p,
                                         ctypes.POINTER(FiniteMDPSampled)] + [c_void_p] * 3 + [c_int32] +
                                 [c_void_p] * 3),
    "b2_selftest_gape_expectation": (c_int, [c_void_p] * 4 + [c_int32] + [c_void_p] * 5 + [c_int32, c_void_p, c_void_p]),
    "b2_highway_step": (c_int, [c_void_p] * 5 + [c_int32, c_void_p]),
    "b2_finite_step": (c_int, [ctypes.POINTER(FiniteMDPSampled), c_void_p, c_int32] + [c_void_p] * 7
                       + [c_int32, c_void_p]),
    "b2_highway_ttc_vi": (c_int, [c_void_p, c_int32, c_double, c_int32, c_double, c_double] + [c_void_p] * 5),
    "b2_vi_sweep": (c_int, [ctypes.POINTER(VIProblem)] + [c_void_p] * 5 + [c_int32, c_void_p]),
    "b2_vi_solve": (c_int, [ctypes.POINTER(VIProblem)] + [c_void_p] * 5 + [c_int32, c_void_p]),
    "b2_vi_robust_sweep": (c_int, [ctypes.POINTER(VIProblem), c_int32] + [c_void_p] * 5 + [c_int32, c_void_p]),
    "b2_p2p_alloc": (c_int, [c_int64, ctypes.POINTER(c_void_p)]),
    "b2_p2p_free": (c_int, [c_void_p]),
    "b2_p2p_export": (c_int, [c_void_p, ctypes.c_char_p]),
    "b2_p2p_import": (c_int, [ctypes.c_char_p, ctypes.POINTER(c_void_p)]),
    "b2_p2p_close": (c_int, [c_void_p]),
    "b2_p2p_memset": (c_int, [c_void_p, c_int32, c_int64, c_void_p]),
    "b2_p2p_read": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "b2_vi_sweep_p2p": (c_int, [ctypes.POINTER(VIProblem), ctypes.POINTER(VIP2P), c_void_p, c_void_p, c_int32, c_void_p]),
    "b2_opd_workspace_bytes": (c_int64, [ctypes.POINTER(OPDConfig)]),
    "b2_opd_plan": (c_int, [ctypes.POINTER(OPDConfig), c_void_p, ctypes.POINTER(OPDTree), c_void_p, c_void_p,
                            c_void_p, c_void_p]),
    "b2_opd_wave_workspace_bytes": (c_int64, [ctypes.POINTER(OPDWaveConfig)]),
    "b2_opd_plan_wave": (c_int, [ctypes.POINTER(OPDWaveConfig), c_void_p, ctypes.POINTER(OPDTree), c_void_p, c_void_p,
                                 c_void_p, c_void_p]),
    "b2_opd_spec_workspace_bytes": (c_int64, [ctypes.POINTER(OPDWaveConfig)]),
    "b2_opd_spec_arena_slots": (c_int64, [ctypes.POINTER(OPDWaveConfig)]),
    "b2_opd_plan_spec": (c_int, [ctypes.POINTER(OPDWaveConfig), c_void_p, ctypes.POINTER(OPDTree), c_void_p, c_void_p,
                                 c_void_p, c_void_p]),
    "b2_gbop_workspace_bytes": (c_int64, [ctypes.POINTER(GBOPConfig)]),
    "b2_gbop_plan": (c_int, [ctypes.POINTER(GBOPConfig), c_void_p, ctypes.POINTER(GBOPTree), c_void_p, c_void_p,
                             c_void_p, c_void_p]),
    "b2_gbopd_plan": (c_int, [ctypes.POINTER(GBOPDConfig)] + [c_void_p] * 9),
    "b2_opd_create": (c_int, [ctypes.POINTER(OPDHostConfig), ctypes.POINTER(c_void_p)]),
    "b2_opd_destroy": (None, [c_void_p]),
    "b2_opd_plan_capacity": (c_int32, [c_void_p]),
    "b2_opd_plan_host": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_opd_copy_tree": (c_int, [c_void_p, c_int32, c_int32] + [c_void_p] * 7),
    "b2_mcts_plan": (c_int, [ctypes.POINTER(MCTSConfig), c_void_p, ctypes.POINTER(MCTSTree), c_void_p, c_void_p,
                             c_void_p, c_void_p]),
    "b2_mcts_plan_sampled": (c_int, [ctypes.POINTER(MCTSConfig), ctypes.POINTER(FiniteMDPSampled), c_void_p, c_int32,
                                     c_void_p, c_void_p, ctypes.POINTER(MCTSTree)] + [c_void_p] * 4),
    "b2_mcts_reroot": (c_int, [ctypes.POINTER(MCTSTree), c_int32, c_int32, c_void_p, c_int32, ctypes.POINTER(MCTSTree),
                               c_int32, c_int32, c_void_p, c_void_p, c_int32, c_void_p, c_void_p]),
    "b2_mcts_wave_workspace_bytes": (c_int64, [ctypes.POINTER(MCTSWaveConfig)]),
    "b2_mcts_plan_wave": (c_int, [ctypes.POINTER(MCTSWaveConfig), c_void_p, ctypes.POINTER(MCTSWaveTree), c_void_p,
                                  c_void_p, c_void_p, c_void_p]),
    "b2_mcts_plan_wave_sampled": (c_int, [ctypes.POINTER(MCTSWaveConfig), ctypes.POINTER(FiniteMDPSampled), c_void_p,
                                          c_int32, c_void_p, c_void_p, ctypes.POINTER(MCTSWaveTree)] + [c_void_p] * 5),
    "b2_olop_plan": (c_int, [ctypes.POINTER(OLOPConfig), c_void_p, ctypes.POINTER(OLOPTree), c_void_p, c_void_p,
                             c_void_p, c_void_p]),
    "b2_olop_plan_sampled": (c_int, [ctypes.POINTER(OLOPConfig), ctypes.POINTER(FiniteMDPSampled), c_void_p, c_int32,
                                     c_void_p, ctypes.POINTER(OLOPTree)] + [c_void_p] * 4),
    "b2_mdp_gape_plan": (c_int, [ctypes.POINTER(MDPGapEConfig), c_void_p, ctypes.POINTER(MDPGapETree), c_void_p,
                                 c_void_p, c_void_p, c_void_p]),
    "b2_mdp_gape_plan_sampled": (c_int, [ctypes.POINTER(MDPGapEConfig), ctypes.POINTER(FiniteMDPSampled), c_void_p,
                                         c_int32, c_void_p, ctypes.POINTER(MDPGapETree)] + [c_void_p] * 5),
    "b2_brue_plan": (c_int, [ctypes.POINTER(BRUEConfig), c_void_p, ctypes.POINTER(BRUETree), c_void_p, c_void_p,
                             c_void_p, c_void_p]),
    "b2_sparse_sampling_workspace_bytes": (c_int64, [ctypes.POINTER(SparseSamplingConfig)]),
    "b2_sparse_sampling_plan": (c_int, [ctypes.POINTER(SparseSamplingConfig), c_void_p,
                                        ctypes.POINTER(SparseSamplingTree)] + [c_void_p] * 6),
    "b2_sparse_sampling_levels_workspace_bytes": (c_int64, [ctypes.POINTER(SparseSamplingConfig)]),
    "b2_sparse_sampling_plan_levels": (c_int, [ctypes.POINTER(SparseSamplingConfig), c_void_p,
                                               ctypes.POINTER(SparseSamplingTree)] + [c_void_p] * 6),
    "b2_mcts_dpw_plan": (c_int, [ctypes.POINTER(MCTSDPWConfig), c_void_p, ctypes.POINTER(MCTSDPWTree), c_void_p,
                                 c_void_p, c_void_p, c_void_p]),
    "b2_platypoos_workspace_bytes": (c_int64, [ctypes.POINTER(PlaTyPOOSConfig)]),
    "b2_platypoos_plan": (c_int, [ctypes.POINTER(PlaTyPOOSConfig), c_void_p, ctypes.POINTER(PlaTyPOOSTree)]
                          + [c_void_p] * 6),
}

_lib = None


class B2Error(RuntimeError):
    pass


def load():
    """Load the CUDA library; fail loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B2Error("%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)" % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in EXPORTS.items():
            fn = getattr(lib, name)      # AttributeError if a declared symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc):
    if rc != 0:
        raise B2Error("libb2planner error %d: %s" % (rc, load().b2_last_error().decode()))


def ptr(t):
    """data pointer of a torch tensor (or None)."""
    return None if t is None else c_void_p(t.data_ptr())


def current_stream():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)
