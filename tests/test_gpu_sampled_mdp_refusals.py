"""GPU tests of the launch check shared by the five planners that step a sampled finite MDP (check_sampled_mdp in
csrc/common.cu): b2_olop_plan_sampled, b2_mdp_gape_plan_sampled, b2_mcts_dpw_plan, b2_platypoos_plan and
b2_sparse_sampling_plan each refuse missing tables, a bad shape and, where the planner reads it, a missing terminal
table, with B2_ERR_INVALID and without launching a kernel."""
import numpy as np
import pytest

from tests.mdp_gape_stochastic_cases import oracle_env
from tests.test_gpu_mdp_gape import pcg64_of, roots

pytestmark = pytest.mark.gpu
N_TREES = 2
UNWRITTEN = -7
KL = {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)",
      "transition_threshold": "0.1*np.log(time)"}
PLANNERS = ["olop", "mdp_gape", "mcts_dpw", "platypoos", "sparse_sampling"]
FAULTS = [("cdf", 0, "tables missing"), ("row_ok", 0, "tables missing"), ("next", 0, "tables missing"),
          ("n_next", 0, "finite MDP shape"), ("n_states", 0, "finite MDP shape"),
          ("n_actions", "mismatch", "finite MDP shape"), ("terminal", 0, None)]


def entry_point(planner, env):
    """-> (engine, call(mdp, terminal) -> the entry point's return code) on a batch of N_TREES trees of `env`."""
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts_dpw import MCTSDPWEngine
    from rl_agents_b200.engine.mdp_gape import MDPGapEEngine
    from rl_agents_b200.engine.olop import OLOPEngine
    from rl_agents_b200.engine.platypoos import PlaTyPOOSEngine
    from rl_agents_b200.engine.sparse_sampling import SparseSamplingEngine
    F, A, mdp = _lib.ENV_FINITE, env.action_space.n, env.mdp
    root = roots([env] * N_TREES)
    s = _lib.current_stream()
    if planner == "olop":
        eng = OLOPEngine(F, N_TREES, A, 4, 3, 0.8, KL, "uniform", mdp=mdp)
        call = lambda m, t: eng.lib.b2_olop_plan_sampled(
            eng.cfg, m, t, 1, _lib.ptr(root), eng.tree, _lib.ptr(eng.rng), _lib.ptr(eng.plan_buf),
            _lib.ptr(eng.result), s)
    elif planner == "mdp_gape":
        eng = MDPGapEEngine(F, N_TREES, A, 4, 2, 0.8, KL, 0.5, 0.9, max_next_states_count=4, mdp=mdp)
        call = lambda m, t: eng.lib.b2_mdp_gape_plan_sampled(
            eng.cfg, m, t, 1, _lib.ptr(root), eng.tree, _lib.ptr(eng.keys), _lib.ptr(eng.rng),
            _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), s)
    else:
        if planner == "mcts_dpw":
            eng = MCTSDPWEngine(F, N_TREES, A, 8, 3, 0.8, mdp=mdp)
            plan = lambda c: eng.lib.b2_mcts_dpw_plan(c, _lib.ptr(root), eng.tree, _lib.ptr(eng.rng),
                                                      _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), s)
        elif planner == "platypoos":
            eng = PlaTyPOOSEngine(F, N_TREES, A, 3, 0.8, mdp=mdp)
            plan = lambda c: eng.lib.b2_platypoos_plan(c, _lib.ptr(root), eng.tree, _lib.ptr(eng.workspace),
                                                       _lib.ptr(eng.rng), _lib.ptr(eng.plan_buf),
                                                       _lib.ptr(eng.candidates), _lib.ptr(eng.result), s)
        else:
            eng = SparseSamplingEngine(F, N_TREES, A, 2, 2, 0.8, mdp=mdp)
            plan = lambda c: eng.lib.b2_sparse_sampling_plan(c, _lib.ptr(root), eng.tree, _lib.ptr(eng.workspace),
                                                             _lib.ptr(eng.rng), _lib.ptr(eng.root_q),
                                                             _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), s)

        def call(m, t):
            c = type(eng.cfg).from_buffer_copy(eng.cfg)
            c.mdp = m
            if hasattr(c, "terminal"):
                c.terminal = t
            return plan(c)
    eng._load_rng(pcg64_of(range(N_TREES)))
    return eng, call


@pytest.mark.parametrize("planner", PLANNERS)
def test_sampled_mdp_launch_check_refuses_without_launching(planner):
    import torch
    env = oracle_env("garnet50")
    eng, call = entry_point(planner, env)
    terminal = torch.as_tensor(np.ascontiguousarray(env.mdp.terminal, dtype=np.uint8), device="cuda")
    good = eng.tables.struct()
    eng.result.fill_(UNWRITTEN)
    assert call(good, terminal.data_ptr()) == 0
    torch.cuda.synchronize()
    assert (eng.result != UNWRITTEN).any()                  # the accepted call launched and wrote its results
    for field, value, match in FAULTS:
        if field == "terminal" and planner == "sparse_sampling":
            continue                                        # sparse sampling does not read terminal
        m, t = eng.tables.struct(), terminal.data_ptr()
        if field == "terminal":
            t = None
        else:
            setattr(m, field, good.n_actions + 1 if value == "mismatch" else value)
        eng.result.fill_(UNWRITTEN)
        rc = call(m, t)
        torch.cuda.synchronize()
        assert rc == 1, (field, rc)                         # B2_ERR_INVALID
        if match is not None:
            assert match in eng.lib.b2_last_error().decode(), field
        assert (eng.result == UNWRITTEN).all(), field       # no kernel ran
