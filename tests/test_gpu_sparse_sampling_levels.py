"""GPU tests of the level-synchronous sparse-sampling search (b2_sparse_sampling_plan_levels,
csrc/sparse_sampling_levels.cu): ONE decision on a deterministic model, searched by the whole GPU.

Every comparison is exact: the creation-order dump (every field, the float64 bytes of `value` included), root_q, the
plan, all eight result words and all six PCG64 words -- against the reference's goldens and against the depth-first
lane kernel (b2_sparse_sampling_plan) on the same roots and streams."""
import types

import numpy as np
import pytest

from oracle import ref_loader
from tests.test_gpu_sparse_sampling import device_digest, pcg64_of, roots, words_state
from tests.test_sparse_sampling_oracle import G, M, case_env, completed_planner_config, golden_root_q

pytestmark = pytest.mark.gpu

DETERMINISTIC_GOLDENS = ("hw0_shipped", "hw1_shipped", "hw2_shipped", "hw3_shipped", "hw1_h2_c2_g0.8",
                         "large1_deterministic_shipped", "trap_deterministic_shipped", "trap_terminal_root_shipped")


def capacity(n_actions, horizon, C):
    """Room for the full-width deterministic tree, and for the lane kernel's look-ahead check of 1 + C nodes."""
    from rl_agents_b200.engine.sparse_sampling import deterministic_nodes
    return deterministic_nodes(n_actions, horizon) + C + 2


def level_engine(kind, n_actions, horizon, C, gamma, mdp=None, record=True, cap=None):
    from rl_agents_b200.engine.sparse_sampling import SparseSamplingLevelEngine
    return SparseSamplingLevelEngine(kind, 1, n_actions, horizon, C, gamma, mdp=mdp, record_tree=record,
                                     capacity=cap if cap is not None else capacity(n_actions, horizon, C))


def tree_bits(eng, i):
    d = eng.tree_dict(i)
    d["value"] = d["value"].view(np.int64)
    return d


def assert_same_decisions(kind, n_actions, horizon, C, gamma, root_t, words, mdp=None):
    """The lane kernel plans every root in one batch; the level kernel plans them one by one: every output equal."""
    from rl_agents_b200.engine.sparse_sampling import SparseSamplingEngine
    n = root_t.shape[0]
    cap = capacity(n_actions, horizon, C)
    lane = SparseSamplingEngine(kind, n, n_actions, horizon, C, gamma, mdp=mdp, record_tree=True, capacity=cap)
    lane.plan(root_t, words)
    lplans, lres, lwords = lane.finish()
    lq = lane.root_q.cpu().numpy()
    lplan = lane.plan_buf.cpu().numpy()
    lev = level_engine(kind, n_actions, horizon, C, gamma, mdp=mdp, cap=cap)
    for i in range(n):
        lev.plan(root_t[i:i + 1].contiguous(), words[i:i + 1])
        plans, res, w = lev.finish()
        ctx = (horizon, C, gamma, i)
        assert plans[0] == lplans[i], ctx
        assert res[0].tolist() == lres[i].tolist(), ctx
        assert w[0].tolist() == lwords[i].tolist(), ctx
        assert lev.plan_buf.cpu().numpy()[0] == lplan[i], ctx
        assert lev.root_q.cpu().numpy()[0].tobytes() == lq[i].tobytes(), ctx
        a, b = tree_bits(lev, 0), tree_bits(lane, i)
        for f in a:
            assert np.array_equal(a[f], b[f]), (f,) + ctx
    return lres


@pytest.mark.parametrize("key", DETERMINISTIC_GOLDENS)
def test_level_kernel_matches_reference_golden(key):
    from oracle import envs as oenvs
    from rl_agents_b200 import _lib
    g = G["cases"][key]
    cfg = completed_planner_config(g["config"])
    env = case_env(g["env"])
    finite = isinstance(env, oenvs.FiniteMDPLite)
    eng = level_engine(_lib.ENV_FINITE if finite else _lib.ENV_HIGHWAY, env.action_space.n, cfg["horizon"], cfg["C"],
                       cfg["gamma"], mdp=env.mdp if finite else None)
    words = pcg64_of([g["seed"]])
    plans = []
    for _ in range(len(g.get("plans", [g["plan"]]))):
        eng.plan(roots([env]), words)
        p, res, words = eng.finish()
        plans.append(p[0])
    assert plans == g.get("plans", [g["plan"]])
    assert (int(res[0, 0]), int(res[0, 1]), int(res[0, 2])) == (g["tree"]["n_nodes"], g["chance_nodes"], g["samples"])
    assert (int(res[0, 3]), int(res[0, 4]), int(res[0, 5])) == (g["plan"][0], 0, -1)
    assert words_state(words[0]) == g["rng_state"]
    assert np.array_equal(eng.root_q[0].cpu().numpy(), golden_root_q(g), equal_nan=True)
    assert device_digest(eng, 0) == g["tree"]


def highway_roots():
    """64 scenes: make_scene(i), and the step's edge families -- crashed vehicles, absent slots with stale words, exact
    x ties at entry and later, jams and kinematic edges."""
    import torch
    from rl_agents_b200.envs.highway_lite import make_scene
    from tests import highway_scenes as hs
    words = [make_scene(i) for i in range(16)]
    for name in ("absent", "entry_ties", "late_ties", "jam", "kinematic", "adapter", "sync_timers"):
        words += [s.pack() for s in hs.family(name)[:7]]
    words = words[:64]
    assert len(words) == 64
    return torch.from_numpy(np.stack(words).astype(np.int32)).cuda()


@pytest.mark.parametrize("horizon", [1, 2, 3, 4, 5])
def test_highway_level_kernel_equals_the_lane_kernel(horizon):
    from rl_agents_b200 import _lib
    root_t = highway_roots()
    words = pcg64_of([500 + i for i in range(64)])
    for C in (1, 2, 3, 5):
        for gamma in (0.7, 0.95):
            assert_same_decisions(_lib.ENV_HIGHWAY, 5, horizon, C, gamma, root_t, words)


def test_one_highway_decision_at_horizon_6_equals_the_lane_kernel():
    from rl_agents_b200 import _lib
    res = assert_same_decisions(_lib.ENV_HIGHWAY, 5, 6, 3, 0.7, highway_roots()[:1], pcg64_of([9]))
    assert res[0, 1] > 1000


def det_mdp(S, A, seed, equal_rewards=False):
    rs = np.random.default_rng(seed)
    return types.SimpleNamespace(mode="deterministic", transition=rs.integers(0, S, size=(S, A)),
                                 reward=np.full((S, A), 0.5) if equal_rewards else rs.random((S, A)),
                                 terminal=np.zeros(S, dtype=bool))


def buffered_words(seeds):
    """Planner streams with a 32-bit half already buffered (one integers(2) draw taken)."""
    from rl_agents_b200.engine.mcts import pcg64_words
    out = []
    for s in seeds:
        g = ref_loader.legacy_np_random(s)[0]
        g.integers(2)
        w = pcg64_words(g)
        assert w[4] == 1
        out.append(w)
    return np.stack(out)


def finite_roots(states):
    import torch
    return torch.tensor(states, dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("horizon", [1, 2, 3, 4, 5, 6])
def test_deterministic_garnet_and_trap_level_kernel_equals_the_lane_kernel(horizon):
    from rl_agents_b200 import _lib
    cases = [(det_mdp(1000, 4, 1), 4, [0, 17, 999, 500]),
             # A = 3, C = 3: an odd number of halves at odd horizons, from an empty and from a full buffer
             (det_mdp(50, 3, 2), 3, [1, 2, 3, 49]),
             # every reward equal: every root action ties and the tie-break draws after the skip
             (det_mdp(20, 4, 3, equal_rewards=True), 4, [0, 5, 6, 7])]
    trap = types.SimpleNamespace(mode="deterministic", transition=M["trap_T"], reward=M["trap_R"],
                                 terminal=M["trap_term"])
    cases.append((trap, M["trap_T"].shape[1], list(range(min(4, M["trap_T"].shape[0])))))
    for mdp, A, states in cases:
        for words in (pcg64_of([10 + s for s in range(len(states))]), buffered_words(range(len(states)))):
            for C, gamma in ((3, 0.7), (2, 0.95)):
                assert_same_decisions(_lib.ENV_FINITE, A, horizon, C, gamma, finite_roots(states), words, mdp=mdp)


def test_all_equal_rewards_tie_break_draws_after_the_skip():
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import set_pcg64_words
    from oracle.pcg64 import PCG64
    from tests.test_pcg64_skip import skip32
    mdp = det_mdp(20, 4, 3, equal_rewards=True)
    eng = level_engine(_lib.ENV_FINITE, 4, 3, 3, 0.7, mdp=mdp)
    w0 = pcg64_of([4])
    eng.plan(finite_roots([0]), w0)
    plans, res, w = eng.finish()
    p = PCG64.from_words(w0[0])
    skip32(p, 3 * int(res[0, 1]))
    g = np.random.Generator(np.random.PCG64(0))
    set_pcg64_words(g, p.words())
    assert plans[0] == [int(g.choice(np.arange(4)))]
    assert PCG64.from_numpy(g).words().tolist() == w[0].tolist()


def test_agent_selects_the_engine_and_plans_the_lane_engine_bits(monkeypatch):
    from rl_agents_b200.agents.tree_search import sparse_sampling as ssmod
    from rl_agents_b200.agents.tree_search.sparse_sampling import SparseSamplingAgent
    from rl_agents_b200.engine.sparse_sampling import SparseSamplingEngine, SparseSamplingLevelEngine
    from rl_agents_b200.envs import FiniteMDPEnv, HighwayLiteEnv
    from rl_agents_b200.envs.adapters import describe
    cfg = {"gamma": 0.7, "horizon": 3, "C": 3}

    def engine_of(env):
        agent = SparseSamplingAgent(env, dict(cfg))
        agent.seed(1)
        if isinstance(env, HighwayLiteEnv):
            agent.act(None)
        else:
            agent.plan(0)
        return type(agent.planner.engine)
    assert engine_of(HighwayLiteEnv(seed=0)) is SparseSamplingLevelEngine
    assert engine_of(FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"])) is SparseSamplingLevelEngine
    for name in ("stoch8", "garnet12"):
        t = G["mdps"][name]
        env = FiniteMDPEnv(np.array(t["transition"]), np.array(t["reward"]), np.array(t["terminal"]), mode=t["mode"],
                           nxt=None if "next" not in t else np.array(t["next"]))
        assert engine_of(env) is SparseSamplingEngine, name
    # above the workspace cap: the lane engine
    d = describe(HighwayLiteEnv(seed=0))
    assert ssmod.use_level_engine(d, 1, 3) and ssmod.use_level_engine(d, 6, 3) and not ssmod.use_level_engine(d, 11, 3)
    # a finite tree below the measured size keeps the lane engine
    d = describe(FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"]))
    assert d.n_actions == 5 and not ssmod.use_level_engine(d, 2, 3) and ssmod.use_level_engine(d, 3, 3)
    monkeypatch.setattr(ssmod, "LEVEL_WORKSPACE_CAP", 1 << 10)
    assert engine_of(HighwayLiteEnv(seed=0)) is SparseSamplingEngine
    monkeypatch.undo()

    # a 10-step closed-loop episode: plans and stream equal those of an agent held on the lane engine
    envs, agents = [HighwayLiteEnv(seed=3), HighwayLiteEnv(seed=3)], []
    for env in envs:
        env.reset()
        agent = SparseSamplingAgent(env, dict(cfg))
        agent.seed(42)
        agents.append(agent)
    lane_rule = lambda *args: False                       # noqa: E731
    for k in range(10):
        a0 = agents[0].act(None)
        with monkeypatch.context() as m:
            m.setattr(ssmod, "use_level_engine", lane_rule)
            a1 = agents[1].act(None)
        assert isinstance(agents[0].planner.engine, SparseSamplingLevelEngine)
        assert isinstance(agents[1].planner.engine, SparseSamplingEngine) and \
            not isinstance(agents[1].planner.engine, SparseSamplingLevelEngine)
        assert a0 == a1, k
        assert agents[0].planner.np_random.bit_generator.state == agents[1].planner.np_random.bit_generator.state, k
        assert agents[0].planner.root_values.tobytes() == agents[1].planner.root_values.tobytes(), k
        out = [env.step(a0) for env in envs]
        assert out[0][1] == out[1][1]
        if out[0][2] or out[0][3]:
            break


def test_c_abi_refusals_and_capacity():
    import ctypes
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.sparse_sampling import SparseSamplingLevelEngine
    lib = _lib.load()
    env = case_env({"name": "stoch8"})
    mdp = det_mdp(30, 4, 5)
    eng = level_engine(_lib.ENV_FINITE, 4, 3, 3, 0.7, mdp=mdp)
    root, words = finite_roots([0]), pcg64_of([0])

    def refused(match):
        with pytest.raises(_lib.B2Error, match=match):
            eng.plan(root, words)
    eng.cfg.n_trees = 2
    refused("n_trees")
    eng.cfg.n_trees = 1
    eng.cfg.mdp.n_next = 3
    refused("n_next")
    eng.cfg.mdp.n_next = 1
    eng.cfg.horizon = 0
    refused("horizon")
    eng.cfg.horizon, eng.cfg.C = 3, 0
    refused("C must be")
    eng.cfg.C, eng.cfg.horizon = 3, 20
    refused("int32")
    eng.cfg.horizon = 3
    assert lib.b2_sparse_sampling_plan_levels(eng.cfg, None, eng.tree, _lib.ptr(eng.workspace), _lib.ptr(eng.rng),
                                              _lib.ptr(eng.root_q), _lib.ptr(eng.plan_buf), _lib.ptr(eng.result),
                                              _lib.current_stream()) == 1      # B2_ERR_INVALID
    assert "null pointer" in lib.b2_last_error().decode()
    cfg = _lib.SparseSamplingConfig(_lib.ENV_HIGHWAY, 1, 5, 20, 3, 0, 0.7, _lib.FiniteMDPSampled())
    assert lib.b2_sparse_sampling_levels_workspace_bytes(ctypes.byref(cfg)) == 0
    # the engine refuses what the kernel refuses
    with pytest.raises(ValueError, match="n_trees"):
        SparseSamplingLevelEngine(_lib.ENV_FINITE, 2, 4, 3, 3, 0.7, mdp=mdp)
    with pytest.raises(ValueError, match="deterministic"):
        SparseSamplingLevelEngine(_lib.ENV_FINITE, 1, env.action_space.n, 3, 3, 0.7, mdp=env.mdp)
    # the plan still runs after the refusals; a dump too small for the tree sets error 1
    eng.plan(root, words)
    assert eng.finish()[1][0, 4] == 0
    small = level_engine(_lib.ENV_FINITE, 4, 3, 3, 0.7, mdp=mdp, cap=50)
    small.plan(root, words)
    with pytest.raises(RuntimeError, match="capacity"):
        small.finish()
    assert int(small.result[0, 4].item()) == 1
