"""GPU tests of MCTS on stochastic finite MDPs: b2_mcts_plan_sampled (csrc/mcts.cu) and b2_mcts_plan_wave_sampled
(csrc/mcts_wave.cu), through MCTSEngine, MCTSWaveEngine and MCTSAgent.

Every episode's env copy replays the live env's generator, whose words the planner hands the device.  The per-tree
kernel is checked against the reference's goldens (tests/golden/golden_mcts_stochastic.json) and node by node against
the oracle (oracle/planners.py::mcts_plan) on batches of 256 trees; the wavefront kernel against its specification
(oracle/planners.py::mcts_plan_wavefront).  Everything is exact, floats included."""
import copy

import numpy as np
import pytest

from oracle import planners
from tests.mcts_stochastic_cases import (MDPS, canonical_digest, live_env, planner_rng, policy, rng_state,
                                         rng_words_state, tree_digest)
from tests.mdp_gape_stochastic_cases import oracle_env, product_env
from tests.test_gpu_mcts_dpw import mixed_finite_mdp
from tests.test_gpu_mdp_gape import roots
from tests.test_gpu_sampled_mdp_refusals import FAULTS
from tests.util import load_golden

pytestmark = pytest.mark.gpu
G = load_golden("golden_mcts_stochastic.json")
UNWRITTEN = -7
PREF_PRIOR = {"type": "preference", "action": 1, "ratio": 3}
PREF_ROLLOUT = {"type": "preference", "action": 2, "ratio": 2}


def case_of(g):
    return (g["mdp"], g["state"], g["config"], g["seed"], g["env_seed"], g["advance"])


def words(gen):
    from rl_agents_b200.engine.mcts import pcg64_words
    return pcg64_words(gen)


def engine_for(mdp, n_trees, n_actions, episodes, horizon, gamma, temperature, prior="random_available",
               rollout="random_available", capacity=None):
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    from rl_agents_b200.engine.mcts import MCTSEngine
    return MCTSEngine(_lib.ENV_FINITE, n_trees, n_actions, episodes, horizon, gamma, temperature, mdp=mdp,
                      prior_policy=MCTSAgent.policy_factory(prior) if isinstance(prior, dict) else prior,
                      rollout_policy=MCTSAgent.policy_factory(rollout) if isinstance(rollout, dict) else rollout,
                      capacity=capacity)


def oracle_plan(env, episodes, horizon, gamma, temperature, rng, prior=None, rollout=None, tree=None):
    return planners.mcts_plan(env, episodes, horizon, gamma, temperature, rng, prior_policy=prior,
                              rollout_policy=rollout, tree=tree)


def assert_tree_equals_oracle(d, t):
    for f in ("parent", "action", "count"):
        assert d[f].astype(int).tolist() == [int(x) for x in getattr(t, f)], f
    for f in ("value", "prior"):
        assert d[f].tobytes() == np.array(getattr(t, f), dtype=np.float64).tobytes(), f


@pytest.mark.parametrize("section,key", [("cases", k) for k in sorted(G["cases"])] +
                         [("closed_loop", k) for k in sorted(G["closed_loop"])])
def test_kernel_matches_reference_golden(section, key):
    """One tree per golden: the device tree hashes to the reference's (closed loop: its action-node projection)."""
    g = G[section][key]
    env = live_env(case_of(g))
    cfg = g["config"]
    eng = engine_for(env.mdp, 1, env.action_space.n, g["episodes"], g["horizon"], g["gamma"], g["temperature"],
                     policy(cfg, "prior_policy"), policy(cfg, "rollout_policy"))
    assert eng.sampled
    eng.plan(roots([env]), words(planner_rng(g["seed"]))[None], None, words(env.np_random))
    plans, res, w = eng.finish()
    assert plans[0] == g.get("plan", g.get("plan_actions")) and rng_words_state(w[0]) == g["rng_state"]
    assert (int(res[0, 3]), int(res[0, 4])) == (0, -1)
    assert tree_digest(eng.tree_dict(0)) == g["tree"]


@pytest.mark.parametrize("section,key", [("cases", "garnet50_b300_g0.8_preference"),
                                         ("cases", "garnet30_b2_b400_g0.8_advanced_env")] +
                         [("closed_loop", k) for k in sorted(G["closed_loop"])])
def test_agent_matches_reference_golden(section, key):
    """MCTSAgent on the product env hands the device its env generator and leaves that generator unchanged."""
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    g = G[section][key]
    env = live_env(case_of(g), product=True)
    agent = MCTSAgent(env, copy.deepcopy(g["config"]))
    agent.seed(g["seed"])
    before = rng_state(env.np_random)
    assert before == g["env_rng_state"]
    plan = agent.plan(int(env.mdp.state))
    assert rng_state(env.np_random) == before
    assert plan == g.get("plan", g.get("plan_actions"))
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    assert tree_digest(agent.planner.last_tree.tree_dict(0)) == g["tree"]


@pytest.mark.parametrize("key", sorted(G["subtree"]))
def test_agent_subtree_matches_reference_golden(key):
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    g = G["subtree"][key]
    env = live_env(case_of(g), product=True)
    agent = MCTSAgent(env, copy.deepcopy(g["config"]))
    agent.seed(g["seed"])
    for k, d in enumerate(g["decisions"]):
        assert (int(env.mdp.state), rng_state(env.np_random)) == (d["state"], d["env_rng_state"])
        plan = agent.plan(int(env.mdp.state))
        assert rng_state(env.np_random) == d["env_rng_state"]
        assert plan == d["plan"] and rng_state(agent.planner.np_random) == d["rng_state"], k
        t = agent.planner.last_tree.tree_dict(0)
        assert canonical_digest(t["first_child"], t["n_children"], t["action"], t["count"], t["value"],
                                t["prior"]) == d["tree"], k
        if k == 0:
            assert agent.planner._resume == 0
        env.step(plan[0])


@pytest.mark.parametrize("prior,rollout", [("random_available", "random_available"), ("random", "random"),
                                           (PREF_PRIOR, PREF_ROLLOUT)], ids=["random_available", "random", "pref"])
def test_batch_of_256_mixed_trees_equals_the_oracle(prior, rollout):
    """One "sparse" table with stochastic, sparse and deterministic rows; every tree its own root, planner stream and
    env generator."""
    make, off = mixed_finite_mdp()
    starts = [off[0], off[0] + 7, off[1], off[1] + 5, off[2], off[2] + 37, off[3], off[3] + 2]
    envs_ = [make(starts[i % len(starts)]) for i in range(256)]
    for i, e in enumerate(envs_):
        e.seed(5000 + i)
    episodes, horizon, gamma, temperature = 60, 6, 0.8, 10.0
    eng = engine_for(envs_[0].mdp, 256, 3, episodes, horizon, gamma, temperature, prior, rollout)
    eng.plan(roots(envs_), np.stack([words(planner_rng(i)) for i in range(256)]), None,
             np.stack([words(e.np_random) for e in envs_]))
    plans, res, w = eng.finish()
    pol = lambda p: p if isinstance(p, dict) else {"type": p}
    for i, env in enumerate(envs_):
        rng = planner_rng(i)
        plan, t = oracle_plan(env, episodes, horizon, gamma, temperature, rng, pol(prior), pol(rollout))
        assert plans[i] == plan and rng_words_state(w[i]) == rng_state(rng), i
        assert (int(res[i, 0]), int(res[i, 3]), int(res[i, 4])) == (len(t.parent), 0, -1), i
        assert_tree_equals_oracle(eng.tree_dict(i), t)
    assert len(set(res[:, 0].tolist())) > 3


def test_deterministic_tables_through_the_sampled_path_are_bit_identical():
    """A deterministic MDP through b2_mcts_plan_sampled with no env draws against b2_mcts_plan."""
    from oracle import envs as oenvs
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.tables import SampledFiniteTables
    T, R = oenvs.garnet(50, 4, 3, seed=0, deterministic=True)
    term = np.zeros(50, bool)
    term[::7] = True
    envs_ = [oenvs.FiniteMDPLite(T, R, term, state=i % 50) for i in range(70)]
    rng_words = np.stack([words(planner_rng(i)) for i in range(70)])
    for prior, rollout in (("random_available", "random_available"), (PREF_PRIOR, PREF_ROLLOUT)):
        ref = engine_for(envs_[0].mdp, 70, 4, 80, 7, 0.85, 6.0, prior, rollout)
        assert not ref.sampled
        ref.plan(roots(envs_), rng_words)
        ref_plans, ref_res, ref_words = ref.finish()
        eng = engine_for(envs_[0].mdp, 70, 4, 80, 7, 0.85, 6.0, prior, rollout)
        tables = SampledFiniteTables(envs_[0].mdp, eng.device)
        assert tables.env_draws == 0
        env_rng = eng.torch.as_tensor(np.stack([words(planner_rng(99))] * 70).view(np.int64), device=eng.device)
        eng._load_rng(rng_words)
        _lib.check(eng.lib.b2_mcts_plan_sampled(eng.cfg, tables.struct(), _lib.ptr(tables.terminal), 0,
                                                _lib.ptr(env_rng), _lib.ptr(roots(envs_)), eng.tree, _lib.ptr(eng.rng),
                                                _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), _lib.current_stream()))
        plans, res, w = eng.finish()
        assert plans == ref_plans and (w == ref_words).all()
        assert (res[:, :3] == ref_res[:, :3]).all() and (res[:, 3] == 0).all() and (res[:, 4] == -1).all()
        for i in range(70):
            a, b = eng.tree_dict(i), ref.tree_dict(i)
            for f in a:
                assert np.asarray(a[f]).tobytes() == np.asarray(b[f]).tobytes(), (i, f)


def test_golden_error_raises_numpys_message_and_stops_its_own_tree_only():
    """bad20: the NaN row (0, 1) is reached from some roots and not from others within the budget; the trees that
    reach it report that row, the others equal the oracle's, and finish() raises numpy's own message."""
    g = G["errors"]["bad20_reached_nan_row"]
    c = G["cases"]["unreached_bad20_b300_g0.8"]
    envs_ = [oracle_env("bad20", s) for s in range(19)]
    for i, e in enumerate(envs_):
        e.seed(g["env_seed"] + i)
    episodes, horizon = 12, 3
    eng = engine_for(envs_[0].mdp, len(envs_), 3, episodes, horizon, c["gamma"], c["temperature"])
    eng.plan(roots(envs_), np.stack([words(planner_rng(g["seed"] + i)) for i in range(len(envs_))]), None,
             np.stack([words(e.np_random) for e in envs_]))
    res = eng._result()
    failed = 0
    for i, env in enumerate(envs_):
        try:
            plan, t = oracle_plan(env, episodes, horizon, c["gamma"], c["temperature"], planner_rng(g["seed"] + i))
        except ValueError as e:
            assert str(e) == g["message"]
            assert (int(res[i, 3]), int(res[i, 4])) == (1, 0 * 3 + 1), i
            failed += 1
            continue
        assert (int(res[i, 3]), int(res[i, 4])) == (0, -1), i
        assert eng.plan_buf[i, :int(res[i, 1])].cpu().numpy().tolist() == plan, i
        assert_tree_equals_oracle(eng.tree_dict(i), t)
    assert 0 < failed < len(envs_)
    with pytest.raises(ValueError) as e:
        eng.finish()
    assert str(e.value) == g["message"]


def test_golden_error_through_the_agent():
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    g = G["errors"]["bad20_reached_nan_row"]
    env = live_env(case_of(g), product=True)
    agent = MCTSAgent(env, copy.deepcopy(g["config"]))
    agent.seed(g["seed"])
    with pytest.raises(ValueError) as e:
        agent.plan(int(env.mdp.state))
    assert str(e.value) == g["message"]


def test_root_parallel_replicas_equal_the_oracle():
    """root_parallel: R trees on streams spawned from the planner's, each replica's env copies starting from the
    same live env generator."""
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    R = 4
    env = product_env("garnet50", 9)
    env.seed(77)
    agent = MCTSAgent(env, {"budget": 600, "gamma": 0.8, "root_parallel": R})
    agent.seed(31)
    before = rng_state(env.np_random)
    agent.plan(9)
    assert rng_state(env.np_random) == before
    cfg = agent.planner.config
    per = -(-int(cfg["episodes"]) // R)
    gens = planner_rng(31).spawn(R)
    eng = agent.planner.last_tree
    for t in range(R):
        oenv = oracle_env("garnet50", 9)
        oenv.seed(77)
        _, tree = oracle_plan(oenv, per, cfg["horizon"], cfg["gamma"], cfg["temperature"], gens[t])
        assert_tree_equals_oracle(eng.tree_dict(t), tree)


def test_agent_loop_of_ten_decisions_equals_the_oracle():
    """Ten decisions of MCTSAgent on a "stochastic" FiniteMDPEnv, the env stepped between them: each decision equals
    the oracle's on the same state and env generator, and plan() leaves the generator unchanged."""
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    env = product_env("dense6", 0)
    env.seed(4)
    agent = MCTSAgent(env, {"budget": 200, "gamma": 0.8})
    agent.seed(21)
    cfg = agent.planner.config
    rng = planner_rng(21)
    for step in range(10):
        s = int(env.mdp.state)
        oenv = oracle_env("dense6", s)
        oenv.np_random = copy.deepcopy(env.np_random)
        expected, _ = oracle_plan(oenv, cfg["episodes"], cfg["horizon"], cfg["gamma"], cfg["temperature"], rng)
        before = rng_state(env.np_random)
        assert agent.plan(s) == expected, step
        assert rng_state(env.np_random) == before and rng_state(agent.planner.np_random) == rng_state(rng), step
        env.step(expected[0])


def wave_engine(env, episodes, horizon, width):
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import MCTSWaveEngine
    return MCTSWaveEngine(_lib.ENV_FINITE, env.action_space.n, episodes, horizon, 0.8, 10.0, width, mdp=env.mdp)


@pytest.mark.parametrize("mdp,state", [("dense6", 1), ("garnet50", 4), ("term40", 1)])
@pytest.mark.parametrize("width", [1, 64, 1024])
def test_wavefront_equals_its_specification(mdp, state, width):
    episodes, horizon, seed = 300, 8, 12345
    env = oracle_env(mdp, state)
    env.seed(900 + width)
    eng = wave_engine(env, episodes, horizon, width)
    assert eng.sampled and (width <= episodes or eng.width > episodes)
    eng.plan(roots([env]), seed, words(env.np_random))
    plan, res = eng.finish()
    before = rng_state(env.np_random)
    ref_plan, t = planners.mcts_plan_wavefront(env, episodes, horizon, 0.8, 10.0, width, seed)
    assert rng_state(env.np_random) == before
    d = eng.tree_dict()
    assert plan == ref_plan
    assert d["parent"].tolist() == t.parent and d["count"].tolist() == t.count and d["vsum"].tolist() == t.vsum
    assert int(res[2]) == t.env_steps
    assert eng.rejected.cpu().numpy().tolist() == [-1, -1]


@pytest.mark.parametrize("width", [1, 8, 1024])
def test_wavefront_reports_the_first_rejected_row(width):
    """bad20: the lowest episode that reaches the NaN row is the one the specification raises on -- it plans the
    episodes before it and raises with that episode included."""
    episodes, horizon, seed = 64, 5, 7
    env = oracle_env("bad20", 2)
    env.seed(3)
    eng = wave_engine(env, episodes, horizon, width)
    eng.plan(roots([env]), seed, words(env.np_random))
    episode, row = eng.rejected.cpu().numpy().tolist()
    assert 0 <= episode < episodes and np.isnan(MDPS["bad20"]["transition"][row // 3, row % 3]).all()
    with pytest.raises(ValueError) as e:
        eng.finish()
    with pytest.raises(ValueError) as e2:
        planners.mcts_plan_wavefront(copy.deepcopy(env), episode + 1, horizon, 0.8, 10.0, width, seed)
    assert str(e.value) == str(e2.value)
    planners.mcts_plan_wavefront(copy.deepcopy(env), episode, horizon, 0.8, 10.0, width, seed)


def per_tree_call(eng, env):
    from rl_agents_b200 import _lib
    root = roots([env, env])
    env_rng = eng.torch.as_tensor(np.stack([words(env.np_random)] * 2).view(np.int64), device=eng.device)
    eng._load_rng(np.stack([words(planner_rng(i)) for i in range(2)]))

    def call(cfg=None, mdp=None, terminal=None, env_draws=1, env_rng_ptr=None):
        return eng.lib.b2_mcts_plan_sampled(
            cfg if cfg is not None else eng.cfg, mdp if mdp is not None else eng.tables.struct(),
            terminal, env_draws, _lib.ptr(env_rng) if env_rng_ptr is None else env_rng_ptr, _lib.ptr(root), eng.tree,
            _lib.ptr(eng.rng), _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), _lib.current_stream())
    return call, [eng.result]


def wave_call(eng, env):
    from rl_agents_b200 import _lib
    root = roots([env])
    env_rng = eng.torch.as_tensor(words(env.np_random).view(np.int64), device=eng.device)

    def call(cfg=None, mdp=None, terminal=None, env_draws=1, env_rng_ptr=None):
        return eng.lib.b2_mcts_plan_wave_sampled(
            cfg if cfg is not None else eng.cfg, mdp if mdp is not None else eng.tables.struct(),
            terminal, env_draws, _lib.ptr(env_rng) if env_rng_ptr is None else env_rng_ptr, _lib.ptr(root), eng.tree,
            _lib.ptr(eng.workspace), _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), _lib.ptr(eng.rejected),
            _lib.current_stream())
    return call, [eng.result, eng.rejected]


@pytest.mark.parametrize("entry", ["per_tree", "wavefront"])
def test_refusals_launch_no_kernel(entry):
    import torch
    from rl_agents_b200 import _lib
    env = oracle_env("garnet50")
    env.seed(0)
    if entry == "per_tree":
        eng = engine_for(env.mdp, 2, 4, 10, 4, 0.8, 10.0)
        call, outputs = per_tree_call(eng, env)
    else:
        eng = wave_engine(env, 10, 4, 4)
        call, outputs = wave_call(eng, env)
    terminal = eng.tables.terminal.data_ptr()
    good = eng.tables.struct()

    def fill():
        for o in outputs:
            o.fill_(UNWRITTEN)

    fill()
    assert call(terminal=terminal) == 0
    torch.cuda.synchronize()
    assert (eng.result != UNWRITTEN).any()                  # the accepted call launched and wrote its results

    def refused(match=None, **kw):
        fill()
        rc = call(**kw)
        torch.cuda.synchronize()
        assert rc == 1, (kw, rc)                            # B2_ERR_INVALID
        if match is not None:
            assert match in eng.lib.b2_last_error().decode(), kw
        for o in outputs:
            assert (o == UNWRITTEN).all(), kw               # no kernel ran

    for field, value, match in FAULTS:
        m, t = eng.tables.struct(), terminal
        if field == "terminal":
            t = None
        else:
            setattr(m, field, good.n_actions + 1 if value == "mismatch" else value)
        refused(match, mdp=m, terminal=t)
    refused("null pointer", terminal=terminal, env_rng_ptr=0)
    refused("env_draws", terminal=terminal, env_draws=2)
    refused("env_draws", terminal=terminal, env_draws=-1)
    c = type(eng.cfg).from_buffer_copy(eng.cfg)
    c.env_kind = _lib.ENV_HIGHWAY
    refused("env_kind", cfg=c, terminal=terminal)
    c = type(eng.cfg).from_buffer_copy(eng.cfg)
    c.n_actions = 9
    refused("n_actions", cfg=c, terminal=terminal)
