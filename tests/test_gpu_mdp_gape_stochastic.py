"""GPU tests of MDP-GapE on stochastic finite MDPs (b2_mdp_gape_plan_sampled, csrc/mdp_gape.cu): the kernel against
the reference's goldens (tests/golden/golden_mdp_gape_stochastic.json) and against the oracle restatement
(oracle/mdp_gape_stochastic.py) on batches in both sampled modes, the deterministic tables through the sampled path,
the error paths and the agent.

Structure, child orders, keys, plans, episodes run and the RNG stream position are exact; the bounds agree within 1e-9
(CUDA's fp64 log / exp against the host's, as for the deterministic MDP-GapE).  Where an exact host tie of value_upper
is one ulp apart on the device, the search is compared exactly up to the episode before the tie decides a selection
(TIE_DIVERGENCE, DESIGN §4.2a)."""
import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import mdp_gape as gape
from oracle import mdp_gape_stochastic as sgape
from oracle import ref_loader
from tests.mdp_gape_stochastic_cases import MDPS, oracle_env, product_env
from tests.test_gpu_mdp_gape import assert_golden_tree, engine_for, pcg64_of, roots, words_state
from tests.test_mdp_gape_oracle import completed_planner_config, rng_state
from tests.util import load_golden

pytestmark = pytest.mark.gpu
G = load_golden("golden_mdp_gape_stochastic.json")
TOL = 1e-9


def assert_device_tree(d, t):
    """Device tree `d` (engine.tree_dict) against an oracle tree `t` (oracle.mdp_gape_stochastic.mdp_gape_plan)."""
    n = len(t.parent)
    assert len(d["parent"]) == n
    for f in ("parent", "action", "kind", "count", "done", "key"):
        assert d[f].astype(int).tolist() == [int(x) for x in getattr(t, f)], f
    assert d["order"] == {int(c): [int(x) for x in o] for c, o in t.order.items()}
    for f in gape.FLOAT_FIELDS:
        ref = np.array([np.nan if x is None else float(x) for x in getattr(t, f)])
        has = ~np.isnan(ref)
        np.testing.assert_allclose(d[f][has], ref[has], rtol=0, atol=TOL, err_msg=f)


def oracle_run(env, cfg, seed):
    rng = ref_loader.legacy_np_random(seed)[0]
    plan, t, episodes_run = sgape.mdp_gape_plan(oenvs.LegacyStepEnv(env), cfg, rng)
    return plan, t, episodes_run, rng


def run_batch_against_oracle(envs_, cfg, seeds):
    eng = engine_for(envs_[0], cfg, len(envs_))
    assert eng.sampled
    eng.plan(roots(envs_), pcg64_of(seeds))
    plans, res, words = eng.finish()
    for i, (env, s) in enumerate(zip(envs_, seeds)):
        plan, t, episodes_run, rng = oracle_run(env, cfg, s)
        assert (plans[i], int(res[i, 1]), words_state(words[i])) == (plan, episodes_run, rng_state(rng)), i
        assert (int(res[i, 4]), int(res[i, 5]), int(res[i, 6])) == (t.best, t.challenger, -1), i
        assert_device_tree(eng.tree_dict(i), t)
    return eng, res


def run_capped_against_oracle(env, cfg, seed, last_episode):
    """One tree stopped after episode `last_episode` (the config's episodes and thresholds unchanged) against the
    oracle stopped there: structure, keys, child orders, RNG words and episodes exact, floats within TOL."""
    eng = engine_for(env, cfg, 1)
    eng.cfg.episodes = last_episode - 1                 # the stopping rule ends the loop after episode last_episode
    eng.plan(roots([env]), pcg64_of([seed]))
    _, res, words = eng.finish()
    rng = ref_loader.legacy_np_random(seed)[0]
    _, t, episodes_run = sgape.mdp_gape_plan(oenvs.LegacyStepEnv(env), cfg, rng, last_episode=last_episode)
    assert (int(res[0, 1]), words_state(words[0])) == (episodes_run, rng_state(rng))
    d = eng.tree_dict(0)
    assert_device_tree(d, t)
    return d, t, res


# Decisions on which an exact tie of value_upper on the host is one ulp apart on the device (DESIGN §4.2a): the
# episode after which the tie decides a selection; up to it the kernel equals the oracle exactly.
TIE_DIVERGENCE = {"term40_K3_hfa_acc1": 5}


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_kernel_matches_reference_golden(key):
    g = G["cases"][key]
    cfg = completed_planner_config(g["config"])
    env = oracle_env(g["mdp"], g["state"])
    if key in TIE_DIVERGENCE:
        run_capped_against_oracle(env, cfg, g["seed"], TIE_DIVERGENCE[key])
        eng = engine_for(env, cfg, 1)
        eng.plan(roots([env]), pcg64_of([g["seed"]]))
        plans, res, _ = eng.finish()
        assert plans[0] == g["plan"] and int(res[0, 1]) == g["episodes_run"]
        return
    eng, res = run_batch_against_oracle([env], cfg, [g["seed"]])
    assert (eng.episodes, eng.horizon) == (g["episodes"], g["horizon"])
    assert [int(res[0, 3])] == g["plan"] and int(res[0, 1]) == g["episodes_run"]
    assert (int(res[0, 4]) - 1, int(res[0, 5]) - 1) == (g["best_index"], g["challenger_index"])
    assert_golden_tree(eng.tree_dict(0), g["tree"])


def test_host_tie_that_the_device_breaks_by_one_ulp():
    """term40_K3_hfa_acc1 after episode 5: root chance nodes 1 and 3 have bit-equal value_upper on the host, so UGapE's
    challenger is the first of them; node 3's backup (p_hat = (0.5, 0.5) over two equal values, one unobserved
    placeholder) computes theta(f*) = q_p @ log(d) + log(q_p @ (1 / d)) - c, whose first two terms cancel exactly with
    glibc's log and leave a residue with CUDA's, and the device's node 3 ends one ulp above node 1."""
    g = G["cases"]["term40_K3_hfa_acc1"]
    d, t, _ = run_capped_against_oracle(oracle_env(g["mdp"], g["state"]), completed_planner_config(g["config"]),
                                        g["seed"], TIE_DIVERGENCE["term40_K3_hfa_acc1"])
    assert t.upper[1] == t.upper[3]
    assert d["upper"][1] == t.upper[1] and d["upper"][3] == np.nextafter(t.upper[3], np.inf)
    assert [t.count[c] for c in t.order[3]] == [0, 1, 1]


@pytest.mark.parametrize("mdp,K,n_trees,budget", [
    ("garnet50", 3, 256, 100),           # sparse, K = B
    ("garnet30_b2", 2, 37, 200),         # sparse, K = B = 2
    ("garnet50", 8, 33, 150),            # sparse, K > B
    ("dense6", 8, 65, 150),              # stochastic, K > S
    ("dense6", 15, 31, 120),             # stochastic, the longest fma chains the host computes in order
    ("term40", 15, 17, 120),
])
def test_batches_equal_the_oracle(mdp, K, n_trees, budget):
    cfg = completed_planner_config({"budget": budget, "gamma": 0.8, "max_next_states_count": K,
                                    "continuation_type": "uniform" if n_trees % 2 else "zeros"})
    S = MDPS[mdp]["reward"].shape[0]
    envs_ = [oracle_env(mdp, state=i % S) for i in range(n_trees)]
    run_batch_against_oracle(envs_, cfg, [100 + i for i in range(n_trees)])


def test_batch_with_mixed_stopping_points_equals_the_oracle():
    cfg = completed_planner_config({"budget": 600, "gamma": 0.7, "accuracy": 3.0, "max_next_states_count": 3})
    _, res = run_batch_against_oracle([oracle_env("garnet50", state=3 * i) for i in range(15)], cfg, list(range(15)))
    assert len(set(res[:, 1].tolist())) > 2 and res[:, 1].min() < gape.mdp_gape_allocation(cfg, 4)[0] + 2


def test_one_decision_at_budget_5000_equals_the_oracle():
    """Exact through episode 166; in episode 167 a host tie of value_upper two levels down is one ulp apart on the
    device (DESIGN §4.2a), and from there only the plan and the episodes run are compared."""
    cfg = completed_planner_config({"budget": 5000, "gamma": 0.8, "max_next_states_count": 3})
    env = oracle_env("garnet50", 0)
    run_capped_against_oracle(env, cfg, 0, 166)
    eng = engine_for(env, cfg, 1)
    eng.plan(roots([env]), pcg64_of([0]))
    plans, res, _ = eng.finish()
    plan, _, episodes_run, _ = oracle_run(env, cfg, 0)
    assert plans[0] == plan and int(res[0, 1]) == episodes_run


def test_deterministic_tables_through_the_sampled_path_match_the_existing_path():
    """A deterministic MDP through b2_mdp_gape_plan_sampled (no env draws) against b2_mdp_gape_plan: structure, plans
    and RNG words exact, floats within 1e-9 (the sampled backup's final sum is an fma chain, the existing one is
    not)."""
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.tables import SampledFiniteTables
    T, R = oenvs.garnet(50, 4, 3, seed=0, deterministic=True)
    term = np.zeros(50, bool)
    term[::7] = True
    envs_ = [oenvs.FiniteMDPLite(T, R, term, state=i % 50) for i in range(40)]
    cfg = completed_planner_config({"budget": 400, "gamma": 0.8, "max_next_states_count": 3})
    seeds = list(range(40))
    ref = engine_for(envs_[0], cfg, 40)
    assert not ref.sampled
    ref.plan(roots(envs_), pcg64_of(seeds))
    ref_plans, ref_res, ref_words = ref.finish()
    eng = engine_for(envs_[0], cfg, 40)
    tables = SampledFiniteTables(envs_[0].mdp, eng.device)
    terminal = torch.as_tensor(term.astype(np.uint8), device=eng.device)
    keys = torch.empty((40, eng.capacity), dtype=torch.int32, device=eng.device)
    root_states = roots(envs_)
    eng._load_rng(pcg64_of(seeds))
    _lib.check(eng.lib.b2_mdp_gape_plan_sampled(eng.cfg, tables.struct(), _lib.ptr(terminal), 0,
                                                _lib.ptr(root_states), eng.tree, _lib.ptr(keys), _lib.ptr(eng.rng),
                                                _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), _lib.current_stream()))
    plans, res, words = eng.finish()
    assert plans == ref_plans and (words == ref_words).all()
    assert (res[:, :6] == ref_res[:, :6]).all() and (res[:, 6] == -1).all()
    for i in range(40):
        a, b = eng.tree_dict(i), ref.tree_dict(i)
        for f in ("parent", "first_child", "count", "meta"):
            assert (a[f] == b[f]).all(), (i, f)
        for f in ("upper", "lower", "mu_ucb", "mu_lcb", "cumulative"):
            np.testing.assert_allclose(a[f], b[f], rtol=0, atol=TOL, err_msg=f)
        assert a["order"] == b["order"]
        k = keys[i, :len(a["parent"])].cpu().numpy()
        observed = k >= 0
        assert (a["kind"][observed] == 0).all() and (a["action"][observed] == 0).all()


def isolated_error_env(kind, state):
    """unreached_bad20 (state 19 unreachable from the others) with one error planted at state 19: a NaN row, rewards
    outside [0, 1], or three successors per row where every other state has one (K = 1 overflows at 19 only)."""
    m = MDPS["unreached_bad20"]
    p, nxt, r = m["transition"].copy(), m["next"].copy(), m["reward"].copy()
    p[19, 0] = p[18, 0]
    if kind == 4:
        p[19, 1] = np.nan
    elif kind == 1:
        r[19] = 1.5
    else:
        nxt[:19] = nxt[:19, :, :1]
    return oenvs.FiniteMDPLite(p, r, m["terminal"], mode="sparse", nxt=nxt, state=state)


@pytest.mark.parametrize("key", sorted(G["errors"]))
def test_golden_errors_raise_as_the_reference(key):
    g = G["errors"][key]
    eng = engine_for(oracle_env(g["mdp"], g["state"]), completed_planner_config(g["config"]), 1)
    eng.plan(roots([oracle_env(g["mdp"], g["state"])]), pcg64_of([g["seed"]]))
    res = eng._result()
    assert int(res[0, 2]) == {"garnet50_K1_placeholders": 3, "bad20_reached_nan_row": 4, "wide20_rewards": 1}[key]
    assert int(res[0, 3]) == -1
    with pytest.raises(ValueError) as e:
        eng.finish()
    assert str(e.value) == g["message"]


@pytest.mark.parametrize("code", [1, 3, 4])
def test_an_error_stops_its_own_tree_only(code):
    """Trees rooted at state 19 meet the planted error; the others of the same launch equal the oracle's."""
    cfg = completed_planner_config({"budget": 200, "gamma": 0.8, "max_next_states_count": 1 if code == 3 else 3})
    states = [19, 0, 5, 19, 11, 18, 3]
    envs_ = [isolated_error_env(code, s) for s in states]
    seeds = [300 + i for i in range(len(states))]
    eng = engine_for(envs_[0], cfg, len(envs_))
    eng.plan(roots(envs_), pcg64_of(seeds))
    res = eng._result()
    for i, (env, s) in enumerate(zip(envs_, seeds)):
        if states[i] == 19:
            with pytest.raises(ValueError):
                oracle_run(env, cfg, s)
            assert (int(res[i, 2]), int(res[i, 3])) == (code, -1), i
            assert int(res[i, 6]) == (19 * 3 + 1 if code == 4 else -1), i
            continue
        plan, t, episodes_run, rng = oracle_run(env, cfg, s)
        assert int(res[i, 2]) == 0 and [int(res[i, 3])] == plan and int(res[i, 1]) == episodes_run, i
        assert_device_tree(eng.tree_dict(i), t)
    with pytest.raises(ValueError):
        eng.finish()


def test_unreached_bad_row_is_fine_and_the_c_abi_refuses_other_env_kinds():
    from rl_agents_b200 import _lib
    g = G["cases"]["unreached_bad20_K3_b300"]
    assert np.isnan(MDPS["unreached_bad20"]["transition"][19, 0]).all()
    env = oracle_env("unreached_bad20")
    eng = engine_for(env, completed_planner_config(g["config"]), 1)
    eng.plan(roots([env]), pcg64_of([g["seed"]]))
    assert eng.finish()[0] == [g["plan"]]
    eng.cfg.env_kind = _lib.ENV_HIGHWAY
    with pytest.raises(_lib.B2Error, match="env_kind"):
        eng.plan(roots([env]), pcg64_of([0]))


def test_agent_from_shipped_config_matches_the_golden():
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapEAgent
    g = G["cases"]["garnet30_b2_mdp_gape_json"]
    # mdp-gape.json as shipped, with its `__class__` pointing at this package's agent
    shipped = dict(g["config"], __class__="<class 'rl_agents_b200.agents.tree_search.mdp_gape.MDPGapEAgent'>")
    agent = MDPGapEAgent(product_env(g["mdp"], g["state"]), shipped)
    agent.seed(g["seed"])
    assert agent.plan(g["state"]) == g["plan"]
    assert agent.planner.budget_used == g["budget_used"]
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    assert_golden_tree(agent.planner.last_tree.tree_dict(0), g["tree"])


def test_closed_loop_on_a_stochastic_env_equals_per_step_oracle_decisions():
    """Ten steps of MDPGapEAgent on a "stochastic" FiniteMDPEnv with receding_horizon 3: every decision equals the
    oracle's from the same state on a copy of the agent's generator."""
    import copy
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapEAgent
    config = {"budget": 300, "gamma": 0.8, "max_next_states_count": 6, "receding_horizon": 3}
    env = product_env("dense6", 0)
    env.seed(4)
    agent = MDPGapEAgent(env, dict(config))
    agent.seed(21)
    cfg = completed_planner_config({k: v for k, v in config.items() if k != "receding_horizon"})
    for step in range(10):
        s = int(env.mdp.state)
        rng = ref_loader.legacy_np_random(0)[0]                 # the reference's randint API on the agent's stream
        rng.bit_generator.state = copy.deepcopy(agent.planner.np_random.bit_generator.state)
        plan, t, episodes_run = sgape.mdp_gape_plan(oenvs.LegacyStepEnv(oracle_env("dense6", s)), cfg, rng)
        assert agent.act(s) == plan[0], step
        assert agent.planner.budget_used == episodes_run * t.horizon, step
        assert rng_state(agent.planner.np_random) == rng_state(rng), step
        env.step(plan[0])
