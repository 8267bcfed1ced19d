"""GPU tests of OLOP / KL-OLOP on stochastic finite MDPs (b2_olop_plan_sampled, csrc/olop.cu): the kernel against the
reference's goldens (tests/golden/golden_olop_stochastic.json) and against the oracle (oracle/planners.py::olop_plan)
on batches of 256 trees in both sampled modes, the deterministic tables through the sampled path, the error paths,
the agents from the shipped configs and a closed loop.

Structure, counts, done bits, cumulative rewards, plans and the RNG stream position are exact; mu_ucb and value_upper
agree within the tolerance of test_gpu_engines.py::test_olop_finite_golden (rtol 1e-9: the KL bound's Newton solve
uses CUDA's fp64 log, which is not the host's)."""
import copy

import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import ref_loader
from tests.mdp_gape_stochastic_cases import MDPS, oracle_env, product_env
from tests.test_gpu_mdp_gape import pcg64_of, roots, words_state
from tests.test_mdp_gape_oracle import rng_state
from tests.test_olop_stochastic_oracle import completed_config, oracle_run, oracle_tree_dict
from tests.olop_stochastic_tree import tree_digest
from tests.util import load_golden

pytestmark = pytest.mark.gpu
G = load_golden("golden_olop_stochastic.json")
RTOL, ATOL = 1e-9, 1e-12
KL = {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)"}
KL_LOCAL = {"type": "kullback-leibler", "time": "local", "threshold": "1*np.log(time)"}
HOEFFDING = {"type": "hoeffding", "time": "global", "threshold": "4*np.log(time)"}


def engine_for(env, cfg, n_trees):
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mcts import allocation
    from rl_agents_b200.engine.olop import OLOPEngine
    n_actions = env.action_space.n
    episodes, horizon = allocation(max(n_actions, cfg["budget"]), cfg["gamma"])
    return OLOPEngine(_lib.ENV_FINITE, n_trees, n_actions, episodes, horizon, cfg["gamma"], cfg["upper_bound"],
                      cfg["continuation_type"], mdp=env.mdp)


def assert_device_tree(d, t):
    """Device tree `d` (OLOPEngine.tree_dict) against an oracle tree `t`: integers, done bits and cumulative rewards
    exact, mu_ucb and upper within RTOL (inf equal to inf)."""
    o = oracle_tree_dict(t)
    for f in ("parent", "action", "count"):
        assert d[f].astype(int).tolist() == [int(x) for x in o[f]], f
    assert d["done"].tolist() == [bool(x) for x in o["done"]]
    assert np.array_equal(d["cumulative_reward"], np.array(o["cumulative_reward"], dtype=np.float64))
    for f in ("mu_ucb", "upper"):
        np.testing.assert_allclose(d[f], np.array(o[f], dtype=np.float64), rtol=RTOL, atol=ATOL, err_msg=f)


def assert_golden_tree(d, g):
    """Device tree `d` against a golden digest: the exact fields' SHA-256 equal, the bounds' sums within RTOL."""
    dg = tree_digest(d)
    assert (dg["n_nodes"], dg["exact_sha256"]) == (g["n_nodes"], g["exact_sha256"])
    for f in ("sum_mu_ucb", "sum_upper"):
        np.testing.assert_allclose(dg[f], g[f], rtol=RTOL, err_msg=f)


def run_batch_against_oracle(envs_, cfg, seeds):
    eng = engine_for(envs_[0], cfg, len(envs_))
    assert eng.sampled
    eng.plan(roots(envs_), pcg64_of(seeds))
    plans, res, words = eng.finish()
    for i, (env, s) in enumerate(zip(envs_, seeds)):
        plan, t, rng = oracle_run(env, cfg, s)
        assert (plans[i], words_state(words[i])) == (plan, rng_state(rng)), i
        assert (int(res[i, 2]), int(res[i, 3])) == (0, -1), i
        assert_device_tree(eng.tree_dict(i), t)
    return eng, res


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_kernel_matches_reference_golden(key):
    g = G["cases"][key]
    cfg = completed_config(g["config"])
    env = oracle_env(g["mdp"], g["state"])
    eng = engine_for(env, cfg, 1)
    assert (eng.episodes, eng.horizon) == (g["episodes"], g["horizon"])
    eng.plan(roots([env]), pcg64_of([g["seed"]]))
    plans, res, words = eng.finish()
    assert plans[0] == g["plan"] and words_state(words[0]) == g["rng_state"]
    d = eng.tree_dict(0)
    assert_golden_tree(d, g["tree"])
    # node by node against the oracle, whose tree hashes to the golden's bit for bit
    assert_device_tree(d, oracle_run(env, cfg, g["seed"])[1])


@pytest.mark.parametrize("mdp,continuation,bound,budget", [
    ("garnet50", "uniform", KL, 120),          # sparse
    ("garnet50", "zeros", HOEFFDING, 100),
    ("dense6", "zeros", KL_LOCAL, 120),        # stochastic
    ("dense6", "uniform", HOEFFDING, 100),
    ("term40", "uniform", KL_LOCAL, 100),
])
def test_batches_of_256_equal_the_oracle(mdp, continuation, bound, budget):
    cfg = completed_config({"budget": budget, "gamma": 0.8, "continuation_type": continuation, "upper_bound": bound})
    S = MDPS[mdp]["reward"].shape[0]
    envs_ = [oracle_env(mdp, state=(7 * i) % S) for i in range(256)]
    run_batch_against_oracle(envs_, cfg, [1000 + i for i in range(256)])


def test_deterministic_tables_through_the_sampled_path_are_bit_identical():
    """A deterministic MDP through b2_olop_plan_sampled with no env draws against b2_olop_plan: trees, floats
    included, plans and RNG words bit for bit."""
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.tables import SampledFiniteTables
    T, R = oenvs.garnet(50, 4, 3, seed=0, deterministic=True)
    term = np.zeros(50, bool)
    term[::7] = True
    envs_ = [oenvs.FiniteMDPLite(T, R, term, state=i % 50) for i in range(70)]
    seeds = list(range(70))
    for continuation, bound in (("uniform", KL), ("zeros", KL_LOCAL), ("uniform", HOEFFDING)):
        cfg = completed_config({"budget": 300, "gamma": 0.8, "continuation_type": continuation,
                                "upper_bound": bound})
        ref = engine_for(envs_[0], cfg, 70)
        assert not ref.sampled
        ref.plan(roots(envs_), pcg64_of(seeds))
        ref_plans, ref_res, ref_words = ref.finish()
        eng = engine_for(envs_[0], cfg, 70)
        tables = SampledFiniteTables(envs_[0].mdp, eng.device)
        terminal = torch.as_tensor(term.astype(np.uint8), device=eng.device)
        eng._load_rng(pcg64_of(seeds))
        _lib.check(eng.lib.b2_olop_plan_sampled(eng.cfg, tables.struct(), _lib.ptr(terminal), 0,
                                                _lib.ptr(roots(envs_)), eng.tree, _lib.ptr(eng.rng),
                                                _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), _lib.current_stream()))
        plans, res, words = eng.finish()
        assert plans == ref_plans and (words == ref_words).all()
        assert (res[:, :3] == ref_res[:, :3]).all() and (res[:, 3] == -1).all()
        for i in range(70):
            a, b = eng.tree_dict(i), ref.tree_dict(i)
            for f in a:
                assert np.asarray(a[f]).tobytes() == np.asarray(b[f]).tobytes(), (continuation, i, f)


def isolated_error_env(code, state):
    """unreached_bad20 (state 19 is unreachable from the others) with one error planted at state 19: a NaN row
    (code 3) or rewards outside [0, 1] (code 1)."""
    m = MDPS["unreached_bad20"]
    p, r = m["transition"].copy(), m["reward"].copy()
    p[19, 0] = p[18, 0]
    if code == 3:
        p[19, 1] = np.nan
    else:
        r[19] = 1.5
    return oenvs.FiniteMDPLite(p, r, m["terminal"], mode="sparse", nxt=m["next"], state=state)


@pytest.mark.parametrize("key", sorted(k for k, g in G["errors"].items() if g["error"] == "ValueError"))
def test_golden_errors_raise_as_the_reference(key):
    g = G["errors"][key]
    env = oracle_env(g["mdp"], g["state"])
    eng = engine_for(env, completed_config(g["config"]), 1)
    eng.plan(roots([env]), pcg64_of([g["seed"]]))
    res = eng._result()
    code = {"bad20_reached_nan_row": 3, "wide20_rewards": 1}[key]
    assert int(res[0, 2]) == code
    if code == 3:
        row = int(res[0, 3])
        assert row // 3 == 0 and np.isnan(MDPS["bad20"]["transition"][0, row % 3]).all()
    with pytest.raises(ValueError) as e:
        eng.finish()
    assert str(e.value) == g["message"]


@pytest.mark.parametrize("code", [1, 3])
def test_an_error_stops_its_own_tree_only(code):
    """Trees rooted at state 19 meet the planted error; the others of the same launch equal the oracle's."""
    cfg = completed_config({"budget": 200, "gamma": 0.8, "continuation_type": "uniform", "upper_bound": KL})
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
            assert int(res[i, 2]) == code, i
            assert int(res[i, 3]) == (19 * 3 + 1 if code == 3 else -1), i
            continue
        plan, t, _ = oracle_run(env, cfg, s)
        assert int(res[i, 2]) == 0 and int(res[i, 3]) == -1, i
        assert eng.plan_buf[i, :int(res[i, 1])].cpu().numpy().tolist() == plan, i
        assert_device_tree(eng.tree_dict(i), t)
    with pytest.raises(ValueError):
        eng.finish()


def test_unreached_bad_row_is_not_an_error():
    g = G["cases"]["unreached_bad20_b300_uniform"]
    assert np.isnan(MDPS["unreached_bad20"]["transition"][19, 0]).all()
    env = oracle_env("unreached_bad20")
    eng = engine_for(env, completed_config(g["config"]), 1)
    eng.plan(roots([env]), pcg64_of([g["seed"]]))
    plans, res, _ = eng.finish()
    assert plans == [g["plan"]] and (int(res[0, 2]), int(res[0, 3])) == (0, -1)


@pytest.mark.parametrize("key", sorted(k for k, g in G["cases"].items() if g["config_name"]))
def test_agent_from_shipped_config_matches_the_golden(key):
    from rl_agents_b200.agents.tree_search.olop import OLOPAgent
    g = G["cases"][key]
    # kl-olop.json as shipped, with its `__class__` pointing at this package's agent
    shipped = dict(g["config"], __class__="<class 'rl_agents_b200.agents.tree_search.olop.OLOPAgent'>")
    agent = OLOPAgent(product_env(g["mdp"], g["state"]), shipped)
    agent.seed(g["seed"])
    assert (agent.planner.config["episodes"], agent.planner.config["horizon"]) == (g["episodes"], g["horizon"])
    assert agent.plan(g["state"]) == g["plan"]
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    assert_golden_tree(agent.planner.last_tree.tree_dict(0), g["tree"])


def oracle_run_on(env, cfg, rng):
    """olop_plan on `env` with the generator `rng`, which it advances."""
    from oracle import planners
    plan, t = planners.olop_plan(oenvs.LegacyStepEnv(env), cfg["budget"], cfg["gamma"], rng,
                                 upper_bound=cfg["upper_bound"], continuation_type=cfg["continuation_type"])
    return plan, t, rng


def test_closed_loop_on_a_stochastic_env_equals_the_oracle_agent_loop():
    """Ten steps of OLOPAgent on a "stochastic" FiniteMDPEnv with receding_horizon 3, against the reference agent's
    loop (abstract.py:49-82) run with the oracle planner on the same generator: the same replanning steps, plans,
    actions and RNG position."""
    from rl_agents_b200.agents.tree_search.olop import OLOPAgent
    config = {"budget": 200, "gamma": 0.8, "continuation_type": "uniform", "upper_bound": KL, "receding_horizon": 3}
    env = product_env("dense6", 0)
    env.seed(4)
    agent = OLOPAgent(env, copy.deepcopy(config))
    agent.seed(21)
    cfg = completed_config({k: v for k, v in config.items() if k != "receding_horizon"})
    rng = ref_loader.legacy_np_random(21)[0]
    previous, remaining, replans = [], 0, 0
    for step in range(10):
        s = int(env.mdp.state)
        if remaining == 0 or len(previous) <= 1:
            remaining = config["receding_horizon"] - 1
            previous, _, rng = oracle_run_on(oracle_env("dense6", s), cfg, rng)
            replans += 1
        else:
            remaining -= 1
            previous = previous[1:]
        assert agent.plan(s) == previous, step
        assert rng_state(agent.planner.np_random) == rng_state(rng), step
        env.step(previous[0])
    assert 3 <= replans < 10



def test_c_abi_refusals():
    import torch
    from rl_agents_b200 import _lib
    env = oracle_env("garnet50")
    cfg = completed_config({"budget": 100, "gamma": 0.8, "continuation_type": "uniform", "upper_bound": KL})
    eng = engine_for(env, cfg, 2)
    root = roots([env, env])
    eng._load_rng(pcg64_of([0, 1]))

    def call(cfg_=None, mdp=None, terminal=None, env_draws=1, root_states=None):
        return eng.lib.b2_olop_plan_sampled(
            cfg_ if cfg_ is not None else eng.cfg, mdp if mdp is not None else eng.tables.struct(),
            _lib.ptr(eng.terminal) if terminal is None else terminal, env_draws,
            _lib.ptr(root) if root_states is None else root_states, eng.tree, _lib.ptr(eng.rng),
            _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), _lib.current_stream())

    def refused(match, **kw):
        with pytest.raises(_lib.B2Error, match=match):
            _lib.check(call(**kw))

    assert call() == 0
    torch.cuda.synchronize()
    refused("null pointer", terminal=0)
    refused("null pointer", root_states=0)
    for field, value, match in [("cdf", 0, "tables missing"), ("row_ok", 0, "tables missing"),
                                ("n_next", 0, "finite MDP shape"), ("n_actions", 3, "finite MDP shape"),
                                ("n_states", 0, "finite MDP shape")]:
        m = eng.tables.struct()
        setattr(m, field, value)
        refused(match, mdp=m)
    refused("env_draws", env_draws=2)
    for field, value, match in [("env_kind", _lib.ENV_HIGHWAY, "env_kind"), ("n_trees", 0, "batch"),
                                ("horizon", 0, "batch"), ("episodes", -1, "batch"), ("n_actions", 9, "n_actions"),
                                ("node_capacity", 10, "node_capacity"), ("thresholds", None, "tables missing"),
                                ("init_upper", None, "tables missing")]:
        c = type(eng.cfg).from_buffer_copy(eng.cfg)
        setattr(c, field, value)
        refused(match, cfg_=c)
