"""Pin the sparse-sampling restatement (oracle/sparse_sampling.py), the agent's completed config and its error paths
against tests/golden/golden_sparse_sampling.json, recorded from the UNMODIFIED reference by
tests/golden/make_golden_sparse_sampling.py; and the host pieces the device replays the env's sampling with (the
SeedSequence / PCG64 seeding twin, Generator.choice's row checks and cdf) against numpy.  Everything is exact."""
import json

import numpy as np
import pytest

from oracle import envs, pcg64, ref_loader, seed_sequence
from oracle import sparse_sampling as ss
from tests.util import load_golden, load_mdps

G = load_golden("golden_sparse_sampling.json")
M = load_mdps()


def case_env(spec):
    """The env a golden case was recorded on (make_golden_sparse_sampling.py::make_env)."""
    if spec["name"] == "highway":
        return envs.HighwayLite(seed=spec["seed"])
    n = spec["name"]
    if n in G["mdps"]:
        t = G["mdps"][n]
        reward = np.array(t["reward"], dtype=np.float64)
        if spec.get("zero_rewards"):
            reward = np.zeros_like(reward)
        return envs.FiniteMDPLite(np.array(t["transition"], dtype=np.float64), reward, np.array(t["terminal"]),
                                  mode=t["mode"], nxt=None if "next" not in t else np.array(t["next"]),
                                  state=spec.get("state", 0))
    reward = np.zeros_like(M[n + "_R"]) if spec.get("zero_rewards") else M[n + "_R"]
    return envs.FiniteMDPLite(M[n + "_T"], reward, M[n + "_term"], state=spec.get("state", 0))


def completed_planner_config(config):
    from rl_agents_b200.agents.tree_search.sparse_sampling import SparseSampling
    cfg = SparseSampling.default_config()
    SparseSampling.rec_update(cfg, json.loads(json.dumps(config)))
    return cfg


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def golden_root_q(g):
    return np.array([np.nan if v is None else v for v in g["root_q"]], dtype=np.float64)


def oracle_case(g):
    """Run the oracle over a golden case's decisions; -> (plans, last tree, last root values, rng)."""
    rng, _ = ref_loader.legacy_np_random(g["seed"])
    cfg = completed_planner_config(g["config"])
    plans = []
    for _ in range(len(g.get("plans", [g["plan"]]))):
        plan, t, root_q = ss.sparse_sampling_plan(envs.LegacyStepEnv(case_env(g["env"])), cfg, rng)
        plans.append(plan)
    return plans, t, root_q, rng


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_sparse_sampling_oracle_matches_reference(key):
    g = G["cases"][key]
    plans, t, root_q, rng = oracle_case(g)
    assert plans == g.get("plans", [g["plan"]])
    assert rng_state(rng) == g["rng_state"]
    assert np.array_equal(root_q, golden_root_q(g), equal_nan=True)
    assert sum(t.kind) == g["chance_nodes"]
    assert ss.tree_digest(ss.tree_dict(t)) == g["tree"]


def test_golden_cases_cover_what_they_are_named_for():
    c, mdps = G["cases"], G["mdps"]
    # the sparse garnet's root rows repeat a next state and hold zero-probability entries
    nxt, p = np.array(mdps["garnet12"]["next"]), np.array(mdps["garnet12"]["transition"])
    assert len(set(nxt[0, 0].tolist())) < nxt.shape[-1] and (p[0, 0] == 0).any() and (p[0, 1] == 0).any()
    # ... and first-visit merging shows in the tree: a next-state child reached by more than one sample
    assert max(c["garnet12_sparse_shipped"]["tree"]["count"]) > 1
    # zero rewards: every root value ties, so the recommendation drew choice(indices) past the C draws per chance node
    def after_seed_draws(g):
        rng = ref_loader.legacy_np_random(g["seed"])[0]
        for _ in range(g["samples"]):
            rng.integers(2 ** 30)
        return rng_state(rng)
    zero = c["stoch8_zero_rewards_shipped"]
    assert len(set(zero["root_q"])) == 1 and after_seed_draws(zero) != zero["rng_state"]
    assert after_seed_draws(c["stoch8_shipped"]) == c["stoch8_shipped"]["rng_state"]
    assert c["stoch8_terminal_root_shipped"]["env"]["state"] == 7 and G["mdps"]["stoch8"]["terminal"][7]
    assert c["stoch8_h4_c5_g0.9"]["tree"]["n_nodes"] > 5000
    assert len(c["stoch8_three_decisions"]["plans"]) == 3
    assert np.isnan(np.array(G["mdps"]["stoch8_unreached_nan_row"]["transition"], dtype=np.float64)).any()
    assert sum(k.startswith("hw") for k in c) == 5


def test_oracle_errors_match_the_reference():
    env = envs.LegacyStepEnv(case_env({"name": "stoch8"}))
    errs = G["errors"]
    with pytest.raises(ValueError) as e:
        ss.sparse_sampling_plan(env, completed_planner_config({"horizon": 0, "C": 3}), ref_loader.legacy_np_random(0)[0])
    assert str(e.value) == errs["horizon_zero"]["message"]
    for cfg, name in (({"C": 3}, "missing_horizon"), ({"horizon": 3}, "missing_c")):
        with pytest.raises(KeyError) as e:
            ss.sparse_sampling_plan(env, completed_planner_config(cfg), ref_loader.legacy_np_random(0)[0])
        assert errs[name]["error"] == "KeyError" and str(e.value) == errs[name]["message"]
    for cfg in ({"horizon": -1, "C": 1}, {"horizon": 2, "C": 0}):
        with pytest.raises(ValueError):
            ss.sparse_sampling_plan(env, completed_planner_config(cfg), ref_loader.legacy_np_random(0)[0])
    bad = envs.LegacyStepEnv(case_env({"name": "stoch8_bad_root_row"}))
    with pytest.raises(ValueError) as e:
        ss.sparse_sampling_plan(bad, completed_planner_config({"horizon": 3, "C": 3}), ref_loader.legacy_np_random(0)[0])
    assert str(e.value) == errs["bad_root_row"]["message"]


@pytest.mark.parametrize("name", sorted(G["configs"]))
def test_agent_completed_config_equals_the_reference(name):
    """SparseSamplingAgent built as agent_factory builds it (`__class__` left in) completes its own config and its
    planner's to the reference's."""
    from rl_agents_b200.agents.tree_search.sparse_sampling import SparseSamplingAgent
    g = G["configs"][name]
    cfg = json.loads(json.dumps(g["config"]))
    if "__class__" in cfg:
        cfg["__class__"] = "<class 'rl_agents_b200.agents.tree_search.sparse_sampling.SparseSamplingAgent'>"
    agent = SparseSamplingAgent(case_env({"name": "stoch8"}), cfg)
    assert json.loads(json.dumps({k: v for k, v in agent.config.items() if k != "__class__"})) == g["completed"]
    assert json.loads(json.dumps({k: v for k, v in agent.planner.config.items() if k != "__class__"})) == g["planner"]


def test_agent_refuses_before_any_device_work():
    """The reference's errors for a missing horizon / C and horizon 0; ValueError where it recurses without end or
    hits an unbound variable; NotImplementedError for what the device does not reproduce."""
    from rl_agents_b200.agents.tree_search.sparse_sampling import SparseSamplingAgent
    from rl_agents_b200.envs import FiniteMDPEnv, IntersectionLiteEnv
    fin = FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"])
    with pytest.raises(KeyError, match="horizon"):
        SparseSamplingAgent(fin, {"C": 3}).plan(0)
    with pytest.raises(KeyError, match="C"):
        SparseSamplingAgent(fin, {"horizon": 3}).plan(0)
    with pytest.raises(ValueError) as e:
        SparseSamplingAgent(fin, {"horizon": 0}).plan(0)          # C is never read at horizon 0
    assert str(e.value) == G["errors"]["horizon_zero"]["message"]
    for bad in ({"horizon": -1, "C": 3}, {"horizon": 3, "C": 0}):
        with pytest.raises(ValueError):
            SparseSamplingAgent(fin, bad).plan(0)
    with pytest.raises(NotImplementedError):
        SparseSamplingAgent(fin, {"horizon": 3, "C": 3, "step_strategy": "subtree"})
    with pytest.raises(NotImplementedError):
        SparseSamplingAgent(IntersectionLiteEnv(seed=0), {"horizon": 3, "C": 3})


def test_seed_sequence_twin_equals_numpy_default_rng():
    """pcg64_from_seed(s) -- the CPU twin of Pcg64::seed_from -- is np.random.default_rng(s)'s bit generator, over
    the seeds a planner's randint(2**30) can draw, ends included, and a few above 2**30."""
    seeds = list(range(1500)) + [2 ** 30 - 1 - i for i in range(500)] + [2 ** 29 + 7 * i for i in range(500)]
    seeds += [2 ** 31, 2 ** 32 - 1]
    rs = np.random.default_rng(12345)
    seeds += rs.integers(0, 2 ** 30, size=1000).tolist()
    for s in seeds:
        a = pcg64.PCG64.from_numpy(np.random.default_rng(s))
        b = seed_sequence.pcg64_from_seed(s)
        assert (a.state, a.inc, a.has_uint32, a.uinteger) == (b.state, b.inc, b.has_uint32, b.uinteger), s
    # and its first random() is the env's first draw
    for s in (0, 1, 2 ** 30 - 1):
        assert seed_sequence.pcg64_from_seed(s).random() == np.random.default_rng(s).random()


def test_sampled_tables_follow_generator_choice():
    """row_ok is exactly the rows Generator.choice accepts; the cdf is the one it searches; searchsorted's right side
    over that cdf with the seeded env's random() is its draw."""
    from rl_agents_b200.engine.tables import choice_rows_ok, sampled_mdp_tables
    rng = np.random.default_rng(7)
    rows = [rng.uniform(size=5) for _ in range(40)]
    rows = [r / r.sum() for r in rows]
    rows += [np.array([0.5, 0.0, 0.5]), np.array([0.0, 0.0, 1.0]), np.array([1.0]), np.array([0.5, np.nan, 0.5]),
             np.array([-0.25, 1.25, 0.0]), np.array([0.5, 0.5 + 1e-9]), np.array([0.5, 0.5 + 1e-7]),
             np.array([0.0, 0.0]), np.array([np.inf, 0.0]), np.array([0.3, 0.3, 0.3])]
    for r in rows:
        try:
            np.random.default_rng(0).choice(r.size, p=r)
            accepted = True
        except ValueError:
            accepted = False
        assert bool(choice_rows_ok(r[None])[0]) == accepted, r
    t = G["mdps"]["garnet12"]
    mdp = envs.FiniteMDPLite(np.array(t["transition"]), np.array(t["reward"]), mode="sparse",
                             nxt=np.array(t["next"])).mdp
    tab = sampled_mdp_tables(mdp)
    assert tab["row_ok"].all()
    for s in range(3):
        for a in range(3):
            p = mdp.transition[s, a]
            cdf = p.cumsum()
            cdf /= cdf[-1]
            assert np.array_equal(tab["cdf"][s, a], cdf)
            for seed in range(50):
                k = int(np.random.default_rng(seed).choice(p.size, p=p))
                u = seed_sequence.pcg64_from_seed(seed).random()
                assert int(np.searchsorted(tab["cdf"][s, a], u, side="right")) == k
