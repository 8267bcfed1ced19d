"""Pin the MDP-GapE restatement (oracle/mdp_gape.py) and the agent's completed config against
tests/golden/golden_mdp_gape.json, recorded from the UNMODIFIED reference by tests/golden/make_golden_mdp_gape.py."""
import json

import numpy as np
import pytest

from oracle import envs, ref_loader
from oracle import mdp_gape as gape
from tests.util import load_golden, load_mdps

G = load_golden("golden_mdp_gape.json")
M = load_mdps()


def case_env(key):
    """The env a golden case was recorded on (see make_golden_mdp_gape.py)."""
    if key.startswith("hw"):
        return envs.HighwayLite(seed=int(key[2]))
    if key.startswith("trap01"):
        return envs.FiniteMDPLite(M["trap_T"], (M["trap_R"] + 1) / 2, M["trap_term"])
    name = key.split("_")[0]
    return envs.FiniteMDPLite(M[name + "_T"], M[name + "_R"], M[name + "_term"])


def completed_planner_config(config):
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapE
    cfg = MDPGapE.default_config()
    MDPGapE.rec_update(cfg, json.loads(json.dumps(config)))
    return cfg


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def assert_gape_tree(t, g, atol=0.0):
    """Oracle tree `t` against a golden digest (oracle.mdp_gape.tree_digest): structure exact; float fields exact,
    or within `atol` (sums: n_nodes * atol) where a different log implementation is involved."""
    d = gape.tree_digest(gape.tree_dict(t))
    for k in ("n_nodes", "structure_sha256") + gape.INT_FIELDS:
        assert d[k] == g[k], k
    for f in gape.FLOAT_FIELDS:
        assert [x is None for x in d[f]] == [x is None for x in g[f]], f
        a = np.array([x for x in d[f] if x is not None] + [d["sum_" + f]])
        b = np.array([x for x in g[f] if x is not None] + [g["sum_" + f]])
        tol = np.full(a.size, float(atol))
        tol[-1] *= g["n_nodes"]
        assert (np.abs(a - b) <= tol).all(), (f, np.abs(a - b).max())


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_mdp_gape_oracle_matches_reference(key):
    g = G["cases"][key]
    rng, _ = ref_loader.legacy_np_random(g["seed"])
    plan, t, episodes_run = gape.mdp_gape_plan(envs.LegacyStepEnv(case_env(key)), completed_planner_config(g["config"]),
                                               rng)
    assert (t.episodes, t.horizon) == (g["episodes"], g["horizon"])
    assert plan == g["plan"] and episodes_run == g["episodes_run"]
    assert episodes_run * t.horizon == g["budget_used"]
    kids = list(t.children(0))
    assert (kids.index(t.best), kids.index(t.challenger)) == (g["best_index"], g["challenger_index"])
    assert rng_state(rng) == g["rng_state"]
    # the reference evaluates theta (utils.py:279-282) in numba-compiled code: its log may differ from this
    # module's by an ulp, which moves the unobserved placeholders' mass z at the 1e-16 level
    k3 = completed_planner_config(g["config"])["max_next_states_count"] > 1
    assert_gape_tree(t, g["tree"], atol=1e-12 if k3 else 0.0)


def test_mdp_gape_oracle_raises_like_the_reference_on_rewards_outside_unit_interval():
    g = G["errors"]["trap_raw_rewards"]
    env = envs.LegacyStepEnv(envs.FiniteMDPLite(M["trap_T"], M["trap_R"], M["trap_term"]))
    with pytest.raises(ValueError, match="normalized in"):
        gape.mdp_gape_plan(env, completed_planner_config(g["config"]), ref_loader.legacy_np_random(g["seed"])[0])


def test_single_root_action_raises_value_error():
    env = envs.LegacyStepEnv(envs.FiniteMDPLite(np.zeros((3, 1), int), np.full((3, 1), 0.5), None))
    with pytest.raises(ValueError):
        gape.mdp_gape_plan(env, completed_planner_config({"budget": 50}), ref_loader.legacy_np_random(0)[0])


def test_one_positive_max_expectation_and_kl_lower_bound_known_answers():
    for f, q, c, ref in G["max_expectation_one_positive"]:
        p = gape.max_expectation_one_positive(np.array(f), np.array(q), c)
        np.testing.assert_allclose(p, ref, rtol=1e-14, atol=1e-15)
    for s, c, th, ref in G["kl_lower_bound"]:
        assert gape.kl_bound(s, c, th, lower=True) == ref
    for s, c, th in [(0.5, 1, 2.0), (3.25, 7, 5.5), (17.5, 40, 9.2)]:
        assert gape.kl_bound(s, c, th, lower=True) <= s / c <= gape.kl_bound(s, c, th)


@pytest.mark.parametrize("name", sorted(G["configs"]))
def test_agent_completed_config_equals_the_reference(name):
    """MDPGapEAgent built as agent_factory builds it (`__class__` left in) completes its config to the
    reference agent's, including the planner keys and the budget allocation."""
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapEAgent
    g = G["configs"][name]
    env = envs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"])
    cfg = json.loads(json.dumps(g["config"]))
    if "__class__" in cfg:
        cfg["__class__"] = "<class 'rl_agents_b200.agents.tree_search.mdp_gape.MDPGapEAgent'>"
    agent = MDPGapEAgent(env, cfg)
    ours = json.loads(json.dumps({k: v for k, v in agent.config.items() if k != "__class__"}))
    assert ours == g["completed"]
    assert agent.planner.budget_used == 0 and agent.planner.next_observation is None


def test_agent_refuses_what_it_does_not_reproduce():
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapEAgent
    env = envs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"])
    with pytest.raises(NotImplementedError):
        MDPGapEAgent(env, {"step_strategy": "subtree"})
    with pytest.raises(NotImplementedError):
        MDPGapEAgent(env, {"upper_bound": {"type": "hoeffding"}})
    from rl_agents_b200.envs import IntersectionLiteEnv
    with pytest.raises(NotImplementedError):
        MDPGapEAgent(IntersectionLiteEnv(seed=0), {})
