"""Pin the PlaTyPOOS restatement (oracle/platypoos.py), the agent's completed config and its error paths against
tests/golden/golden_platypoos.json, recorded from the UNMODIFIED reference by tests/golden/make_golden_platypoos.py; and
the host tables the device reads (h_max, p_top, the per-(h, p) quotas, the cross-validation counts, gamma**d) against
the reference's own expressions.  Everything is exact."""
import json
import re

import numpy as np
import pytest

from oracle import envs, ref_loader
from oracle import platypoos as opl
from tests.util import load_golden, load_mdps

G = load_golden("golden_platypoos.json")
M = load_mdps()


def case_env(spec, finite_cls=envs.FiniteMDPLite, highway_cls=None):
    """The env a golden case was recorded on (make_golden_platypoos.py::make_env)."""
    n = spec["name"]
    if n == "highway":
        return (highway_cls or envs.HighwayLite)(seed=spec["seed"])
    if n == "garnet":
        T, R = envs.garnet(spec["states"], spec["actions"], 1, seed=spec["seed"], deterministic=True)
        return finite_cls(T, R, state=spec.get("state", 0))
    if n in G["mdps"]:
        t = G["mdps"][n]
        reward = np.array(t["reward"], dtype=np.float64)
        if spec.get("zero_rewards"):
            reward = np.zeros_like(reward)
        return finite_cls(np.array(t["transition"], dtype=np.float64), reward, np.array(t["terminal"]),
                          mode=t["mode"], nxt=None if "next" not in t else np.array(t["next"]),
                          state=spec.get("state", 0))
    a = spec.get("actions", M[n + "_R"].shape[1])
    reward = M[n + "_R"][:, :a]
    if spec.get("zero_rewards"):
        reward = np.zeros_like(reward)
    return finite_cls(M[n + "_T"][:, :a], reward, M[n + "_term"], state=spec.get("state", 0))


def completed_planner_config(config, env):
    from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOSAgent
    return PlaTyPOOSAgent(env, json.loads(json.dumps(config))).planner.config


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def golden_tree_arrays(g):
    """A golden tree with its float fields decoded from their float64 bytes."""
    t = dict(g["tree"])
    for f in opl.FLOAT_FIELDS:
        t[f] = np.frombuffer(bytes.fromhex(t[f]), dtype=np.float64)
    return t


def assert_tree_equals_golden(d, g):
    """d: a dump with the oracle's fields (lists or arrays); exact, float64 bytes included."""
    t = golden_tree_arrays(g)
    for f in opl.INT_FIELDS:
        assert [int(x) for x in d[f]] == t[f], f
    for f in opl.FLOAT_FIELDS:
        assert np.asarray(d[f], dtype=np.float64).tobytes() == t[f].tobytes(), f


def oracle_case(g):
    rng, _ = ref_loader.legacy_np_random(g["seed"])
    env = case_env(g["env"])
    cfg = completed_planner_config(g["config"], env)
    return opl.platypoos_plan(env, cfg, rng) + (rng,)


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_platypoos_oracle_matches_reference(key):
    g = G["cases"][key]
    plan, t, openings, candidates, rng = oracle_case(g)
    assert plan == g["plan"]
    assert openings == g["openings"]
    assert [list(c) for c in candidates] == g["candidates"]
    assert rng_state(rng) == g["rng_state"]
    assert_tree_equals_golden(opl.tree_dict(t), g)


def test_golden_cases_cover_what_they_are_named_for():
    c = G["cases"]
    # multi-action plans, the widest layer of the budget-50 000 trees, the 200 000 garnet's horizon
    assert max(len(g["plan"]) for g in c.values()) >= 5
    assert c["garnet1000_deterministic_budget200000"]["horizon"] == 90
    assert c["hw3_budget50000_gamma0.9"]["horizon"] == 24
    # the terminal roots: every child of the root is done and none is expanded further
    for key in ("trap_terminal_root", "stoch8_terminal_root"):
        t = c[key]["tree"]
        assert all(d == 1 for d, dep in zip(t["done"], t["depth"]) if dep == 1) and max(t["depth"]) == 1
    # two actions: only action 1 is expanded
    assert set(c["trap_two_actions"]["tree"]["action"][1:]) == {1}
    # zero rewards: every value ties
    t = golden_tree_arrays(c["stoch8_zero_rewards"])
    assert (t["value"] == 0).all() and len(c["stoch8_zero_rewards"]["candidates"]) > 1
    # the explicit horizons are the ones given
    assert c["stoch8_explicit_horizon"]["horizon"] == 7 and c["hw1_explicit_horizon"]["horizon"] == 4


@pytest.mark.parametrize("budget", [3, 7, 100, 500, 2500, 10000, 50000, 200000, 1234567])
@pytest.mark.parametrize("n_actions", [2, 3, 4, 5, 8])
@pytest.mark.parametrize("gamma", [0.5, 0.7, 0.8, 0.9, 0.95, 0.99, 1.0])
def test_host_tables_equal_the_reference_expressions(budget, n_actions, gamma):
    """The engine's tables against the reference's own expressions, evaluated here as platypoos.py writes them."""
    from rl_agents_b200.engine import platypoos as epl
    expansion_budget = budget / n_actions
    h_max = int(np.floor(expansion_budget / (2 * (np.log2(expansion_budget) + 1) ** 2)))
    assert epl.horizon_of(budget, n_actions) == opl.horizon_of(budget, n_actions) == h_max
    if h_max < 2:
        return
    try:
        expected = reference_tables(h_max, gamma)
    except OverflowError:
        # gamma ** (2 h) underflows to 0 deep in a long horizon: the reference's p_top is int(inf), and so is the host's
        with pytest.raises(OverflowError):
            epl.quota_tables(h_max, gamma)
        return
    t = epl.quota_tables(h_max, gamma)
    for h, pt, quotas in expected["explore"]:
        assert t["p_top"][h] == pt
        for p, (nc, ev, mv) in quotas:
            assert (t["nodes_count"][h, p], t["evaluations"][h, p], t["min_visits"][h, p]) == (min(nc, 2 ** 31 - 1), ev, mv)
    for d, cv in enumerate(expected["cv"]):
        assert t["cv_count"][d] == cv
        assert t["gamma_pow"][d].tobytes() == np.float64(gamma ** d).tobytes()


def reference_tables(h_max, gamma):
    """platypoos.py:41-46 and :75-76 as written there."""
    out = {"explore": [], "cv": []}
    for h in range(1, h_max):
        p_top = max(int(np.floor(np.log2(h_max / np.ceil(h ** 2 * gamma ** (2 * h))))), 0)
        quotas = []
        for p in range(p_top, -1, -1):
            nodes_count = int(np.floor(h_max / h * np.ceil(h * 2 ** p * gamma ** (2 * h))))
            evaluations = int(np.ceil(h * 2 ** p * gamma ** (2 * h)))
            min_visits = int(np.ceil((h - 1) * 2 ** p * gamma ** (2 * (h - 1))))
            quotas.append((p, (nodes_count, evaluations, min_visits)))
        out["explore"].append((h, p_top, quotas))
    for d in range(h_max):
        out["cv"].append(int(np.floor((d + 1) * 5 * h_max * gamma ** (2 * d) * (1 - gamma ** 2) ** 2)))
    return out


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_worst_case_arena_bounds_every_golden_tree(key):
    """The default arena holds each golden tree: per depth, the layer widths are within the worst case."""
    from rl_agents_b200.engine import platypoos as epl
    g = G["cases"][key]
    highway = g["env"]["name"] == "highway"
    n_actions = 5 if highway else case_env(g["env"]).action_space.n
    t = epl.quota_tables(g["horizon"], g["config"].get("gamma", 0.8))
    widths = epl.worst_case_layers(g["horizon"], 5 if highway else n_actions - 1, t)
    depth = np.array(g["tree"]["depth"])
    assert len(depth) <= sum(widths)
    for d in range(depth.max() + 1):
        assert (depth == d).sum() <= widths[d], d


@pytest.mark.parametrize("name", sorted(G["configs"]))
def test_completed_configs_equal_the_reference(name):
    c = G["configs"][name]
    from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOSAgent
    agent = PlaTyPOOSAgent(case_env(c["env"]), json.loads(json.dumps(c["config"])))
    assert json.loads(json.dumps(agent.config)) == c["completed"]
    assert json.loads(json.dumps(agent.planner.config)) == c["planner"]


def test_shipped_baseline_config_with_its_class_switched_completes_to_the_reference():
    """scripts/configs/HighwayEnv/agents/PlaTyPOOSAgent/baseline.json with only `__class__` switched, built as
    agent_factory builds it (`__class__` left in)."""
    from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOSAgent
    from rl_agents_b200.envs import HighwayLiteEnv
    c = G["configs"]["baseline_highway"]
    config = dict(c["config"], __class__="<class 'rl_agents_b200.agents.tree_search.platypoos.PlaTyPOOSAgent'>")
    agent = PlaTyPOOSAgent(HighwayLiteEnv(seed=0), json.loads(json.dumps(config)))
    assert json.loads(json.dumps({k: v for k, v in agent.config.items() if k != "__class__"})) == c["completed"]
    assert json.loads(json.dumps({k: v for k, v in agent.planner.config.items() if k != "__class__"})) == c["planner"]
    assert agent.planner.config["horizon"] == 2


def test_error_types_match_the_reference():
    from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOSAgent
    from rl_agents_b200.engine.platypoos import check_plannable
    e = G["errors"]
    # a negative budget: the same expression fails at construction, with the same message
    with pytest.raises(ValueError) as err:
        PlaTyPOOSAgent(case_env({"name": "stoch8"}), {"budget": -10})
    assert e["negative_budget"]["error"] == "ValueError" and str(err.value) == e["negative_budget"]["message"]
    # no candidate: h_max < 2 (the default budget on HighwayLite; horizon 1) or one finite action
    for key, (h, n, finite) in (("default_budget_highway", (0, 5, False)), ("horizon_1", (1, 4, True)),
                                ("one_action", (14, 1, True))):
        assert e[key]["error"] == "ValueError"
        with pytest.raises(ValueError) as err:
            check_plannable(h, n, finite)
        assert str(err.value).startswith(e[key]["message"])
    # the oracle: the same message from get_plan's max()
    with pytest.raises(ValueError, match=re.escape(e["horizon_1"]["message"])):
        opl.platypoos_plan(case_env({"name": "stoch8"}), {"horizon": 1, "gamma": 0.8, "step_strategy": "reset"},
                           ref_loader.legacy_np_random(0)[0])
    # a reached row that Generator.choice rejects: numpy's own message
    g = G["errors"]["bad_row"]
    env = case_env({"name": "stoch8_bad_row"})
    with pytest.raises(ValueError, match=re.escape(g["message"])):
        opl.platypoos_plan(env, completed_planner_config({"budget": 10000, "gamma": 0.9}, env),
                           ref_loader.legacy_np_random(0)[0])
    # "subtree" fails in the reference at the next decision; the port refuses it at construction
    assert e["subtree_second_decision"]["error"] == "ValueError"
    with pytest.raises(NotImplementedError):
        PlaTyPOOSAgent(case_env({"name": "stoch8"}), {"step_strategy": "subtree"})
    # IntersectionLite
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv
    with pytest.raises(NotImplementedError):
        PlaTyPOOSAgent(IntersectionLiteEnv(seed=0), {"budget": 10000})
