"""Pin the BRUE restatement (oracle/brue.py) and the agent's completed config against tests/golden/golden_brue.json,
recorded from the UNMODIFIED reference by tests/golden/make_golden_brue.py.  Everything is exact, floats included."""
import json

import numpy as np
import pytest

from oracle import brue, envs, ref_loader
from tests.util import load_golden, load_mdps

G = load_golden("golden_brue.json")
M = load_mdps()


def case_env(spec):
    """The env a golden case was recorded on (make_golden_brue.py::make_env)."""
    if spec["name"] == "highway":
        return envs.HighwayLite(seed=spec["seed"])
    n = spec["name"]
    reward = np.zeros_like(M[n + "_R"]) if spec.get("zero_rewards") else M[n + "_R"]
    return envs.FiniteMDPLite(M[n + "_T"], reward, M[n + "_term"], state=spec.get("state", 0))


def completed_planner_config(config):
    from rl_agents_b200.agents.tree_search.brue import BRUE
    cfg = BRUE.default_config()
    BRUE.rec_update(cfg, json.loads(json.dumps(config)))
    return cfg


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def oracle_case(g):
    """Run the oracle over a golden case's decisions; -> (plans, last tree, last rollouts, rng)."""
    rng, _ = ref_loader.legacy_np_random(g["seed"])
    cfg = completed_planner_config(g["config"])
    plans = []
    for _ in range(len(g.get("plans", [g["plan"]]))):
        plan, t, rollouts = brue.brue_plan(envs.LegacyStepEnv(case_env(g["env"])), cfg, rng)
        plans.append(plan)
    return plans, t, rollouts, rng


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_brue_oracle_matches_reference(key):
    g = G["cases"][key]
    plans, t, rollouts, rng = oracle_case(g)
    assert plans == g.get("plans", [g["plan"]])
    assert (t.horizon, rollouts, t.budget_left) == (g["horizon"], g["rollouts"], g["budget_left"])
    assert rng_state(rng) == g["rng_state"]
    assert brue.tree_digest(brue.tree_dict(t)) == g["tree"]


def test_golden_cases_cover_what_they_are_named_for():
    c = G["cases"]
    assert max(c["trap_terminal_root_b50_g0.8"]["tree"]["depth"]) == 1                       # one-step rollouts
    assert c["trap_terminal_root_b50_g0.8"]["rollouts"] == 50
    assert min(c["trap_raw_b300_g0.8"]["tree"]["value"]) < 0                                 # raw [-1, 1] rewards
    assert any(g["budget_left"] < 0 for g in c.values())                                     # last rollout overshoots
    assert len(set(tuple(p) for p in c["large1_receding3_three_decisions"]["plans"])) > 1


def test_budget_and_horizon_below_one_raise_value_error():
    env = envs.LegacyStepEnv(case_env({"name": "large1"}))
    with pytest.raises(ValueError) as e:
        brue.brue_plan(env, completed_planner_config({"budget": 0}), ref_loader.legacy_np_random(0)[0])
    assert str(e.value) == G["errors"]["budget_zero"]["message"]
    with pytest.raises(ValueError):
        brue.brue_plan(env, completed_planner_config({"horizon": 0}), ref_loader.legacy_np_random(0)[0])


@pytest.mark.parametrize("name", sorted(G["configs"]))
def test_agent_completed_config_equals_the_reference(name):
    """BRUEAgent built as agent_factory builds it (`__class__` left in) completes its config to the reference
    agent's, OLOP's keys and budget allocation included."""
    from rl_agents_b200.agents.tree_search.brue import BRUEAgent
    g = G["configs"][name]
    env = envs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"])
    cfg = json.loads(json.dumps(g["config"]))
    if "__class__" in cfg:
        cfg["__class__"] = "<class 'rl_agents_b200.agents.tree_search.brue.BRUEAgent'>"
    agent = BRUEAgent(env, cfg)
    ours = json.loads(json.dumps({k: v for k, v in agent.config.items() if k != "__class__"}))
    assert ours == g["completed"]


def test_agent_refuses_what_it_does_not_reproduce():
    from rl_agents_b200.agents.tree_search.brue import BRUEAgent
    env = envs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"])
    with pytest.raises(NotImplementedError):
        BRUEAgent(env, {"step_strategy": "subtree"})
    from rl_agents_b200.envs import IntersectionLiteEnv
    with pytest.raises(NotImplementedError):
        BRUEAgent(IntersectionLiteEnv(seed=0), {})
    from rl_agents_b200.envs import FiniteMDPEnv
    fin = FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"])
    for bad in ({"budget": 0}, {"horizon": 0}):
        with pytest.raises(ValueError):
            BRUEAgent(fin, bad).plan(0)            # refused before any device work
