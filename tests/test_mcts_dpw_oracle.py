"""Pin the MCTS-DPW restatement (oracle/mcts_dpw.py), the agent's completed config and its error paths against
tests/golden/golden_mcts_dpw.json, recorded from the UNMODIFIED reference by tests/golden/make_golden_mcts_dpw.py; and
the host tables the device reads (widening thresholds, exploration bonus, observation keys) against the reference's
own expressions.  Everything is exact."""
import hashlib
import json

import numpy as np
import pytest

from oracle import envs, ref_loader
from oracle import mcts_dpw as dpw
from tests.util import load_golden, load_mdps

G = load_golden("golden_mcts_dpw.json")
M = load_mdps()


def case_env(spec):
    """The env a golden case was recorded on (make_golden_mcts_dpw.py::make_env)."""
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
    """The planner config MCTSDPWAgent completes `config` to (episodes / horizon allocated when horizon is unset)."""
    from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPWAgent
    return MCTSDPWAgent(envs.FiniteMDPLite(M["trap_T"], M["trap_R"]), json.loads(json.dumps(config))).planner.config


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def oracle_case(g):
    """Run the oracle over a golden case's decisions; -> (plans, last tree, last env steps, rng)."""
    rng, _ = ref_loader.legacy_np_random(g["seed"])
    cfg = completed_planner_config(g["config"])
    plans = []
    for _ in range(len(g.get("plans", [g["plan"]]))):
        plan, t, steps = dpw.mcts_dpw_plan(case_env(g["env"]), cfg, rng)
        plans.append(plan)
    return plans, t, steps, rng


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_mcts_dpw_oracle_matches_reference(key):
    g = G["cases"][key]
    plans, t, steps, rng = oracle_case(g)
    assert plans == g.get("plans", [g["plan"]])
    assert steps == g["steps"]
    assert rng_state(rng) == g["rng_state"]
    assert dpw.tree_digest(dpw.tree_dict(t)) == g["tree"]


def test_golden_cases_cover_what_they_are_named_for():
    c = G["cases"]
    # the two states whose keys collide reach one shared decision node under the root's action 0
    assert dpw.obs_key(406) == dpw.obs_key(678)
    nxt = np.array(G["mdps"]["collide680"]["next"])
    assert sorted(nxt[0, 0].tolist()) == [406, 678]
    _, t, _, _ = oracle_case(c["collide680_closed_loop"])
    a0 = next(k for k in t.children[0] if t.key[k] == 0)
    assert [t.key[k] for k in t.children[a0]] == [dpw.obs_key(406)] and t.count[t.children[a0][0]] > 10
    # closed loop: some chance node holds several next states
    for key in ("stoch8_closed_loop_h6_e200", "garnet12_closed_loop_h6_e200", "stoch8_closed_loop_k2_a0.5"):
        _, t, _, _ = oracle_case(c[key])
        assert max(len(t.children[i]) for i in range(len(t)) if t.kind[i] == dpw.CHANCE) > 1
    # open loop: every chance node has one child
    _, t, _, _ = oracle_case(c["stoch8_h6_e200"])
    assert all(len(t.children[i]) == 1 for i in range(len(t)) if t.kind[i] == dpw.CHANCE and t.children[i])
    # the terminal root is stepped from and the run ends there: no rollout
    assert c["trap_terminal_root_default"]["steps"] == c["trap_terminal_root_default"]["episodes"]
    assert sum(k.startswith("hw") for k in c) == 7 and len(c["stoch8_three_decisions"]["plans"]) == 3


def test_state_widening_draw_fires_in_closed_loop():
    """The closed-loop goldens take ChanceNode.get_child's choice(list(children)) branch; open loop never does."""
    for key in ("stoch8_closed_loop_h6_e200", "garnet12_closed_loop_h6_e200"):
        assert oracle_case(G["cases"][key])[1].state_draws > 0, key
    assert oracle_case(G["cases"]["stoch8_h6_e200"])[1].state_draws == 0


def test_oracle_errors_match_the_reference():
    errs = G["errors"]
    env = case_env({"name": "stoch8"})
    with pytest.raises(ZeroDivisionError) as e:
        dpw.mcts_dpw_plan(env, completed_planner_config({"alpha_action": -0.5}), ref_loader.legacy_np_random(0)[0])
    assert str(e.value) == errs["alpha_action_negative"]["message"]
    with pytest.raises(ValueError) as e:
        dpw.mcts_dpw_plan(case_env({"name": "stoch8_bad_row"}), completed_planner_config({"horizon": 6, "episodes": 200}),
                          ref_loader.legacy_np_random(0)[0])
    assert str(e.value) == errs["bad_row"]["message"]
    # the reference returns None for horizon < 1 (a childless root): refused here
    assert errs["horizon_negative_plan"]["plan"] is None
    with pytest.raises(ValueError, match="horizon"):
        dpw.mcts_dpw_plan(env, completed_planner_config({"horizon": -1, "episodes": 3}), ref_loader.legacy_np_random(0)[0])
    with pytest.raises(NotImplementedError):
        dpw.mcts_dpw_plan(env, completed_planner_config({"step_strategy": "subtree"}), ref_loader.legacy_np_random(0)[0])


@pytest.mark.parametrize("name", sorted(G["configs"]))
def test_agent_completed_config_equals_the_reference(name):
    from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPWAgent
    g = G["configs"][name]
    agent = MCTSDPWAgent(case_env({"name": "stoch8"}), json.loads(json.dumps(g["config"])))
    assert json.loads(json.dumps(agent.config)) == g["completed"]
    assert json.loads(json.dumps(agent.planner.config)) == g["planner"]


def test_agent_refuses_before_any_device_work():
    from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPWAgent
    from rl_agents_b200.envs import FiniteMDPEnv, IntersectionLiteEnv
    fin = FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"])
    with pytest.raises(KeyError, match="episodes"):
        MCTSDPWAgent(fin, {"horizon": 3}).plan(0)
    with pytest.raises(ValueError, match="horizon"):
        MCTSDPWAgent(fin, {"horizon": -1, "episodes": 3}).plan(0)
    with pytest.raises(ZeroDivisionError):
        MCTSDPWAgent(fin, {"alpha_action": -0.5}).plan(0)
    with pytest.raises(NotImplementedError):
        MCTSDPWAgent(fin, {"step_strategy": "subtree"})
    with pytest.raises(NotImplementedError):
        MCTSDPWAgent(IntersectionLiteEnv(seed=0), {})
    for ext in ({"wavefront": 64}, {"root_parallel": 4}):
        with pytest.raises(NotImplementedError):
            MCTSDPWAgent(fin, ext)


@pytest.mark.parametrize("k, alpha", [(3, 0.3), (1, 0.3), (2, 0.5), (10, 0.3), (3, 0), (0, 0.3), (0.5, 1.0),
                                      (1.7, 0.25), (-1, 0.3), (float("nan"), 0.3), (float("inf"), 0.5)])
def test_widening_table_equals_the_reference_expression(k, alpha):
    from rl_agents_b200.engine.mcts_dpw import widening_table
    cap = 8
    w = widening_table(k, alpha, 300, cap)
    for N in range(301):
        allowed = [m for m in range(cap + 1) if not (k * N ** alpha < m)]
        assert w[N] == (max(allowed) if allowed else -1), N
        assert allowed == list(range(w[N] + 1))               # down-closed: m widens iff m <= W[N]
    with pytest.raises(ZeroDivisionError):
        widening_table(3, -0.5, 10, cap)


def test_bonus_table_equals_the_reference_expression():
    from rl_agents_b200.engine.mcts_dpw import bonus_table
    E = 300
    t = bonus_table(E)
    assert t.dtype == np.float64 and t.size == E * (E + 1) // 2
    ref = np.array([np.sqrt(np.log(N / n)) for N in range(1, E + 1) for n in range(1, N + 1)])
    assert t.tobytes() == ref.tobytes()


def test_observation_keys_equal_sha1_prefixes():
    from rl_agents_b200.engine.mcts_dpw import OPEN_LOOP_KEY, observation_keys
    keys = observation_keys(1000)
    for s in range(1000):
        assert keys[s] == int(hashlib.sha1(str(s).encode("UTF-8")).hexdigest()[:5], 16)
    assert keys[406] == keys[678]
    assert OPEN_LOOP_KEY == dpw.OPEN_LOOP_KEY == int(hashlib.sha1(b"None").hexdigest()[:5], 16)


def test_bonus_table_cap():
    from rl_agents_b200.engine.mcts_dpw import MAX_BONUS_BYTES, check_bonus_table
    check_bonus_table(4000)
    with pytest.raises(ValueError, match="MiB"):
        check_bonus_table(5000)
    assert 8 * 4000 * 4001 // 2 <= MAX_BONUS_BYTES < 8 * 5000 * 5001 // 2
