"""Pin MCTS and OLOP on IntersectionLite: oracle/planners.py's mcts_plan / olop_plan on oracle.intersection.IntersectionLite
against tests/golden/golden_intersection_planners.json, recorded from the UNMODIFIED reference by
tests/golden/make_golden_intersection_planners.py (trees, plans and RNG words, exact), and the C statement of the MCTS
search (oracle/c_mcts_intersection.py) against the Python oracle."""
import filecmp
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import envs, planners, ref_loader
from oracle import intersection as oit
from tests.util import GOLDEN, load_golden

G = load_golden("golden_intersection_planners.json")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def case_env(spec):
    """make_golden_intersection_planners.py::make_env."""
    st = oit.make_intersection_state(spec["seed"])
    if "speed_index" in spec:
        st.speed_index = int(spec["speed_index"])
    return oit.IntersectionLite(st)


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def oracle_mcts(g, rng, env=None, tree=None):
    c = g["config"]
    return planners.mcts_plan(env or case_env(g["env"]), g["episodes"], g["horizon"], c["gamma"], g["temperature"], rng,
                              prior_policy=c.get("prior_policy"), rollout_policy=c.get("rollout_policy"), tree=tree)


def oracle_olop(g, rng):
    c = g["config"]
    return planners.olop_plan(envs.LegacyStepEnv(case_env(g["env"])), c.get("budget", 0), c["gamma"], rng,
                              upper_bound=c["upper_bound"], continuation_type=c["continuation_type"],
                              episodes=g["episodes"], horizon=g["horizon"])


def canonical(t):
    from tests.util import canonical_tree
    return canonical_tree(t.first_child, t.n_children, [t.count, t.value, t.prior])


@pytest.mark.skipif(not ref_loader.reference_available(), reason="needs the reference tree")
def test_golden_generator_reproduces_its_json(tmp_path):
    out = tmp_path / "golden.json"
    subprocess.run([sys.executable, os.path.join(GOLDEN, "make_golden_intersection_planners.py"), "--out", str(out)],
                   check=True, cwd=ROOT, stdout=subprocess.DEVNULL)
    assert filecmp.cmp(str(out), os.path.join(GOLDEN, "golden_intersection_planners.json"), shallow=False)


def test_golden_cases_cover_what_they_are_named_for():
    m = G["mcts"]
    # the two-action roots
    assert sorted(m["s5_top_speed_b300_g0.85"]["tree"]["action"][1:3]) == [oit.A_SLOWER, oit.A_IDLE]
    assert sorted(m["s6_bottom_speed_ep60_h5"]["tree"]["action"][1:3]) == [oit.A_IDLE, oit.A_FASTER]
    # horizons past DURATION; the "zeros" KeyError; plans several actions long
    assert m["s1_ep40_h16_g0.9"]["horizon"] > oit.DURATION and G["olop"]["s1_ep12_h15_kl_uniform"]["horizon"] > oit.DURATION
    assert G["olop"]["s2_b200_kl_zeros_keyerror"]["error"] == {"error": "KeyError", "message": "0"}
    assert min(len(g["plan"]) for g in m.values()) >= 5
    # the preference policies put SLOWER first where it is available: a prior above the uniform one
    t = m["s0_preference_b300_g0.8"]["tree"]
    assert any(a == oit.A_SLOWER and p > 1 / 3 for a, p in zip(t["action"], t["prior"]))


@pytest.mark.parametrize("key", sorted(G["mcts"]))
def test_mcts_oracle_matches_reference(key):
    g = G["mcts"][key]
    rng = np_random(g["seed"])
    plan, t = oracle_mcts(g, rng)
    assert plan == g["plan"]
    for f in ("parent", "action", "count"):
        assert getattr(t, f) == g["tree"][f], f
    for f in ("value", "prior"):
        assert np.array_equal(np.array(getattr(t, f)), np.array(g["tree"][f])), f
    assert rng_state(rng) == g["rng_state"]


def test_mcts_closed_loop_equals_the_open_loop_oracle():
    """closed_loop=True on a deterministic env: the observation nodes carry their action node's statistics."""
    g = G["closed_loop"]
    from rl_agents_b200.agents.tree_search.mcts import allocation
    episodes, horizon = allocation(g["config"]["budget"], g["config"]["gamma"])
    rng = np_random(g["seed"])
    plan, t = planners.mcts_plan(case_env(g["env"]), episodes, horizon, g["config"]["gamma"], 2 / (1 - 0.8), rng)
    assert plan == g["plan_actions"]             # the reference's plan interleaves the observation keys
    assert [[t.action[c], t.count[c], t.value[c]] for c in t.children(0)] == g["root"]
    assert (t.count[0], t.value[0]) == (g["root_count"], g["root_value"])
    assert rng_state(rng) == g["rng_state"]


def test_mcts_subtree_decisions_match_reference():
    g = G["subtree"]
    env = case_env(g["env"])
    rng = np_random(g["seed"])
    tree = None
    for k in range(3):
        assert env.state.pack().tolist() == g["words"][k]
        plan, t = oracle_mcts(g, rng, env=env, tree=tree)
        assert plan == g["plans"][k], k
        assert canonical(t) == g["trees"][k], k
        env.step(plan[0])
        tree = planners.mcts_reroot(t, plan[0])
    assert rng_state(rng) == g["rng_state"]


@pytest.mark.parametrize("key", sorted(G["olop"]))
def test_olop_oracle_matches_reference(key):
    g = G["olop"][key]
    rng, _ = ref_loader.legacy_np_random(g["seed"])
    if "error" in g:
        # the reference's children[0] KeyError is the oracle's missing child (StopIteration), at the same point
        with pytest.raises(StopIteration):
            oracle_olop(g, rng)
        assert rng_state(rng) == g["rng_state"]
        return
    plan, t = oracle_olop(g, rng)
    assert plan == g["plan"]
    for f in ("parent", "action", "count"):
        assert getattr(t, f) == g["tree"][f], f
    assert [bool(x) for x in t.done] == g["tree"]["done"]
    for f in ("cumulative_reward", "mu_ucb", "upper"):
        assert np.array_equal(np.array(getattr(t, f), dtype=np.float64), np.array(g["tree"][f])), f
    assert rng_state(rng) == g["rng_state"]


def test_receding_horizon_decisions_match_reference():
    """Four agent.plan() calls on one env with receding_horizon 3: one plan served three times, then a new search
    on the planner's continued stream."""
    for key, g in G["agents"].items():
        c = g["config"]
        if key.startswith("mcts"):
            rng = np_random(g["seed"])
            episodes, horizon = planners.olop_allocation(c["budget"], c["gamma"])

            def search():
                return planners.mcts_plan(case_env(g["env"]), episodes, horizon, c["gamma"], 2 / (1 - 0.8), rng)[0]
        else:
            rng, _ = ref_loader.legacy_np_random(g["seed"])

            def search():
                return planners.olop_plan(envs.LegacyStepEnv(case_env(g["env"])), c["budget"], c["gamma"], rng,
                                          upper_bound=c["upper_bound"], continuation_type=c["continuation_type"])[0]
        first = search()
        assert g["decisions"][:3] == [first, first[1:], first[2:]], key
        assert g["decisions"][3] == search(), key
        assert rng_state(rng) == g["rng_state"], key


@pytest.mark.parametrize("seed,episodes,horizon,gamma", [(0, 60, 6, 0.8), (5, 40, 16, 0.9), (7, 120, 4, 0.85)])
@pytest.mark.parametrize("speed_index", [None, 0, 2])
def test_c_mcts_intersection_equals_the_python_oracle(seed, episodes, horizon, gamma, speed_index):
    from oracle import c_mcts_intersection
    from rl_agents_b200.engine.mcts import pcg64_words
    spec = {"seed": seed} if speed_index is None else {"seed": seed, "speed_index": speed_index}
    temperature = 2 / (1 - 0.8)
    rng = np_random(seed + 100)
    words = pcg64_words(rng)
    plan, t = planners.mcts_plan(case_env(spec), episodes, horizon, gamma, temperature, rng)
    d, words_after = c_mcts_intersection.mcts_intersection_plan(case_env(spec).state.pack(), episodes, horizon, gamma,
                                                                temperature, words)
    for f in ("parent", "action", "count", "first_child", "n_children"):
        assert d[f].tolist() == getattr(t, f), f
    assert np.array_equal(d["value"], np.array(t.value)) and np.array_equal(d["prior"], np.array(t.prior))
    assert words_after.tolist() == pcg64_words(rng).tolist()
