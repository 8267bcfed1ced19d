"""Pin MCTS's restatement (oracle/planners.py::mcts_plan) on stochastic finite MDPs against
tests/golden/golden_mcts_stochastic.json, recorded from the UNMODIFIED reference by
tests/golden/make_golden_mcts_stochastic.py: trees with their floats (through the digests of
tests/mcts_stochastic_cases.py), plans, planner RNG words and the reference's error bit for bit, with the live env's
generator unchanged by planning.  The reference never reseeds its env copies, so every episode replays that generator."""
import filecmp
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import planners, ref_loader
from tests.mcts_stochastic_cases import (CASES, CLOSED_LOOP, ERRORS, MDPS, SUBTREE, canonical_digest, live_env,
                                         planner_rng, policy, rng_state, tree_digest)
from tests.util import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
G = load_golden("golden_mcts_stochastic.json")


def case_of(g):
    return (g["mdp"], g["state"], g["config"], g["seed"], g["env_seed"], g["advance"])


def oracle_plan(env, g, rng, tree=None):
    cfg = g["config"]
    return planners.mcts_plan(env, g["episodes"], g["horizon"], g["gamma"], g["temperature"], rng,
                              prior_policy=policy(cfg, "prior_policy"), rollout_policy=policy(cfg, "rollout_policy"),
                              tree=tree)


def oracle_tree_dict(t):
    return {"parent": t.parent, "action": t.action, "count": t.count, "value": t.value, "prior": t.prior}


def run_case(g):
    """mcts_plan on the case's live env -> (plan, tree, planner generator after, env generator before)."""
    env = live_env(case_of(g))
    before = rng_state(env.np_random)
    rng = planner_rng(g["seed"])
    plan, t = oracle_plan(env, g, rng)
    assert rng_state(env.np_random) == before
    return plan, t, rng, before


@pytest.mark.skipif(not ref_loader.reference_available(), reason="needs the reference tree")
def test_golden_generator_reproduces_its_json(tmp_path):
    out = tmp_path / "golden.json"
    subprocess.run([sys.executable, os.path.join(GOLDEN, "make_golden_mcts_stochastic.py"), "--out", str(out)],
                   check=True, cwd=ROOT, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    assert filecmp.cmp(str(out), os.path.join(GOLDEN, "golden_mcts_stochastic.json"), shallow=False)


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_oracle_equals_the_reference_golden_bit_for_bit(key):
    g = G["cases"][key]
    plan, t, rng, before = run_case(g)
    assert before == g["env_rng_state"]
    assert plan == g["plan"]
    assert rng_state(rng) == g["rng_state"]
    assert tree_digest(oracle_tree_dict(t)) == g["tree"]


@pytest.mark.parametrize("key", sorted(G["closed_loop"]))
def test_closed_loop_projection_equals_the_open_loop_oracle(key):
    """closed_loop: True in the reference: one observation child per action node, and with those taken out the tree
    is the open-loop tree, node for node."""
    g = G["closed_loop"][key]
    assert g["config"]["closed_loop"] and g["n_observation_nodes"] > 0
    plan, t, rng, before = run_case(g)
    assert before == g["env_rng_state"]
    # the reference's plan interleaves the observation keys (the last action may have none)
    assert plan == g["plan_actions"] and g["plan_len"] in (2 * len(plan) - 1, 2 * len(plan))
    assert rng_state(rng) == g["rng_state"]
    assert tree_digest(oracle_tree_dict(t)) == g["tree"]


@pytest.mark.parametrize("key", sorted(G["subtree"]))
def test_subtree_over_two_decisions(key):
    g = G["subtree"][key]
    env = live_env(case_of(g))
    rng = planner_rng(g["seed"])
    tree = None
    for k, d in enumerate(g["decisions"]):
        assert (int(env.mdp.state), rng_state(env.np_random)) == (d["state"], d["env_rng_state"])
        plan, tree = oracle_plan(env, dict(d, config=g["config"]), rng, tree=tree)
        assert rng_state(env.np_random) == d["env_rng_state"]
        assert plan == d["plan"] and rng_state(rng) == d["rng_state"], k
        assert canonical_digest(tree.first_child, tree.n_children, tree.action, tree.count, tree.value,
                                tree.prior) == d["tree"], k
        env.step(plan[0])
        tree = planners.mcts_reroot(tree, plan[0])
    # the real step between the decisions moved the env generator: the second decision replays another stream
    assert g["decisions"][0]["env_rng_state"] != g["decisions"][1]["env_rng_state"]


def test_golden_cases_cover_what_they_are_named_for():
    C = G["cases"]
    assert MDPS["dense6"]["mode"] == "stochastic" and {MDPS[c["mdp"]]["mode"] for c in C.values()} == {"stochastic",
                                                                                                     "sparse"}
    assert {c["mdp"] for c in C.values()} >= {"dense6", "garnet50", "dup20", "term40", "unreached_bad20"}
    kinds = {policy(c["config"], k)["type"] for c in C.values() for k in ("prior_policy", "rollout_policy")}
    assert kinds == {"random_available", "random", "preference"}
    big = C["garnet50_b2000_g0.9"]
    assert big["gamma"] == 0.9 and big["episodes"] * big["horizon"] >= 1900
    assert any(c["advance"] > 0 for c in C.values())
    assert MDPS["term40"]["terminal"].any()
    assert np.isnan(MDPS["unreached_bad20"]["transition"]).any()


@pytest.mark.parametrize("key", sorted(G["errors"]))
def test_oracle_raises_the_reference_error(key):
    g = G["errors"][key]
    env = live_env(case_of(g))
    cfg = G["cases"]["unreached_bad20_b300_g0.8"]        # the same budget and gamma: the same allocation
    assert (cfg["config"]["budget"], cfg["config"]["gamma"]) == (g["config"]["budget"], g["config"]["gamma"])
    with pytest.raises(ValueError) as e:
        planners.mcts_plan(env, cfg["episodes"], cfg["horizon"], cfg["gamma"], cfg["temperature"],
                           planner_rng(g["seed"]))
    assert str(e.value) == g["message"]
