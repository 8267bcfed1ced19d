"""Pin OLOP's restatement (oracle/planners.py::olop_plan) on stochastic finite MDPs against
tests/golden/golden_olop_stochastic.json, recorded from the UNMODIFIED reference by
tests/golden/make_golden_olop_stochastic.py: trees with their floats (through the digests of
tests/olop_stochastic_tree.py), plans and RNG words bit for bit, and the reference's errors, the TypeError of the
shipped olop.json included."""
import filecmp
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import envs, planners, ref_loader
from tests.mdp_gape_stochastic_cases import MDPS, oracle_env, product_env
from tests.test_mdp_gape_oracle import rng_state
from tests.olop_stochastic_tree import tree_digest
from tests.util import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
G = load_golden("golden_olop_stochastic.json")


def completed_config(config):
    """The planner config the agent builds from `config` (OLOP.default_config updated recursively)."""
    import json
    from rl_agents_b200.agents.tree_search.olop import OLOP
    cfg = OLOP.default_config()
    OLOP.rec_update(cfg, json.loads(json.dumps(config)))
    return cfg


def oracle_run(env, cfg, seed):
    """olop_plan on `env` (an oracle FiniteMDPLite) from the planner seed -> (plan, tree, generator after)."""
    rng = ref_loader.legacy_np_random(seed)[0]
    plan, t = planners.olop_plan(envs.LegacyStepEnv(env), cfg["budget"], cfg["gamma"], rng,
                                 upper_bound=cfg["upper_bound"], continuation_type=cfg["continuation_type"])
    return plan, t, rng


def oracle_tree_dict(t):
    return {"parent": t.parent, "action": t.action, "count": t.count, "cumulative_reward": t.cumulative_reward,
            "mu_ucb": t.mu_ucb, "upper": t.upper, "done": t.done}


def run_case(g):
    return oracle_run(oracle_env(g["mdp"], g["state"]), completed_config(g["config"]), g["seed"])


@pytest.mark.skipif(not ref_loader.reference_available(), reason="needs the reference tree")
def test_golden_generator_reproduces_its_json(tmp_path):
    out = tmp_path / "golden.json"
    subprocess.run([sys.executable, os.path.join(GOLDEN, "make_golden_olop_stochastic.py"), "--out", str(out)],
                   check=True, cwd=ROOT, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    assert filecmp.cmp(str(out), os.path.join(GOLDEN, "golden_olop_stochastic.json"), shallow=False)


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_oracle_equals_the_reference_golden_bit_for_bit(key):
    g = G["cases"][key]
    cfg = completed_config(g["config"])
    assert cfg["upper_bound"] == g["completed_upper_bound"] and cfg["continuation_type"] == g["continuation_type"]
    plan, t, rng = run_case(g)
    assert (t.episodes, t.horizon) == (g["episodes"], g["horizon"])
    assert plan == g["plan"]
    assert rng_state(rng) == g["rng_state"]
    assert tree_digest(oracle_tree_dict(t)) == g["tree"]


def test_golden_cases_cover_what_they_are_named_for():
    C = G["cases"]
    shipped = {c["config_name"] for c in C.values() if c["config_name"]}
    assert shipped == {"FiniteMDPEnv/agents/kl-olop.json", "DummyEnv/agents/kl-olop.json"}
    assert {c["mdp"] for c in C.values() if c["config_name"]} == {"garnet30_b2", "garnet50"}
    assert {c["continuation_type"] for c in C.values()} == {"zeros", "uniform"}
    assert {c["completed_upper_bound"]["time"] for c in C.values()} == {"local", "global"}
    # the hoeffding bound is not implemented by the reference: mu_ucb stays infinite everywhere
    h = C["garnet50_b200_hoeffding_uniform"]
    assert h["completed_upper_bound"]["type"] == "hoeffding" and np.isinf(h["tree"]["sum_mu_ucb"])
    assert all(np.isinf(run_case(h)[1].mu_ucb))
    big = C["garnet50_b2000_g0.8_uniform"]
    assert big["gamma"] == 0.8 and big["episodes"] * big["horizon"] >= 1900
    assert MDPS["dense6"]["mode"] == "stochastic" and {c["mdp"] for c in C.values()} >= {"dense6", "dup20",
                                                                                         "term40", "unreached_bad20"}
    # terminal states: done nodes, and nodes below a done node still counted (the episode steps on after done)
    for key in ("term40_b600_zeros", "term40_b400_uniform"):
        t = run_case(C[key])[1]
        done = [i for i, d in enumerate(t.done) if d]
        assert done and any(t.parent[i] in done and t.count[i] > 0 for i in range(len(t.parent))), key
    assert np.isnan(MDPS["unreached_bad20"]["transition"]).any()


@pytest.mark.parametrize("key", sorted(G["errors"]))
def test_oracle_raises_the_reference_errors(key):
    g = G["errors"][key]
    if g["error"] == "TypeError":
        # the shipped olop.json: "upper_bound" is the bare string "hoeffding", and the agent raises when it is built
        from rl_agents_b200.agents.tree_search.olop import OLOPAgent
        assert g["config"]["upper_bound"] == "hoeffding"
        with pytest.raises(TypeError) as e:
            OLOPAgent(product_env(g["mdp"], g["state"]), dict(g["config"]))
        assert str(e.value) == g["message"]
        return
    with pytest.raises(ValueError) as e:
        oracle_run(oracle_env(g["mdp"], g["state"]), completed_config(g["config"]), g["seed"])
    assert str(e.value) == g["message"]
