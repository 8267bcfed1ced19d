"""Pin the stochastic MDP-GapE restatement (oracle/mdp_gape_stochastic.py) against
tests/golden/golden_mdp_gape_stochastic.json, recorded from the UNMODIFIED reference by
tests/golden/make_golden_mdp_gape_stochastic.py: trees with their floats, child orders, plans, episodes run and RNG
words bit for bit, the reference's errors, and known answers of max_expectation_under_constraint."""
import filecmp
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import envs, ref_loader
from oracle import mdp_gape as gape
from oracle import mdp_gape_stochastic as sgape
from tests.mdp_gape_stochastic_cases import MDPS, oracle_env
from tests.test_mdp_gape_oracle import completed_planner_config, rng_state
from tests.util import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
G = load_golden("golden_mdp_gape_stochastic.json")


def case_config(g):
    return completed_planner_config(g["config"])


def run_case(g):
    rng = ref_loader.legacy_np_random(g["seed"])[0]
    plan, t, episodes_run = sgape.mdp_gape_plan(envs.LegacyStepEnv(oracle_env(g["mdp"], g["state"])), case_config(g),
                                                rng)
    return plan, t, episodes_run, rng


@pytest.mark.skipif(not ref_loader.reference_available(), reason="needs the reference tree")
def test_golden_generator_reproduces_its_json(tmp_path):
    out = tmp_path / "golden.json"
    subprocess.run([sys.executable, os.path.join(GOLDEN, "make_golden_mdp_gape_stochastic.py"), "--out", str(out)],
                   check=True, cwd=ROOT, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    assert filecmp.cmp(str(out), os.path.join(GOLDEN, "golden_mdp_gape_stochastic.json"), shallow=False)


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_oracle_equals_the_reference_golden_bit_for_bit(key):
    g = G["cases"][key]
    plan, t, episodes_run, rng = run_case(g)
    assert (t.episodes, t.horizon) == (g["episodes"], g["horizon"])
    assert plan == g["plan"] and episodes_run == g["episodes_run"]
    kids = list(t.children(0))
    assert (kids.index(t.best), kids.index(t.challenger)) == (g["best_index"], g["challenger_index"])
    assert rng_state(rng) == g["rng_state"]
    assert gape.tree_digest(gape.tree_dict(t)) == g["tree"]


def test_golden_cases_cover_what_they_are_named_for():
    """Several observed next states per chance node, placeholders left unobserved, early stops and runs to the cap,
    and the shipped mdp-gape.json with its two placeholders."""
    observed = {}
    for key, g in G["cases"].items():
        _, t, episodes_run, _ = run_case(g)
        n_obs = [sum(t.key[c] >= 0 for c in t.children(n)) for n in t.order]
        observed[key] = max(n_obs)
        assert t.key[0] == -1 and all(t.key[n] == -1 for n in t.order)
        if "stop" in key:
            assert episodes_run < g["episodes"] + 2, key
        else:
            assert episodes_run == g["episodes"] + 2, key
    assert all(v >= 2 for v in observed.values()), observed
    assert observed["dense6_K6_b600"] >= 4 and observed["garnet50_K5_b600"] == 3      # placeholders left free
    # four successors per row but at most three distinct ids: K = 3 never overflows
    assert MDPS["dup20"]["next"].shape[-1] == 4 and 2 <= observed["dup20_K3_b600"] <= 3
    assert case_config(G["cases"]["garnet30_b2_mdp_gape_json"])["max_next_states_count"] == 2
    # mdp-gape.json's "threshold_transition" key is a typo: the default transition_threshold stays
    assert case_config(G["cases"]["garnet30_b2_mdp_gape_json"])["upper_bound"]["transition_threshold"] == \
        "0.1*np.log(time)"
    assert MDPS["term40"]["terminal"].any()
    assert any(G["cases"]["term40_K3_b600_zeros"]["tree"]["done"])


@pytest.mark.parametrize("key", sorted(G["errors"]))
def test_oracle_raises_the_reference_errors(key):
    g = G["errors"][key]
    with pytest.raises(ValueError) as e:
        run_case(g)
    assert str(e.value) == g["message"]


def test_max_expectation_under_constraint_known_answers_bit_for_bit():
    tags = set()
    for tag, f, q, c, ref in G["max_expectation_under_constraint"]:
        p = sgape.max_expectation_under_constraint(np.array(f), np.array(q), c)
        assert np.asarray(p, dtype=np.float64).tobytes() == np.array(ref, dtype=np.float64).tobytes(), (tag, len(f))
        tags.add(tag)
    assert len(tags) == 6
    assert {len(v[1]) for v in G["max_expectation_under_constraint"]} == set(range(2, 16))


def test_max_expectation_with_one_positive_entry_is_the_deterministic_restatement():
    for f, q, c, _ in gape_one_positive_vectors():
        a = sgape.max_expectation_under_constraint(np.array(f), np.array(q), c)
        b = gape.max_expectation_one_positive(np.array(f), np.array(q), c)
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()


def gape_one_positive_vectors():
    return load_golden("golden_mdp_gape.json")["max_expectation_one_positive"]


def test_dot_fma_rounds_once():
    # 1 + 2**-60 is not representable: an unfused a * b + c loses it, a fused one keeps it in the sum
    a = 1.0 + 2.0 ** -30
    assert sgape.fma(a, a, -1.0) == 2.0 ** -29 + 2.0 ** -60
    assert a * a - 1.0 != sgape.fma(a, a, -1.0)
    assert sgape.dot_fma([a, 1.0], [a, -1.0]) == sgape.fma(1.0, -1.0, sgape.fma(a, a, 0.0))
