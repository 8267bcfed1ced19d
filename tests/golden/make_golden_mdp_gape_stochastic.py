"""Generate tests/golden/golden_mdp_gape_stochastic.json by running the UNMODIFIED reference MDPGapEAgent
(rl_agents/agents/tree_search/mdp_gape.py) on stochastic finite MDPs (tests/mdp_gape_stochastic_cases.py), with the
shims, instrumentation and tree_digest of make_golden_mdp_gape.py; tree_digest covers each chance node's child order.
Also records known answers of the reference's max_expectation_under_constraint (rl_agents/utils.py:292-342) for
lengths 2..15.

Build-container only (the reference tree does not travel to the GPU box); the output is committed and the same bytes
on every run.  Writes only golden_mdp_gape_stochastic.json (or the --out path).
Usage:  python tests/golden/make_golden_mdp_gape_stochastic.py [--out PATH]
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import make_golden_mdp_gape as base  # noqa: E402  (loads the reference and instruments its nodes)
from oracle import ref_loader  # noqa: E402
from tests.mdp_gape_stochastic_cases import oracle_env  # noqa: E402

from rl_agents.utils import max_expectation_under_constraint  # noqa: E402

# (case name, MDP, root state, planner config, planner seed)
CASES = [
    ("garnet30_b2_mdp_gape_json", "garnet30_b2", 0, "mdp-gape.json", 0),
    ("garnet50_K3_b200_uniform", "garnet50", 0, {"budget": 200, "gamma": 0.8, "max_next_states_count": 3}, 1),
    ("garnet50_K3_b1000_zeros", "garnet50", 7, {"budget": 1000, "gamma": 0.8, "max_next_states_count": 3,
                                                 "continuation_type": "zeros"}, 2),
    ("garnet50_K3_b1000_acc3_stop", "garnet50", 3, {"budget": 1000, "gamma": 0.7, "accuracy": 3.0,
                                                     "max_next_states_count": 3}, 3),
    ("garnet50_K3_b2000_acc3.1_zeros_stop", "garnet50", 11, {"budget": 2000, "gamma": 0.7, "accuracy": 3.1,
                                                              "max_next_states_count": 3,
                                                              "continuation_type": "zeros"}, 4),
    ("garnet50_K3_b2000_logtime", "garnet50", 20, {"budget": 2000, "gamma": 0.8, "max_next_states_count": 3,
                                                    "accuracy": 0.5, "confidence": 1.0,
                                                    "upper_bound": {"threshold": "1*np.log(time)"}}, 5),
    ("dense6_K6_b600", "dense6", 0, {"budget": 600, "gamma": 0.8, "max_next_states_count": 6}, 6),
    ("garnet50_K5_b600", "garnet50", 5, {"budget": 600, "gamma": 0.8, "max_next_states_count": 5}, 7),
    ("dup20_K3_b600", "dup20", 0, {"budget": 600, "gamma": 0.8, "max_next_states_count": 3}, 8),
    ("term40_K3_b600_zeros", "term40", 1, {"budget": 600, "gamma": 0.8, "max_next_states_count": 3,
                                            "continuation_type": "zeros"}, 9),
    ("term40_K3_hfa_acc1", "term40", 2, {"budget": 400, "gamma": 0.8, "max_next_states_count": 3,
                                          "horizon_from_accuracy": True, "accuracy": 1.0}, 10),
    ("unreached_bad20_K3_b300", "unreached_bad20", 0, {"budget": 300, "gamma": 0.8, "max_next_states_count": 3}, 11),
]
ERRORS = [
    ("garnet50_K1_placeholders", "garnet50", 0, {"budget": 200, "gamma": 0.8, "max_next_states_count": 1}, 12),
    ("bad20_reached_nan_row", "bad20", 0, {"budget": 300, "gamma": 0.8, "max_next_states_count": 3}, 13),
    ("wide20_rewards", "wide20", 0, {"budget": 300, "gamma": 0.8, "max_next_states_count": 3}, 14),
]


def shipped_config():
    with open(os.path.join(ref_loader.REFERENCE_ROOT, "scripts/configs/DummyEnv/agents/mdp-gape.json")) as f:
        cfg = json.load(f)
    return {k: v for k, v in cfg.items() if k != "__class__"}


def record(mdp, state, config, seed):
    cfg = shipped_config() if config == "mdp-gape.json" else config
    out = base.run(oracle_env(mdp, state), cfg, seed)
    out.update(mdp=mdp, state=state, config_name=config if isinstance(config, str) else None)
    return out


def expectation_vectors():
    """[tag, f, q, c, p] with p = max_expectation_under_constraint(f, q, c): ties, isclose shortcuts, mass moved to
    unobserved entries (theta(f*) < 0) and Newton solves of several iterations, for every length 2..15."""
    rng = np.random.default_rng(23)
    out = []
    for n in range(2, 16):
        for tag in ("newton", "newton_small_c", "unobserved", "ties", "isclose", "all_observed_tied"):
            f = rng.uniform(-2.0, 3.0, size=n)
            counts = rng.integers(1, 6, size=n).astype(float)
            c = float(rng.uniform(0.05, 1.5))
            if tag == "newton_small_c":
                c = float(rng.uniform(1e-4, 1e-2))
            if tag == "unobserved":
                counts[: max(1, n // 2)] = 0
                f[0] = f.max() + 1.0
                c = float(rng.uniform(1.0, 3.0))
            if tag == "ties":
                f = np.round(f * 2) / 2
                counts[rng.integers(0, n)] = 0
            if tag == "isclose":
                f[:] = f[0] + rng.uniform(-1e-9, 1e-9, size=n)
                f[-1] = f[0] + 2e-5 * abs(f[0]) if n % 3 == 0 else f[-1]
            if tag == "all_observed_tied":
                f[:] = f[0]
                counts[0] = 0
                f[0] = f[1] - 1.0
            q = counts / counts.sum()
            out.append([tag, f.tolist(), q.tolist(), c, max_expectation_under_constraint(f, q, c).tolist()])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(HERE, "golden_mdp_gape_stochastic.json"))
    path = ap.parse_args().out
    out = {"cases": {}, "errors": {}}
    for name, mdp, state, cfg, seed in CASES:
        out["cases"][name] = c = record(mdp, state, cfg, seed)
        print(name, c["episodes"], "x", c["horizon"], "->", c["episodes_run"], "plan", c["plan"])
    for name, mdp, state, cfg, seed in ERRORS:
        try:
            record(mdp, state, cfg, seed)
            raise AssertionError("%s was expected to raise" % name)
        except ValueError as e:
            out["errors"][name] = {"mdp": mdp, "state": state, "config": cfg, "seed": seed, "error": "ValueError",
                                   "message": str(e)}
            print(name, "ValueError:", e)
    out["max_expectation_under_constraint"] = expectation_vectors()
    with open(path, "w") as f:
        json.dump(out, f)
    print("mdp_gape_stochastic done")


if __name__ == "__main__":
    main()
