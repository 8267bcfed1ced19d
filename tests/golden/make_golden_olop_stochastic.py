"""Generate tests/golden/golden_olop_stochastic.json by running the UNMODIFIED reference OLOPAgent
(rl_agents/agents/tree_search/olop.py) on stochastic finite MDPs (tests/mdp_gape_stochastic_cases.py), with the shims
and node instrumentation of make_golden.py (oracle.envs.LegacyStepEnv for the 4-tuple `step`,
oracle.ref_loader.legacy_np_random for `np_random.randint`).  Each case records the tree in the digest form of
tests/olop_stochastic_tree.py (SHA-256 of its node arrays in creation order), the plan and the planner's RNG words after
the search.  The shipped FiniteMDPEnv/agents/olop.json, whose "upper_bound" is the bare string "hoeffding", is recorded
as the error the reference raises when the agent is built.

Build-container only (the reference tree does not travel to the GPU box); the output is committed and the same bytes
on every run.  Writes only golden_olop_stochastic.json (or the --out path).
Usage:  python tests/golden/make_golden_olop_stochastic.py [--out PATH]
"""
import argparse
import json
import logging
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import make_golden as base  # noqa: E402  (loads the reference and instruments its nodes)
from oracle import envs, ref_loader  # noqa: E402
from tests.mdp_gape_stochastic_cases import oracle_env  # noqa: E402
from tests.olop_stochastic_tree import tree_digest  # noqa: E402

KL_LOCAL = {"type": "kullback-leibler", "time": "local", "threshold": "2*np.log(time)"}
HOEFFDING = {"type": "hoeffding", "time": "global", "threshold": "4*np.log(time)"}

# (case name, MDP, root state, planner config or shipped config path, planner seed)
CASES = [
    ("garnet30_b2_finite_kl_olop_json", "garnet30_b2", 0, "FiniteMDPEnv/agents/kl-olop.json", 0),
    ("garnet50_finite_kl_olop_json", "garnet50", 0, "FiniteMDPEnv/agents/kl-olop.json", 1),
    ("garnet30_b2_dummy_kl_olop_json", "garnet30_b2", 4, "DummyEnv/agents/kl-olop.json", 2),
    ("garnet50_dummy_kl_olop_json", "garnet50", 7, "DummyEnv/agents/kl-olop.json", 3),
    ("garnet50_b300_uniform_local", "garnet50", 11, {"budget": 300, "gamma": 0.8, "continuation_type": "uniform",
                                                     "upper_bound": KL_LOCAL}, 4),
    ("garnet50_b300_zeros_local", "garnet50", 12, {"budget": 300, "gamma": 0.8, "continuation_type": "zeros",
                                                   "upper_bound": KL_LOCAL}, 5),
    ("garnet50_b200_hoeffding_uniform", "garnet50", 3, {"budget": 200, "gamma": 0.8, "continuation_type": "uniform",
                                                        "upper_bound": HOEFFDING}, 6),
    ("garnet50_b2000_g0.8_uniform", "garnet50", 20, {"budget": 2000, "gamma": 0.8, "continuation_type": "uniform",
                                                     "upper_bound": {"type": "kullback-leibler"}}, 7),
    ("dense6_b400_uniform", "dense6", 0, {"budget": 400, "gamma": 0.8, "continuation_type": "uniform",
                                          "upper_bound": {"type": "kullback-leibler"}}, 8),
    ("dup20_b400_uniform_local", "dup20", 0, {"budget": 400, "gamma": 0.8, "continuation_type": "uniform",
                                              "upper_bound": KL_LOCAL}, 9),
    ("term40_b600_zeros", "term40", 1, {"budget": 600, "gamma": 0.9, "continuation_type": "zeros",
                                        "upper_bound": {"type": "kullback-leibler"}}, 10),
    ("term40_b400_uniform", "term40", 0, {"budget": 400, "gamma": 0.8, "continuation_type": "uniform",
                                          "upper_bound": {"type": "kullback-leibler"}}, 11),
    ("unreached_bad20_b300_uniform", "unreached_bad20", 0, {"budget": 300, "gamma": 0.8,
                                                            "continuation_type": "uniform",
                                                            "upper_bound": {"type": "kullback-leibler"}}, 12),
]
ERRORS = [
    ("bad20_reached_nan_row", "bad20", 0, {"budget": 300, "gamma": 0.8, "continuation_type": "uniform",
                                           "upper_bound": {"type": "kullback-leibler"}}, 13),
    ("wide20_rewards", "wide20", 0, {"budget": 300, "gamma": 0.8, "continuation_type": "uniform",
                                     "upper_bound": {"type": "kullback-leibler"}}, 14),
    ("garnet50_finite_olop_json", "garnet50", 0, "FiniteMDPEnv/agents/olop.json", 15),
]


def shipped_config(path):
    with open(os.path.join(ref_loader.REFERENCE_ROOT, "scripts/configs", path)) as f:
        cfg = json.load(f)
    return {k: v for k, v in cfg.items() if k != "__class__"}


def run(env, config, seed):
    """make_golden.run_olop, plus the planner's RNG words after the search."""
    del base.CREATED[:]
    agent = base.ref_olop.OLOPAgent(envs.LegacyStepEnv(env), json.loads(json.dumps(config)))
    agent.planner.np_random, _ = ref_loader.legacy_np_random(seed)
    plan = agent.plan(None)
    pl = agent.planner
    for n in base.CREATED:
        n.upper = n.value_upper
    tree = base.dump_tree(["cumulative_reward", "mu_ucb", "upper", "done"], pl.root)
    st = pl.np_random.bit_generator.state
    return {"config": config, "seed": seed, "plan": [int(a) for a in plan],
            "episodes": int(pl.config["episodes"]), "horizon": int(pl.config["horizon"]),
            "completed_upper_bound": pl.config["upper_bound"],
            "continuation_type": pl.config["continuation_type"], "gamma": pl.config["gamma"],
            "rng_state": {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
                          "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])},
            "tree": tree_digest(tree)}


def record(mdp, state, config, seed):
    cfg = shipped_config(config) if isinstance(config, str) else config
    out = run(oracle_env(mdp, state), cfg, seed)
    out.update(mdp=mdp, state=state, config_name=config if isinstance(config, str) else None)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(HERE, "golden_olop_stochastic.json"))
    path = ap.parse_args().out
    # the hoeffding bound logs "Unknown upper-bound type" at every node update (olop.py:162-163)
    logging.getLogger(base.ref_olop.__name__).setLevel(logging.CRITICAL)
    out = {"cases": {}, "errors": {}}
    for name, mdp, state, cfg, seed in CASES:
        out["cases"][name] = c = record(mdp, state, cfg, seed)
        print(name, c["episodes"], "x", c["horizon"], "nodes", c["tree"]["n_nodes"], "plan", c["plan"])
    for name, mdp, state, cfg, seed in ERRORS:
        try:
            record(mdp, state, cfg, seed)
            raise AssertionError("%s was expected to raise" % name)
        except (ValueError, TypeError) as e:
            out["errors"][name] = {"mdp": mdp, "state": state, "seed": seed,
                                   "config": shipped_config(cfg) if isinstance(cfg, str) else cfg,
                                   "config_name": cfg if isinstance(cfg, str) else None,
                                   "error": type(e).__name__, "message": str(e)}
            print(name, type(e).__name__ + ":", e)
    with open(path, "w") as f:
        json.dump(out, f)
    print("olop_stochastic done")


if __name__ == "__main__":
    main()
