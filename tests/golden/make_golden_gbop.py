"""Generate tests/golden/golden_gbop.json by running the UNMODIFIED reference StateAwarePlannerAgent (GBOP-T,
rl_agents/agents/tree_search/state_aware.py) and GraphBasedPlannerAgent (GBOP-D, graph_based.py) on finite MDPs:
the searches whose backup queues outgrow a fixed multiple of the tree or state count (`loop`), get_plan ties on
quantized rewards, terminal states with a terminal reward, and GBOP-D's tie-heavy sampling on `trap`.

GBOP-D runs at accuracy 0 only: above 0 the reference pushes `list(node.parents)`, a Python set, so its bounds
depend on memory addresses (see the note in golden_finite.json).  The tables of every generated MDP are stored in
the JSON; finite_mdps.npz is only read.  Needs the reference tree (oracle.ref_loader.REFERENCE_ROOT), so the output
is committed and the tests only read it.  Writes only golden_gbop.json, reproducibly byte for byte.
Usage:  python tests/golden/make_golden_gbop.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_loader  # noqa: E402
from oracle import envs  # noqa: E402

ref_loader.load_reference()
from rl_agents.agents.tree_search.state_aware import StateAwarePlannerAgent  # noqa: E402
from rl_agents.agents.tree_search.graph_based import GraphBasedPlannerAgent  # noqa: E402


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def tables(T, R, term):
    return {"T": np.asarray(T).astype(int).tolist(), "R": np.asarray(R, dtype=np.float64).tolist(),
            "term": np.asarray(term).astype(bool).tolist()}


def quantized_mdp(seed, S=6, A=3):
    """S states, A actions, uniform random transitions, rewards in {0, 0.5}: get_plan ties often."""
    rng = np.random.default_rng(seed)
    return tables(rng.integers(0, S, size=(S, A)), rng.choice([0.0, 0.5], size=(S, A)), np.zeros(S, dtype=bool))


def finite(mdp):
    return envs.FiniteMDPLite(mdp["T"], mdp["R"], mdp["term"], mode="deterministic", state=0)


def run_gbopt(mdp_name, mdp, config, seed):
    agent = StateAwarePlannerAgent(finite(mdp), dict(config))
    agent.seed(seed)
    plan = agent.plan(0)
    pl = agent.planner
    return {"mdp": mdp_name, "config": config, "seed": seed, "plan": [int(a) for a in plan],
            "state_values": {str(k): float(v) for k, v in pl.state_values.items()},
            "n_leaves": len(pl.leaves), "n_states": len(pl.state_nodes),
            "leaf_depth_sum": int(sum(leaf.depth for leaf in pl.leaves)),
            "leaf_lower_sum": float(sum(leaf.value_lower for leaf in pl.leaves)),
            "rng_state": rng_state(pl.np_random), "tied": rng_state(pl.np_random) != rng_state(np_random(seed))}


def run_gbopd(mdp_name, mdp, config, seed):
    agent = GraphBasedPlannerAgent(envs.LegacyStepEnv(finite(mdp)), dict(config))
    agent.seed(seed)
    plan = agent.plan(0)
    pl = agent.planner
    return {"mdp": mdp_name, "config": config, "seed": seed, "accuracy": agent.config["accuracy"],
            "sampling_timeout": agent.config["sampling_timeout"], "plan": [int(a) for a in plan],
            "nodes": {str(k): [float(n.value_lower), float(n.value_upper), bool(n.children)]
                      for k, n in sorted(pl.nodes.items())},
            "rng_state": rng_state(pl.np_random)}


def main():
    m = np.load(os.path.join(HERE, "finite_mdps.npz"))
    mdps = {n: tables(m[n + "_T"], m[n + "_R"], m[n + "_term"]) for n in ("loop", "trap")}
    # the first seed whose quantized MDP makes get_plan break a tie at budget 90
    for seed in range(100):
        mdps["quantized6"] = quantized_mdp(seed)
        if run_gbopt("quantized6", mdps["quantized6"], {"budget": 90, "gamma": 0.9}, 3)["tied"]:
            mdps["quantized6"]["seed"] = seed
            break
    term = np.asarray(m["large1_term"]).copy()
    term[[3, 17, 66, 91]] = True
    mdps["large1_term4"] = tables(m["large1_T"], m["large1_R"], term)

    out = {"mdps": mdps, "gbopt": {}, "gbopd": {}, "errors": {}}
    gt = out["gbopt"]
    # one backup of this search pushes more entries than 64 x the node capacity
    gt["loop_b1000_g0.9"] = run_gbopt("loop", mdps["loop"], {"budget": 1000, "gamma": 0.9}, 0)
    gt["quantized6_b90_g0.9"] = run_gbopt("quantized6", mdps["quantized6"], {"budget": 90, "gamma": 0.9}, 3)
    gt["large1_term4_tr0.3_b400_g0.85"] = run_gbopt("large1_term4", mdps["large1_term4"],
                                                    {"budget": 400, "gamma": 0.85, "terminal_reward": 0.3}, 1)
    gd = out["gbopd"]
    # one backup of this search pushes more entries than 256 x the state count
    gd["loop_b500_g0.9_acc0"] = run_gbopd("loop", mdps["loop"], {"budget": 500, "gamma": 0.9, "accuracy": 0}, 0)
    # rewards in [-1, 1] (GBOP-D checks no range) and ties in almost every sampling step
    gd["trap_b500_g0.9_acc0"] = run_gbopd("trap", mdps["trap"], {"budget": 500, "gamma": 0.9, "accuracy": 0}, 0)

    # GBOP-T expands trap's state 4 (rewards -1) and raises
    try:
        run_gbopt("trap", mdps["trap"], {"budget": 100, "gamma": 0.9}, 0)
        raise AssertionError("GBOP-T on trap was expected to raise")
    except ValueError as e:
        out["errors"]["gbopt_trap_b100_g0.9"] = {"error": "ValueError", "message": str(e)}

    for k, c in list(gt.items()) + list(gd.items()):
        print(k, "plan", len(c["plan"]), c["plan"][:12], "rng", c["rng_state"]["state"][:12])
    with open(os.path.join(HERE, "golden_gbop.json"), "w") as f:
        json.dump(out, f)
    print("gbop done")


if __name__ == "__main__":
    main()
