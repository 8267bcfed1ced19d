"""Generate tests/golden/golden_mdp_gape.json by running the UNMODIFIED reference MDPGapEAgent
(rl_agents/agents/tree_search/mdp_gape.py) on the oracle env models, through the same shims as the OLOP
goldens (oracle.envs.LegacyStepEnv for the 4-tuple `step`, oracle.ref_loader.legacy_np_random for
`np_random.randint`).

Build-container only (the reference tree does not travel to the GPU box); the output is committed.  Writes only
golden_mdp_gape.json.  Usage:  python tests/golden/make_golden_mdp_gape.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_loader  # noqa: E402
from oracle import envs  # noqa: E402
from oracle.mdp_gape import tree_digest  # noqa: E402

ref_loader.load_reference()
from rl_agents.agents.tree_search import mdp_gape as ref_gape  # noqa: E402

CREATED = []


def _instrument(cls):
    """Record node creation order at run time (sources stay unmodified)."""
    orig = cls.__init__

    def init(self, *a, **k):
        orig(self, *a, **k)
        CREATED.append(self)
    cls.__init__ = init


for _cls in (ref_gape.DecisionNode, ref_gape.ChanceNode):
    _instrument(_cls)


def dump_tree(root):
    """Creation-order dump.  Chance nodes are keyed by action in their parent; decision nodes below a chance node
    are keyed by "placeholder_<i>" until an observation takes them over, so their `action` is the placeholder
    index (their rank among the siblings, which are created in index order).  `order` lists the children of every
    chance node in the final dict order."""
    def top(n):
        while n.parent is not None:
            n = n.parent
        return n
    nodes = [n for n in CREATED if top(n) is root]
    assert nodes[0] is root
    ids = {id(n): i for i, n in enumerate(nodes)}
    out = {k: [] for k in ("parent", "action", "kind", "depth", "count", "done", "cumulative_reward", "mu_ucb",
                           "mu_lcb", "upper", "lower")}
    out["order"] = {}
    for n in nodes:
        chance = isinstance(n, ref_gape.ChanceNode)
        p = n.parent
        out["parent"].append(ids[id(p)] if p is not None else -1)
        act = -1
        if p is not None:
            for k, c in p.children.items():
                if c is n:
                    if chance:
                        act = int(k)
                    else:
                        siblings = sorted(ids[id(s)] for s in p.children.values())
                        act = siblings.index(ids[id(n)])
        out["action"].append(act)
        out["kind"].append(1 if chance else 0)
        out["depth"].append(int(n.depth))
        out["count"].append(int(n.count))
        out["done"].append(bool(n.done))
        for f in ("cumulative_reward", "mu_ucb", "mu_lcb"):
            out[f].append(None if chance else float(getattr(n, f)))
        out["upper"].append(float(n.value_upper))
        out["lower"].append(float(n.value_lower))
        if chance and n.children:
            out["order"][str(ids[id(n)])] = [ids[id(c)] for c in n.children.values()]
    return out


def run(env, config, seed=0):
    del CREATED[:]
    agent = ref_gape.MDPGapEAgent(envs.LegacyStepEnv(env), dict(config))
    agent.planner.np_random, _ = ref_loader.legacy_np_random(seed)
    plan = agent.plan(None)
    pl = agent.planner
    episodes_run = pl.budget_used // pl.config["horizon"]
    _, best, challenger = pl.root.best_arm_identification_selection()
    children = list(pl.root.children.values())
    st = pl.np_random.bit_generator.state
    return {"config": config, "seed": seed, "plan": [int(a) for a in plan],
            "episodes": int(pl.config["episodes"]), "horizon": int(pl.config["horizon"]),
            "episodes_run": int(episodes_run), "budget_used": int(pl.budget_used),
            "best_action": int(next(best.path())), "challenger_action": int(next(challenger.path())),
            "best_index": children.index(best), "challenger_index": children.index(challenger),
            "rng_state": {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
                          "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])},
            "tree": tree_digest(dump_tree(pl.root))}


def main():
    m = np.load(os.path.join(HERE, "finite_mdps.npz"))

    def finite(name="large1"):
        return envs.FiniteMDPLite(m[name + "_T"], m[name + "_R"], m[name + "_term"], mode="deterministic", state=0)

    with open(os.path.join(ref_loader.REFERENCE_ROOT,
                           "scripts/configs/HighwayEnv/agents/MDPGapEAgent/baseline.json")) as f:
        baseline = json.load(f)
    baseline_run = {k: v for k, v in baseline.items() if k not in ("__class__", "env_preprocessors")}
    log_time = {"type": "kullback-leibler", "time": "global", "threshold": "1*np.log(time)"}

    out = {"cases": {}, "configs": {}}
    cases = out["cases"]
    # finite MDPs (finite_mdps.npz): run-to-cap and early-stopping cases
    cases["large1_b200_g0.8_default"] = run(finite(), {"budget": 200, "gamma": 0.8})
    cases["large1_b200_g0.8_K3"] = run(finite(), {"budget": 200, "gamma": 0.8, "max_next_states_count": 3})
    cases["large1_b2000_g0.7_acc3_stop"] = run(finite(), {"budget": 2000, "gamma": 0.7, "accuracy": 3.0})
    cases["large1_b2000_g0.7_acc3_K3_zeros_stop"] = run(
        finite(), {"budget": 2000, "gamma": 0.7, "accuracy": 3.0, "max_next_states_count": 3,
                   "continuation_type": "zeros"}, seed=1)
    # the trap MDP's rewards lie in [-1, 1]: the reference raises; mapped to [0, 1] by (r + 1) / 2 it exercises
    # terminal states (done nodes count rewards as 0)
    trap_cfg = {"budget": 300, "gamma": 0.8, "continuation_type": "zeros", "max_next_states_count": 3}
    try:
        run(finite("trap"), trap_cfg, seed=2)
        raise AssertionError("the trap MDP's raw rewards were expected to raise")
    except ValueError as e:
        out["errors"] = {"trap_raw_rewards": {"config": trap_cfg, "seed": 2, "error": "ValueError", "message": str(e)}}
    trap01 = envs.FiniteMDPLite(m["trap_T"], (m["trap_R"] + 1) / 2, m["trap_term"], mode="deterministic", state=0)
    cases["trap01_b300_g0.8_zeros_K3"] = run(trap01, trap_cfg, seed=2)
    cases["large2_b400_g0.8_logtime"] = run(finite("large2"), {"budget": 400, "gamma": 0.8, "upper_bound": log_time},
                                            seed=3)
    cases["large1_hfa_acc1_b200_g0.8"] = run(
        finite(), {"budget": 200, "gamma": 0.8, "horizon_from_accuracy": True, "accuracy": 1.0}, seed=4)
    # HighwayLite scenes: the shipped baseline.json, early stopping, run to the cap, K = 3 / zeros
    cases["hw0_baseline"] = run(envs.HighwayLite(seed=0), baseline_run)
    cases["hw1_b1000_g0.7_acc2_stop"] = run(envs.HighwayLite(seed=1), dict(baseline_run, budget=1000, gamma=0.7,
                                                                           accuracy=2.0))
    cases["hw1_b1000_g0.7_acc0.5_cap"] = run(envs.HighwayLite(seed=1), dict(baseline_run, budget=1000, gamma=0.7,
                                                                            accuracy=0.5))
    cases["hw2_b300_g0.8_K3_zeros_default"] = run(
        envs.HighwayLite(seed=2), {"budget": 300, "gamma": 0.8, "max_next_states_count": 3,
                                   "continuation_type": "zeros"}, seed=5)
    cases["hw3_hfa_acc2_b300_g0.7_K3"] = run(
        envs.HighwayLite(seed=3), dict(baseline_run, budget=300, gamma=0.7, accuracy=2.0, horizon_from_accuracy=True,
                                       max_next_states_count=3), seed=6)
    for k, c in cases.items():
        print(k, c["episodes"], "x", c["horizon"], "->", c["episodes_run"], "plan", c["plan"])

    # completed configs of the agent, as agent_factory builds it (the `__class__` key is left in)
    env = finite()
    for name, cfg in (("empty", {}), ("baseline", baseline),
                      ("hfa", {"budget": 200, "gamma": 0.8, "horizon_from_accuracy": True, "accuracy": 1.0})):
        agent = ref_gape.MDPGapEAgent(env, json.loads(json.dumps(cfg)))
        completed = {k: v for k, v in agent.config.items() if k != "__class__"}
        out["configs"][name] = {"config": cfg, "completed": json.loads(json.dumps(completed))}

    # max_expectation_under_constraint with one positive entry of q, straight from the reference
    from rl_agents.utils import max_expectation_under_constraint
    rng = np.random.default_rng(11)
    mec = []
    for k in range(24):
        n = 1 + k % 4
        f = rng.uniform(-2, 3, size=n)
        if k % 5 == 0:
            f[:-1] = f[-1]
        q = np.zeros(n)
        q[-1] = 1.0
        c = float(rng.uniform(0.0, 2.0))
        mec.append([f.tolist(), q.tolist(), c, max_expectation_under_constraint(f, q, c).tolist()])
    out["max_expectation_one_positive"] = mec
    from rl_agents.utils import kl_upper_bound
    out["kl_lower_bound"] = [[s, c, th, float(kl_upper_bound(s, c, th, lower=True))]
                             for s, c, th in [(0.5, 1, 2.0), (3.25, 7, 5.5), (0, 4, 3.0), (4, 4, 3.0), (17.5, 40, 9.2)]]
    with open(os.path.join(HERE, "golden_mdp_gape.json"), "w") as f:
        json.dump(out, f)
    print("mdp_gape done")


if __name__ == "__main__":
    main()
