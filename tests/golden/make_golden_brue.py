"""Generate tests/golden/golden_brue.json by running the UNMODIFIED reference BRUEAgent
(rl_agents/agents/tree_search/brue.py) on the oracle env models, through the same shims as the OLOP and MDP-GapE
goldens (oracle.envs.LegacyStepEnv for the 4-tuple `step`, oracle.ref_loader.legacy_np_random for
`np_random.randint`).

Needs the reference tree (oracle.ref_loader.REFERENCE_ROOT), so the output is committed and the tests only read it.
Writes only golden_brue.json, reproducibly byte for byte.  Usage:  python tests/golden/make_golden_brue.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_loader  # noqa: E402
from oracle import envs  # noqa: E402
from oracle.brue import tree_digest  # noqa: E402

ref_loader.load_reference()
from rl_agents.agents.tree_search import brue as ref_brue  # noqa: E402

CREATED = []
ROLLOUTS = [0]


def _instrument(cls):
    """Record node creation order at run time (sources stay unmodified)."""
    orig = cls.__init__

    def init(self, *a, **k):
        orig(self, *a, **k)
        CREATED.append(self)
    cls.__init__ = init


for _cls in (ref_brue.DecisionNode, ref_brue.ChanceNode):
    _instrument(_cls)
_orig_rollout = ref_brue.BRUE.rollout


def _counted_rollout(self, *a, **k):
    ROLLOUTS[0] += 1
    return _orig_rollout(self, *a, **k)


ref_brue.BRUE.rollout = _counted_rollout


def dump_tree(root):
    """Creation-order dump: a chance node's action is its key in the parent; decision nodes carry action -1 and
    their mean reward as `value`.  Every node's children must be in creation order (dict insertion order)."""
    def top(n):
        while n.parent is not None:
            n = n.parent
        return n
    nodes = [n for n in CREATED if top(n) is root]
    assert nodes[0] is root
    ids = {id(n): i for i, n in enumerate(nodes)}
    out = {k: [] for k in ("parent", "action", "kind", "depth", "count", "value")}
    for n in nodes:
        chance = isinstance(n, ref_brue.ChanceNode)
        p = n.parent
        out["parent"].append(ids[id(p)] if p is not None else -1)
        out["action"].append(int(next(k for k, c in p.children.items() if c is n)) if chance else -1)
        out["kind"].append(1 if chance else 0)
        out["depth"].append(int(n.depth))
        out["count"].append(int(n.count))
        out["value"].append(float(n.value if chance else n.reward))
        kids = [ids[id(c)] for c in n.children.values()]
        assert kids == sorted(kids)
        assert not chance or len(kids) <= 1           # deterministic env models: one observed next state
    return out


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def make_env(spec, m):
    """The env a case runs on: {"name": "highway", "seed": s} or a finite MDP of finite_mdps.npz, optionally with
    zero rewards, rooted at `state`."""
    if spec["name"] == "highway":
        return envs.HighwayLite(seed=spec["seed"])
    n = spec["name"]
    reward = np.zeros_like(m[n + "_R"]) if spec.get("zero_rewards") else m[n + "_R"]
    return envs.FiniteMDPLite(m[n + "_T"], reward, m[n + "_term"], mode="deterministic", state=spec.get("state", 0))


def run(m, spec, config, seed=0, decisions=1):
    del CREATED[:]
    ROLLOUTS[0] = 0
    agent = ref_brue.BRUEAgent(envs.LegacyStepEnv(make_env(spec, m)), dict(config))
    agent.planner.np_random, _ = ref_loader.legacy_np_random(seed)
    plans = []
    for _ in range(decisions):
        del CREATED[:]
        ROLLOUTS[0] = 0
        plans.append([int(a) for a in agent.plan(None)])
    pl = agent.planner
    out = {"env": spec, "config": config, "seed": seed, "horizon": int(pl.config["horizon"]),
           "plan": plans[-1], "rollouts": ROLLOUTS[0], "budget_left": int(pl.available_budget),
           "rng_state": rng_state(pl.np_random), "tree": tree_digest(dump_tree(pl.root))}
    if decisions > 1:
        out["plans"] = plans
    return out


def main():
    m = np.load(os.path.join(HERE, "finite_mdps.npz"))
    with open(os.path.join(ref_loader.REFERENCE_ROOT, "scripts/configs/DummyEnv/agents/brue.json")) as f:
        brue_json = json.load(f)
    shipped = {k: v for k, v in brue_json.items() if k != "__class__"}     # gamma 0.7, budget 200, horizon 6
    large1 = {"name": "large1"}
    trap_terminal = int(np.nonzero(m["trap_term"])[0][0])

    out = {"cases": {}, "configs": {}, "errors": {}}
    cases = out["cases"]
    cases["large1_brue_json"] = run(m, large1, shipped)
    cases["large1_b200_g0.7_allocated"] = run(m, large1, {"budget": 200, "gamma": 0.7}, seed=1)
    cases["large2_b400_g0.8"] = run(m, {"name": "large2"}, {"budget": 400, "gamma": 0.8}, seed=2)
    # BRUE checks no reward range: the trap MDP plans with its raw [-1, 1] rewards
    cases["trap_raw_b300_g0.8"] = run(m, {"name": "trap"}, {"budget": 300, "gamma": 0.8}, seed=3)
    # rooted at a terminal state: done on the first step, every rollout is one step long
    cases["trap_terminal_root_b50_g0.8"] = run(m, {"name": "trap", "state": trap_terminal},
                                               {"budget": 50, "gamma": 0.8}, seed=4)
    # all rewards zero: every root value ties and get_plan draws choice(indices)
    cases["large1_zero_rewards_b50_g0.8"] = run(m, {"name": "large1", "zero_rewards": True},
                                                {"budget": 50, "gamma": 0.8}, seed=5)
    cases["loop_b200_g0.9"] = run(m, {"name": "loop"}, {"budget": 200, "gamma": 0.9}, seed=6)
    cases["hw0_brue_json"] = run(m, {"name": "highway", "seed": 0}, shipped)
    cases["hw1_brue_json"] = run(m, {"name": "highway", "seed": 1}, shipped, seed=7)
    cases["hw2_b500_g0.7"] = run(m, {"name": "highway", "seed": 2}, {"budget": 500, "gamma": 0.7}, seed=8)
    cases["hw3_b2000_g0.8"] = run(m, {"name": "highway", "seed": 3}, {"budget": 2000, "gamma": 0.8}, seed=9)
    # three consecutive decisions of one agent: a one-action plan is replanned at every call
    cases["large1_receding3_three_decisions"] = run(m, large1, {"budget": 100, "gamma": 0.8, "receding_horizon": 3},
                                                    seed=10, decisions=3)
    for k, c in cases.items():
        print(k, "horizon", c["horizon"], "rollouts", c["rollouts"], "left", c["budget_left"], "plan", c["plan"],
              "nodes", c["tree"]["n_nodes"])

    # budget <= 0 runs no rollout; get_plan's np.amax of the empty root values raises
    agent = ref_brue.BRUEAgent(envs.LegacyStepEnv(make_env(large1, m)), {"budget": 0, "gamma": 0.8})
    try:
        agent.plan(None)
        raise AssertionError("budget 0 was expected to raise")
    except ValueError as e:
        out["errors"]["budget_zero"] = {"error": "ValueError", "message": str(e)}

    # completed configs of the agent, as agent_factory builds it (the `__class__` key is left in)
    evaluation_entry = {"__class__": "<class 'rl_agents.agents.tree_search.brue.BRUEAgent'>", "gamma": 0.7,
                        "step_strategy": "reset"}          # scripts/planners_evaluation.py:90-94 (gamma = 0.7, :40)
    for name, cfg in (("empty", {}), ("brue_json", brue_json), ("planners_evaluation", evaluation_entry)):
        agent = ref_brue.BRUEAgent(make_env(large1, m), json.loads(json.dumps(cfg)))
        completed = {k: v for k, v in agent.config.items() if k != "__class__"}
        out["configs"][name] = {"config": cfg, "completed": json.loads(json.dumps(completed))}
    with open(os.path.join(HERE, "golden_brue.json"), "w") as f:
        json.dump(out, f)
    print("brue done")


if __name__ == "__main__":
    main()
