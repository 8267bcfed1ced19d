"""Generate tests/golden/golden_drop_intersection.json by running the UNMODIFIED reference DiscreteRobustPlannerAgent
(rl_agents/agents/robust/robust.py, DROP) on IntersectionLite route hypotheses.

The true env is oracle.intersection_routes.IntersectionLiteRoutes, so the reference's own preprocess_env builds each
model from the config's `models` chains through `set_route_at_intersection` (a `change_vehicles` entry is skipped with
the reference's warning).  The reference's JointEnv.step returns the legacy 4-tuple, which its DeterministicNode.expand
cannot unpack: JointEnv is swapped for the 5-tuple re-pack shim make_golden.py uses for "drop", and nothing else.
Node creation order is recorded by make_golden.py's instrumentation.

Per case: the root scene's 136 words, the config, the planner seed, the plan, the PCG64 state after the decision,
and every node in creation order (parent, action, count, and the little-endian float64 bytes, in hex, of the
minima over the models of value_lower / value_upper).  Cases: routes_behaviours.json verbatim (budget 20, gamma
0.9) on three scenes; M = 2 and M = 3 at budgets 200 and 600; "random" hypotheses; terminal_reward > 0; roots with
only two actions (speed index 0 and 2); scenes of tests/intersection_scenes.py families where a crash or an arrival
is reached inside the tree; a root at t = 12.

Needs the reference tree (oracle.ref_loader.REFERENCE_ROOT), so the output is committed and the tests only read it.
Writes only golden_drop_intersection.json (or --out PATH), reproducibly byte for byte.
Usage:  python tests/golden/make_golden_drop_intersection.py [--out PATH]
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import make_golden as mg  # noqa: E402  (loads the reference and instruments its node classes)
from oracle import intersection as oit, ref_loader  # noqa: E402
from oracle.intersection_routes import IntersectionLiteRoutes  # noqa: E402
from tests import intersection_scenes as isc  # noqa: E402
from rl_agents.agents.robust import robust as ref_robust  # noqa: E402

ROUTES_BEHAVIOURS = os.path.join(ref_loader.REFERENCE_ROOT, "scripts", "configs", "IntersectionEnv", "agents",
                                 "DiscreteRobustPlannerAgent", "routes_behaviours.json")


class JointEnv5(ref_robust.JointEnv):
    """robust.py:9-26 with step's tuple re-packed to the five values deterministic.py:41 unpacks."""

    def step(self, action):
        transitions = [state.step(action) for state in self.joint_state]
        observations, rewards, terminals, truncated, info = zip(*transitions)
        return observations, np.array(rewards), np.array(terminals), np.array(truncated), info


ref_robust.JointEnv = JointEnv5


def f64_hex(values):
    return np.asarray(values, dtype="<f8").tobytes().hex()


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def hypotheses(*turns):
    """One model chain per turn: set_route_at_intersection(turn)."""
    return [[{"method": "set_route_at_intersection", "args": a}] for a in turns]


def run(words, config, seed=0):
    del mg.CREATED[:]
    env = IntersectionLiteRoutes(oit.IntersectionLiteState.unpack(np.array(words, dtype=np.int32)))
    agent = ref_robust.DiscreteRobustPlannerAgent(env, json.loads(json.dumps(config)))
    agent.seed(seed)
    plan = [int(a) for a in agent.plan(None)]
    for n in mg.CREATED:
        n.lower, n.upper = float(np.min(n.value_lower)), float(np.min(n.value_upper))
    tree = mg.dump_tree(["lower", "upper"], agent.planner.root)
    assert env.state.pack().tolist() == list(words)          # preprocess_env worked on copies
    return {"words": [int(x) for x in words], "config": config, "seed": seed, "plan": plan,
            "rng_state": rng_state(agent.planner.np_random),
            "tree": {"parent": tree["parent"], "action": tree["action"], "count": tree["count"],
                     "lower": f64_hex(tree["lower"]), "upper": f64_hex(tree["upper"])}}


def scene(seed, speed_index=None):
    st = oit.make_intersection_state(seed)
    if speed_index is not None:
        st.speed_index = int(speed_index)
    return st.pack().tolist()


def at_t12(seed):
    """The scene of `seed` after 12 IDLE decisions (t = 12: one decision left before truncation)."""
    st = oit.make_intersection_state(seed)
    for _ in range(12):
        oit.intersection_step(st, oit.A_IDLE)
    assert st.t == 12
    return st.pack().tolist()


def main():
    with open(ROUTES_BEHAVIOURS) as f:
        shipped = json.load(f)
    out = {"routes_behaviours": shipped, "cases": {}}
    cases = out["cases"]
    for s in (0, 1, 2):
        cases["routes_behaviours_s%d" % s] = run(scene(s), shipped, seed=s)
    for budget in (200, 600):
        cases["m2_s3_b%d" % budget] = run(scene(3), {"budget": budget, "gamma": 0.9, "models": hypotheses(0, 2)})
        cases["m3_s4_b%d" % budget] = run(scene(4), {"budget": budget, "gamma": 0.85,
                                                     "models": hypotheses(0, 1, 2)}, seed=1)
    cases["random_s5_b200"] = run(scene(5), {"budget": 200, "gamma": 0.9, "models": hypotheses("random", 1)}, seed=2)
    cases["random_only_s6_b150"] = run(scene(6), {"budget": 150, "gamma": 0.8, "models": hypotheses("random")})
    cases["terminal_s0_b300"] = run(scene(0), {"budget": 300, "gamma": 0.9, "terminal_reward": 0.5,
                                               "models": hypotheses(0, 1, 2)})
    cases["si0_s1_b200"] = run(scene(1, 0), {"budget": 200, "gamma": 0.9, "models": hypotheses(0, 1, 2)})
    cases["si2_s2_b200"] = run(scene(2, 2), {"budget": 200, "gamma": 0.9, "models": hypotheses(2, 0)})
    # crashes and arrivals inside the tree
    for fam, i in (("arrival", 4), ("full", 0), ("crossing", 1), ("ties", 4)):
        words = isc.family(fam)[i].pack().tolist()
        cases["%s%d_b300" % (fam, i)] = run(words, {"budget": 300, "gamma": 0.9, "terminal_reward": 0.2,
                                                    "models": hypotheses(0, 1, 2)}, seed=3)
    cases["arrival0_random_b200"] = run(isc.family("arrival")[0].pack().tolist(),
                                        {"budget": 200, "gamma": 0.9, "models": hypotheses(1, "random", 5)}, seed=4)
    cases["t12_s7_b200"] = run(at_t12(7), {"budget": 200, "gamma": 0.9, "models": hypotheses(0, 1, 2, "random")})
    return out


if __name__ == "__main__":
    path = os.path.join(HERE, "golden_drop_intersection.json")
    if "--out" in sys.argv:
        path = sys.argv[sys.argv.index("--out") + 1]
    data = main()
    with open(path, "w") as f:
        json.dump(data, f, sort_keys=True, separators=(",", ":"))
        f.write("\n")
    print("wrote", path, "(%d cases)" % len(data["cases"]))
