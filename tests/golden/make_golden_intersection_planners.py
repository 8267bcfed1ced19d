"""Generate tests/golden/golden_intersection_planners.json by running the UNMODIFIED reference MCTSAgent / MCTS and
OLOPAgent (rl_agents/agents/tree_search/mcts.py, olop.py) on IntersectionLite (oracle.intersection.IntersectionLite).

MCTS drives the env as it is (5-tuple step); OLOP goes through oracle.envs.LegacyStepEnv and a
oracle.ref_loader.legacy_np_random generator, as tests/golden/make_golden.py does for HighwayLite.  Node creation order
is recorded by make_golden.py's instrumentation, and its dump_tree writes the trees.

Per case: the env (scene seed, optionally a root speed index), the config, the planner seed, the plan, the episodes,
horizon (and MCTS temperature) the planner completed, every node in creation order (parent, action, count and the
float fields) and the PCG64 state after the decision.  Cases: MCTS by budget and by explicit episodes / horizon on
several scenes, one with only two actions available at the root; preference (one preferring SLOWER) and random
policies; closed_loop; three consecutive "subtree" decisions; receding_horizon 3; OLOP with the KL bound and the
"uniform" / "zeros" continuations ("zeros" fails with the reference's KeyError once SLOWER is unavailable); a horizon
past the env's DURATION (13), so that truncation ends MCTS rollouts.

Needs the reference tree (oracle.ref_loader.REFERENCE_ROOT), so the output is committed and the tests only read it.
Writes only golden_intersection_planners.json (or --out PATH), reproducibly byte for byte.
Usage:  python tests/golden/make_golden_intersection_planners.py [--out PATH]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import make_golden as mg  # noqa: E402  (loads the reference and instruments its node classes)
from oracle import envs, ref_loader  # noqa: E402
from oracle import intersection as oit  # noqa: E402

ref_mcts, ref_olop = mg.ref_mcts, mg.ref_olop

KL_GLOBAL = {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)"}
KL_LOCAL = {"type": "kullback-leibler", "time": "local", "threshold": "1*np.log(time)"}


def make_env(spec):
    """{"seed": s} -> IntersectionLite on make_intersection_state(s); "speed_index" overrides the ego's speed index."""
    st = oit.make_intersection_state(spec["seed"])
    if "speed_index" in spec:
        st.speed_index = int(spec["speed_index"])
    return oit.IntersectionLite(st)


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def mcts_agent(spec, config, seed):
    agent = ref_mcts.MCTSAgent(make_env(spec), json.loads(json.dumps(config)))
    agent.seed(seed)
    return agent


def run_mcts(spec, config, seed):
    del mg.CREATED[:]
    agent = mcts_agent(spec, config, seed)
    plan = [int(a) for a in agent.plan(None)]
    pc = agent.planner.config
    return {"env": spec, "config": config, "seed": seed, "plan": plan, "episodes": int(pc["episodes"]),
            "horizon": int(pc["horizon"]), "temperature": float(pc["temperature"]),
            "tree": mg.dump_tree(["value", "prior"], agent.planner.root), "rng_state": rng_state(agent.planner.np_random)}


def olop_agent(spec, config, seed):
    agent = ref_olop.OLOPAgent(envs.LegacyStepEnv(make_env(spec)), json.loads(json.dumps(config)))
    agent.planner.np_random, _ = ref_loader.legacy_np_random(seed)
    return agent


def run_olop(spec, config, seed):
    del mg.CREATED[:]
    agent = olop_agent(spec, config, seed)
    out = {"env": spec, "config": config, "seed": seed, "episodes": int(agent.planner.config["episodes"]),
           "horizon": int(agent.planner.config["horizon"])}
    try:
        out["plan"] = [int(a) for a in agent.plan(None)]
    except KeyError as e:                  # "zeros" continuation on a node without action 0 (olop.py:82,88)
        out["error"] = {"error": type(e).__name__, "message": str(e)}
        out["rng_state"] = rng_state(agent.planner.np_random)
        return out
    for n in mg.CREATED:
        n.upper = n.value_upper
    out["tree"] = mg.dump_tree(["cumulative_reward", "mu_ucb", "upper", "done"], agent.planner.root)
    out["rng_state"] = rng_state(agent.planner.np_random)
    return out


def canonical(root):
    """Breadth first, children in insertion order: [n_children, count, value, prior] per node."""
    nodes, head, rows = [root], 0, []
    while head < len(nodes):
        nd = nodes[head]
        rows.append([len(nd.children), int(nd.count), float(nd.value), float(nd.prior)])
        nodes.extend(nd.children.values())
        head += 1
    return rows


def main():
    out = {"mcts": {}, "olop": {}, "agents": {}}
    mc = out["mcts"]
    for seed, budget, gamma in ((0, 200, 0.8), (1, 400, 0.9), (3, 300, 0.85)):
        mc["s%d_b%d_g%s" % (seed, budget, gamma)] = run_mcts({"seed": seed}, {"budget": budget, "gamma": gamma},
                                                             seed=seed + 10)
    mc["s2_ep80_h6_g0.8"] = run_mcts({"seed": 2}, {"episodes": 80, "horizon": 6, "gamma": 0.8}, seed=4)
    mc["s4_ep50_h5_g0.9_T3"] = run_mcts({"seed": 4}, {"episodes": 50, "horizon": 5, "gamma": 0.9, "temperature": 3.0},
                                        seed=5)
    # only IDLE and SLOWER are available at the root (top speed index)
    mc["s5_top_speed_b300_g0.85"] = run_mcts({"seed": 5, "speed_index": 2}, {"budget": 300, "gamma": 0.85}, seed=6)
    # only IDLE and FASTER (bottom speed index)
    mc["s6_bottom_speed_ep60_h5"] = run_mcts({"seed": 6, "speed_index": 0}, {"episodes": 60, "horizon": 5, "gamma": 0.8},
                                             seed=7)
    # horizon past DURATION: rollouts end on truncation
    mc["s1_ep40_h16_g0.9"] = run_mcts({"seed": 1}, {"episodes": 40, "horizon": 16, "gamma": 0.9}, seed=8)
    # policies: preference for SLOWER in the priors and FASTER in the rollouts; uniform over all actions
    mc["s0_preference_b300_g0.8"] = run_mcts({"seed": 0}, {
        "budget": 300, "gamma": 0.8, "prior_policy": {"type": "preference", "action": 0, "ratio": 3},
        "rollout_policy": {"type": "preference", "action": 2, "ratio": 2}}, seed=9)
    mc["s5_top_speed_preference_slower"] = run_mcts({"seed": 5, "speed_index": 2}, {
        "episodes": 60, "horizon": 6, "gamma": 0.85, "prior_policy": {"type": "preference", "action": 0, "ratio": 2},
        "rollout_policy": {"type": "preference", "action": 0, "ratio": 4}}, seed=10)
    mc["s2_random_b300_g0.85"] = run_mcts({"seed": 2}, {
        "budget": 300, "gamma": 0.85, "prior_policy": {"type": "random"}, "rollout_policy": {"type": "random"}}, seed=11)

    # closed loop on a deterministic env: one observation node per action node (mcts.py:125,147,267-273)
    agent = mcts_agent({"seed": 3}, {"budget": 300, "gamma": 0.8, "closed_loop": True}, 12)
    plan = agent.plan(None)
    root = agent.planner.root
    out["closed_loop"] = {"env": {"seed": 3}, "config": {"budget": 300, "gamma": 0.8, "closed_loop": True}, "seed": 12,
                          "plan_actions": [int(a) for a in plan[0::2]], "plan_len": len(plan),
                          "root": [[int(a), int(c.count), float(c.value)] for a, c in root.children.items()],
                          "root_count": int(root.count), "root_value": float(root.value),
                          "rng_state": rng_state(agent.planner.np_random)}

    # step_strategy "subtree": three consecutive decisions, the env stepped by each plan's first action
    config = {"budget": 300, "gamma": 0.85, "step_strategy": "subtree"}
    agent = mcts_agent({"seed": 1}, config, 13)
    env = agent.env
    sub = {"env": {"seed": 1}, "config": config, "seed": 13, "plans": [], "trees": [], "words": []}
    for _ in range(3):
        sub["words"].append(env.state.pack().tolist())
        plan = agent.plan(None)
        sub["plans"].append([int(a) for a in plan])
        sub["trees"].append(canonical(agent.planner.root))
        env.step(plan[0])
    sub["episodes"], sub["horizon"] = int(agent.planner.config["episodes"]), int(agent.planner.config["horizon"])
    sub["temperature"] = float(agent.planner.config["temperature"])
    sub["rng_state"] = rng_state(agent.planner.np_random)
    out["subtree"] = sub

    ol = out["olop"]
    ol["s0_b200_g0.9_kl_uniform"] = run_olop({"seed": 0}, {"budget": 200, "gamma": 0.9, "continuation_type": "uniform",
                                                           "upper_bound": KL_GLOBAL}, seed=0)
    ol["s3_b500_g0.8_kl_local_uniform"] = run_olop({"seed": 3}, {"budget": 500, "gamma": 0.8,
                                                                 "continuation_type": "uniform",
                                                                 "upper_bound": KL_LOCAL}, seed=1)
    ol["s5_top_speed_b150_g0.8_kl_uniform"] = run_olop({"seed": 5, "speed_index": 2}, {
        "budget": 150, "gamma": 0.8, "continuation_type": "uniform", "upper_bound": KL_GLOBAL}, seed=2)
    # "zeros": SLOWER (action 0) is available at the root, so a one-step horizon plans ...
    ol["s2_ep30_h1_kl_zeros"] = run_olop({"seed": 2}, {"episodes": 30, "horizon": 1, "gamma": 0.8,
                                                       "continuation_type": "zeros", "upper_bound": KL_GLOBAL}, seed=3)
    # ... and a longer one reaches a node at the bottom speed index, where children[0] is a KeyError
    ol["s2_b200_kl_zeros_keyerror"] = run_olop({"seed": 2}, {"budget": 200, "gamma": 0.8, "continuation_type": "zeros",
                                                             "upper_bound": KL_GLOBAL}, seed=4)
    ol["s1_ep12_h15_kl_uniform"] = run_olop({"seed": 1}, {"episodes": 12, "horizon": 15, "gamma": 0.9,
                                                          "continuation_type": "uniform", "upper_bound": KL_GLOBAL},
                                            seed=5)

    # receding_horizon 3: three agent.plan() calls on one env, the last two served from the first plan
    ag = out["agents"]
    for name, make, config, seed in (
            ("mcts_receding_horizon3", mcts_agent, {"budget": 300, "gamma": 0.8, "receding_horizon": 3}, 14),
            ("olop_receding_horizon3", olop_agent, {"budget": 200, "gamma": 0.9, "continuation_type": "uniform",
                                                    "upper_bound": KL_GLOBAL, "receding_horizon": 3}, 15)):
        agent = make({"seed": 4}, config, seed)
        decisions = [[int(a) for a in agent.plan(None)] for _ in range(4)]
        ag[name] = {"env": {"seed": 4}, "config": config, "seed": seed, "decisions": decisions,
                    "rng_state": rng_state(agent.planner.np_random)}

    path = os.path.join(HERE, "golden_intersection_planners.json")
    if "--out" in sys.argv:
        path = sys.argv[sys.argv.index("--out") + 1]
    with open(path, "w") as f:
        json.dump(out, f)
    print("IntersectionLite MCTS / OLOP done:", path)


if __name__ == "__main__":
    main()
