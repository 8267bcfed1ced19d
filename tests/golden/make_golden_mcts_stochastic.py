"""Generate tests/golden/golden_mcts_stochastic.json by running the UNMODIFIED reference MCTSAgent
(rl_agents/agents/tree_search/mcts.py) on stochastic finite MDPs (the cases of tests/mcts_stochastic_cases.py), with the
node instrumentation of make_golden.py.  The oracle env's 5-tuple `step` is the one MCTS calls, so no adapter is needed.
The reference never reseeds its env copies: every episode replays the live env's generator, which each case seeds and
may move forward before the decision.

Each case records the tree in the digest form of tests/mcts_stochastic_cases.py, the plan, the planner's RNG words after
the search and the live env's generator, which planning leaves unchanged.  Closed-loop cases also check that every
action node has at most one observation child, and record the tree with the observation nodes taken out (the action-node
projection), which the open-loop search builds.  Subtree cases plan twice with one real env step in between.

Build-container only (the reference tree does not travel to the GPU box); the output is committed and the same bytes
on every run.  Writes only golden_mcts_stochastic.json (or the --out path).
Usage:  python tests/golden/make_golden_mcts_stochastic.py [--out PATH]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import make_golden as base  # noqa: E402  (loads the reference and instruments its nodes)
from tests.mcts_stochastic_cases import (CASES, CLOSED_LOOP, ERRORS, SUBTREE, canonical_digest, live_env,  # noqa: E402
                                         rng_state, tree_digest)


def agent_for(case):
    env = live_env(case)
    agent = base.ref_mcts.MCTSAgent(env, json.loads(json.dumps(case[2])))
    agent.seed(case[3])
    return env, agent


def planner_record(agent):
    pl = agent.planner
    return {"episodes": int(pl.config["episodes"]), "horizon": int(pl.config["horizon"]),
            "temperature": float(pl.config["temperature"]), "gamma": float(pl.config["gamma"]),
            "rng_state": rng_state(pl.np_random)}


def case_header(case):
    mdp, state, config, seed, env_seed, advance = case
    return {"mdp": mdp, "state": state, "config": config, "seed": seed, "env_seed": env_seed, "advance": advance}


def run(case):
    del base.CREATED[:]
    env, agent = agent_for(case)
    before = rng_state(env.np_random)
    plan = agent.plan(int(env.mdp.state))
    assert rng_state(env.np_random) == before
    out = case_header(case)
    out.update(planner_record(agent), plan=[int(a) for a in plan], env_rng_state=before,
               tree=tree_digest(base.dump_tree(["value", "prior"], agent.planner.root)))
    return out


def run_closed_loop(case):
    """The reference tree interleaves observation nodes under the action nodes: check there is at most one per action
    node, with the action node's count and value, and digest the action-node projection."""
    del base.CREATED[:]
    env, agent = agent_for(case)
    before = rng_state(env.np_random)
    plan = agent.plan(int(env.mdp.state))
    assert rng_state(env.np_random) == before
    root = agent.planner.root

    def top(n):
        while n.parent is not None:
            n = n.parent
        return n
    created = [n for n in base.CREATED if top(n) is root]
    obs, actions = set(), set()
    for n in created:                     # parents come before their children
        if n is root:
            continue
        if id(n.parent) in actions:
            obs.add(id(n))
            continue
        # n is an action node (a child of the root or of an observation node): at most one observation child, which
        # carries its statistics
        actions.add(id(n))
        assert len(n.children) <= 1
        for o in n.children.values():
            assert (o.count, o.value) == (n.count, n.value)
    kept = [n for n in created if id(n) not in obs]
    ids = {id(n): i for i, n in enumerate(kept)}

    def action_parent(n):
        p = n.parent
        if p is not None and id(p) in obs:
            p = p.parent
        return p

    tree = {"parent": [], "action": [], "count": [], "value": [], "prior": []}
    for n in kept:
        p = n.parent
        tree["parent"].append(ids[id(action_parent(n))] if p is not None else -1)
        act = -1
        if p is not None:
            act = int(next(a for a, c in p.children.items() if c is n))
        tree["action"].append(act)
        tree["count"].append(int(n.count))
        tree["value"].append(float(n.value))
        tree["prior"].append(float(n.prior))
    out = case_header(case)
    out.update(planner_record(agent), plan_actions=[int(a) for a in plan[0::2]], plan_len=len(plan),
               env_rng_state=before, n_observation_nodes=len(obs), tree=tree_digest(tree))
    return out


def bfs_digest(root):
    nodes, head = [root], 0
    first_child, n_children, action, count, value, prior = [], [], [], [], [], []
    while head < len(nodes):
        nd = nodes[head]
        first_child.append(len(nodes) if nd.children else -1)
        n_children.append(len(nd.children))
        for a, c in nd.children.items():
            nodes.append(c)
        head += 1
    for nd in nodes:
        p = nd.parent
        act = -1 if p is None or nd is root else int(next(a for a, c in p.children.items() if c is nd))
        action.append(act)
        count.append(int(nd.count))
        value.append(float(nd.value))
        prior.append(float(nd.prior))
    return canonical_digest(first_child, n_children, action, count, value, prior)


def run_subtree(case):
    """Two decisions with step_strategy "subtree", the live env stepped once in between."""
    env, agent = agent_for(case)
    out = case_header(case)
    out["decisions"] = []
    for k in range(2):
        state, before = int(env.mdp.state), rng_state(env.np_random)
        plan = agent.plan(state)
        assert rng_state(env.np_random) == before
        d = planner_record(agent)
        d.update(state=state, env_rng_state=before, plan=[int(a) for a in plan], tree=bfs_digest(agent.planner.root))
        out["decisions"].append(d)
        if k == 0:
            env.step(plan[0])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(HERE, "golden_mcts_stochastic.json"))
    path = ap.parse_args().out
    out = {"cases": {}, "closed_loop": {}, "subtree": {}, "errors": {}}
    for name, case in CASES.items():
        out["cases"][name] = c = run(case)
        print(name, c["episodes"], "x", c["horizon"], "nodes", c["tree"]["n_nodes"], "plan", c["plan"])
    for name, case in CLOSED_LOOP.items():
        out["closed_loop"][name] = c = run_closed_loop(case)
        print(name, "nodes", c["tree"]["n_nodes"], "observation nodes", c["n_observation_nodes"], c["plan_actions"])
    for name, case in SUBTREE.items():
        out["subtree"][name] = c = run_subtree(case)
        print(name, [(d["state"], d["tree"]["n_nodes"], d["plan"][:3]) for d in c["decisions"]])
    for name, case in ERRORS.items():
        try:
            run(case)
            raise AssertionError("%s was expected to raise" % name)
        except ValueError as e:
            out["errors"][name] = dict(case_header(case), error=type(e).__name__, message=str(e))
            print(name, type(e).__name__ + ":", e)
    with open(path, "w") as f:
        json.dump(out, f)
    print("mcts_stochastic done")


if __name__ == "__main__":
    main()
