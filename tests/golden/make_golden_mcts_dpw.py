"""Generate tests/golden/golden_mcts_dpw.json by running the UNMODIFIED reference MCTSDPW planner
(rl_agents/agents/tree_search/mcts_dpw.py) on the oracle env models.

The reference cannot run as it stands, so two shims close its gaps, as the DROP goldens re-pack a tuple
(tests/golden/make_golden.py):
- MCTSDPW.run unpacks a 4-tuple `step` (:76) while the inherited MCTS.evaluate unpacks a 5-tuple (mcts.py:171).  The env
  is an oracle.envs.LegacyStepEnv, and the planner's `evaluate` is bound on the instance to the unmodified
  MCTS.evaluate applied to the wrapped 5-tuple env (`state.env`).
- DecisionNode.get_child calls `state.get_available_actions()` with no fallback (:121).  A finite MDP is wrapped in an
  adapter whose get_available_actions is list(range(n)), the fallback of unexplored_actions (:110-113).
The goldens pin the planner's plan(), which returns a bare action (the reference agent's act() raises on it).

The stochastic finite MDPs the cases run on are stored in the output, so the tests need nothing else.  Needs the
reference tree (oracle.ref_loader.REFERENCE_ROOT), so the output is committed and the tests only read it.  Writes only
golden_mcts_dpw.json, reproducibly byte for byte.  Usage:  python tests/golden/make_golden_mcts_dpw.py
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_loader  # noqa: E402
from oracle import envs  # noqa: E402
from oracle.mcts_dpw import tree_digest  # noqa: E402

ref_loader.load_reference()
from rl_agents.agents.tree_search import mcts as ref_mcts  # noqa: E402
from rl_agents.agents.tree_search import mcts_dpw as ref_dpw  # noqa: E402

CREATED = []


def _instrument(cls):
    """Record node creation order at run time (sources stay unmodified)."""
    orig = cls.__init__

    def init(self, *a, **k):
        orig(self, *a, **k)
        CREATED.append(self)
    cls.__init__ = init


for _cls in (ref_dpw.DecisionNode, ref_dpw.ChanceNode):
    _instrument(_cls)


class FiniteActionsEnv(envs.LegacyStepEnv):
    """A 4-tuple finite MDP with get_available_actions = range(action_space.n)."""

    def get_available_actions(self):
        return list(range(self.action_space.n))

    def __deepcopy__(self, memo):
        import copy
        return FiniteActionsEnv(copy.deepcopy(self.env, memo))


def stochastic_mdps():
    """The stochastic tables of the cases, as JSON-ready lists."""
    rng = np.random.default_rng(2025)
    # dense "stochastic" MDP: 8 states, 3 actions, about 40 % zero entries per row, state 7 terminal
    p = rng.uniform(size=(8, 3, 8))
    p[p < 0.4] = 0.0
    p[:, :, 0] += 0.05
    p /= p.sum(axis=-1, keepdims=True)
    stoch8 = {"mode": "stochastic", "transition": p, "reward": rng.uniform(size=(8, 3)), "terminal": np.arange(8) == 7}
    # "sparse" garnet: 12 states, 3 actions, 4 successors; the root's rows repeat a next state and hold zero entries
    gp, gn, gr = envs.garnet(12, 3, 4, seed=5)
    gn[0, 0] = [4, 4, 9, 1]
    gp[0, 0] = [0.25, 0.25, 0.0, 0.5]
    gn[0, 1] = [2, 7, 2, 7]
    gp[0, 1] = [0.0, 0.5, 0.0, 0.5]
    garnet = {"mode": "sparse", "transition": gp, "next": gn, "reward": gr, "terminal": np.zeros(12, bool)}
    # sha1("406")[:5] == sha1("678")[:5]: 680 states, 2 actions, 2 successors; (0, 0) reaches both, and both lead
    # back to the root, so in closed loop the two share one decision node
    S = 680
    nxt = rng.integers(0, 8, size=(S, 2, 2))
    prob = rng.choice([0.25, 0.5, 0.75], size=(S, 2, 1))
    prob = np.concatenate([prob, 1.0 - prob], axis=-1)
    nxt[0, 0] = [406, 678]
    prob[0, 0] = [0.5, 0.5]
    nxt[406] = 0
    nxt[678] = 0
    collide = {"mode": "sparse", "transition": prob, "next": nxt, "reward": np.round(rng.uniform(size=(S, 2)), 3),
               "terminal": np.zeros(S, bool)}
    # a negative entry in a row of state 5, reachable from the root
    bad = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in stoch8.items()}
    bad["transition"][5, 0] = 0.0
    bad["transition"][5, 0, :2] = [-0.25, 1.25]
    out = {"stoch8": stoch8, "garnet12": garnet, "collide680": collide, "stoch8_bad_row": bad}
    return {name: {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in m.items()}
            for name, m in out.items()}


def dump_tree(root):
    """Creation-order dump: a chance node's key is its action; a decision node's key is its observation key
    int(sha1(str(obs))[:5], 16), -1 at the root.  Every node's children must be in creation order."""
    def top(n):
        while n.parent is not None:
            n = n.parent
        return n
    nodes = [n for n in CREATED if top(n) is root]
    assert nodes[0] is root
    ids = {id(n): i for i, n in enumerate(nodes)}
    out = {k: [] for k in ("parent", "kind", "key", "count", "value")}
    for n in nodes:
        chance = isinstance(n, ref_dpw.ChanceNode)
        p = n.parent
        out["parent"].append(ids[id(p)] if p is not None else -1)
        out["kind"].append(1 if chance else 0)
        if p is None:
            key = -1
        else:
            key = next(k for k, c in p.children.items() if c is n)
            key = int(key) if chance else int(key, 16)
        out["key"].append(key)
        out["count"].append(int(n.count))
        out["value"].append(float(n.value))
        kids = [ids[id(c)] for c in n.children.values()]
        assert kids == sorted(kids)
    return out


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def make_env(spec, m, tables):
    """The env a case runs on: {"name": "highway", "seed": s}, a deterministic MDP of finite_mdps.npz or one of the
    stored stochastic tables, optionally with zero rewards, rooted at `state`."""
    if spec["name"] == "highway":
        return envs.HighwayLite(seed=spec["seed"])
    n = spec["name"]
    if n in tables:
        t = tables[n]
        reward = np.zeros_like(np.array(t["reward"])) if spec.get("zero_rewards") else np.array(t["reward"])
        return envs.FiniteMDPLite(np.array(t["transition"]), reward, np.array(t["terminal"]), mode=t["mode"],
                                  nxt=None if "next" not in t else np.array(t["next"]), state=spec.get("state", 0))
    reward = np.zeros_like(m[n + "_R"]) if spec.get("zero_rewards") else m[n + "_R"]
    return envs.FiniteMDPLite(m[n + "_T"], reward, m[n + "_term"], mode="deterministic", state=spec.get("state", 0))


def wrap(env):
    return envs.LegacyStepEnv(env) if isinstance(env, envs.HighwayLite) else FiniteActionsEnv(env)


def make_planner(env, config, seed):
    agent = ref_dpw.MCTSDPWAgent(wrap(env), dict(config))
    planner = agent.planner
    planner.np_random, _ = ref_loader.legacy_np_random(seed)

    def evaluate(self, state, observation, total_reward=0, depth=0):
        return ref_mcts.MCTS.evaluate(self, state.env, observation, total_reward, depth=depth)
    planner.evaluate = types.MethodType(evaluate, planner)
    return agent, planner


def run(m, tables, spec, config, seed=0, decisions=1):
    agent, planner = make_planner(make_env(spec, m, tables), config, seed)
    plans = []
    for _ in range(decisions):
        del CREATED[:]
        planner.step_by_reset()                 # a fresh root, as the agent's "reset" step strategy gives
        del planner.observations[:]
        a = planner.plan(agent.env, None)
        plans.append(int(a))
    tree = dump_tree(planner.root)
    out = {"env": spec, "config": config, "seed": seed, "plan": plans[-1], "steps": len(planner.observations),
           "episodes": planner.config["episodes"], "horizon": planner.config["horizon"],
           "rng_state": rng_state(planner.np_random), "tree": tree_digest(tree)}
    if decisions > 1:
        out["plans"] = plans
    return out


def error_of(fn):
    try:
        fn()
    except Exception as e:              # noqa: BLE001 -- the reference's own exception is what is recorded
        return {"error": type(e).__name__, "message": str(e)}
    raise AssertionError("expected an error")


def main():
    m = np.load(os.path.join(HERE, "finite_mdps.npz"))
    tables = stochastic_mdps()
    stoch8, garnet12 = {"name": "stoch8"}, {"name": "garnet12"}
    trap_terminal = int(np.nonzero(m["trap_term"])[0][0])
    big = {"horizon": 6, "episodes": 200}                      # a wider tree than budget 100's 5 episodes

    out = {"mdps": tables, "cases": {}, "configs": {}, "errors": {}}
    cases = out["cases"]
    cases["stoch8_default"] = run(m, tables, stoch8, {})
    cases["stoch8_default_budget1000"] = run(m, tables, stoch8, {"budget": 1000}, seed=1)
    cases["stoch8_h6_e200"] = run(m, tables, stoch8, big, seed=2)
    cases["garnet12_sparse_h6_e200"] = run(m, tables, garnet12, big, seed=3)
    cases["garnet12_sparse_default"] = run(m, tables, garnet12, {}, seed=4)
    cases["large1_deterministic_h6_e200"] = run(m, tables, {"name": "large1"}, big, seed=5)
    cases["trap_deterministic_default"] = run(m, tables, {"name": "trap"}, {}, seed=6)
    cases["trap_terminal_root_default"] = run(m, tables, {"name": "trap", "state": trap_terminal}, {}, seed=7)
    cases["stoch8_terminal_root_h6_e200"] = run(m, tables, {"name": "stoch8", "state": 7}, big, seed=8)
    # closed loop: k_state * N**alpha_state < len(children) blocks new states, and choice(list(children)) fires
    cases["stoch8_closed_loop_h6_e200"] = run(m, tables, stoch8, dict(big, closed_loop=True), seed=9)
    cases["garnet12_closed_loop_h6_e200"] = run(m, tables, garnet12, dict(big, closed_loop=True), seed=10)
    cases["stoch8_closed_loop_k2_a0.5"] = run(m, tables, stoch8, dict(big, closed_loop=True, k_state=2,
                                                                      alpha_state=0.5), seed=11)
    cases["collide680_closed_loop"] = run(m, tables, {"name": "collide680"},
                                          {"horizon": 3, "episodes": 60, "closed_loop": True, "k_state": 4,
                                           "alpha_state": 0.5}, seed=12)
    # all rewards zero: every UCB index of equal counts ties, and random_argmax draws
    cases["stoch8_zero_rewards_h6_e200"] = run(m, tables, {"name": "stoch8", "zero_rewards": True}, big, seed=13)
    cases["stoch8_random_rollout"] = run(m, tables, stoch8, dict(big, rollout_policy={"type": "random"}), seed=14)
    cases["stoch8_preference_rollout"] = run(m, tables, stoch8, dict(
        big, rollout_policy={"type": "preference", "action": 1, "ratio": 3}), seed=15)
    cases["stoch8_temperature0"] = run(m, tables, stoch8, dict(big, temperature=0), seed=16)
    cases["stoch8_k_action_10"] = run(m, tables, stoch8, dict(big, k_action=10), seed=17)
    cases["stoch8_alpha_action_0"] = run(m, tables, stoch8, dict(big, alpha_action=0), seed=18)
    for s in range(4):
        cases["hw%d_default" % s] = run(m, tables, {"name": "highway", "seed": s}, {}, seed=20 + s)
    cases["hw1_closed_loop_h4_e40"] = run(m, tables, {"name": "highway", "seed": 1},
                                          {"horizon": 4, "episodes": 40, "closed_loop": True}, seed=24)
    cases["hw2_preference_rollout_h4_e30"] = run(m, tables, {"name": "highway", "seed": 2}, {
        "horizon": 4, "episodes": 30, "rollout_policy": {"type": "preference", "action": 3, "ratio": 2}}, seed=25)
    cases["hw3_random_rollout_h4_e30"] = run(m, tables, {"name": "highway", "seed": 3},
                                             {"horizon": 4, "episodes": 30, "rollout_policy": {"type": "random"}},
                                             seed=26)
    # three consecutive decisions of one planner: its np_random carries on
    cases["stoch8_three_decisions"] = run(m, tables, stoch8, big, seed=27, decisions=3)
    for k, c in cases.items():
        print(k, "plan", c["plan"], "nodes", c["tree"]["n_nodes"], "steps", c["steps"])

    def plan_with(config, spec=stoch8):
        agent, planner = make_planner(make_env(spec, m, tables), config, 0)
        return planner.plan(agent.env, None)
    errs = out["errors"]
    # horizon < 1 leaves the root childless: get_plan returns None
    errs["horizon_negative_plan"] = {"plan": plan_with({"horizon": -1, "episodes": 3})}
    errs["missing_episodes"] = error_of(lambda: plan_with({"horizon": 3}))
    errs["alpha_action_negative"] = error_of(lambda: plan_with({"alpha_action": -0.5}))
    errs["bad_row"] = error_of(lambda: plan_with(big, {"name": "stoch8_bad_row"}))
    errs["agent_act"] = error_of(lambda: make_planner(make_env(stoch8, m, tables), {}, 0)[0].act(None))

    # completed configs of the agent and its planner (the `__class__` key is left out)
    for name, cfg in (("empty", {}), ("closed_loop_budget_500", {"budget": 500, "closed_loop": True, "k_state": 2}),
                      ("horizon_given", {"horizon": 5, "episodes": 50, "gamma": 0.9})):
        agent = ref_dpw.MCTSDPWAgent(wrap(make_env(stoch8, m, tables)), json.loads(json.dumps(cfg)))
        out["configs"][name] = {"config": cfg, "completed": json.loads(json.dumps(agent.config)),
                                "planner": json.loads(json.dumps(agent.planner.config))}
    with open(os.path.join(HERE, "golden_mcts_dpw.json"), "w") as f:
        json.dump(out, f)
    print("MCTS-DPW done")


if __name__ == "__main__":
    main()
