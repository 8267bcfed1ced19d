"""Generate tests/golden/golden_platypoos.json by running the UNMODIFIED reference PlaTyPOOS planner
(rl_agents/agents/tree_search/platypoos.py) on the oracle env models.

The reference cannot run as it stands, so shims close its gaps:
- It calls a 4-tuple `step` and `np_random.randint`: the env is an oracle.envs.LegacyStepEnv and the planner's generator
  an oracle.ref_loader.legacy_np_random, as for the other goldens.
- Its root has no `value` attribute, so the first child update raises AttributeError.  PlaTyPOOS.reset is wrapped to set
  `root.value = 0.0` after the unmodified reset, the position the port takes.
A finite MDP has no get_available_actions, so the reference's own fallback, range(1, n), applies unchanged.

Per case: every node in creation order (parent, action, depth, count, the float64 bytes of cumulative_reward and value
as hex, done, to_expand), the openings, the candidates in dict order as [p, node id], the plan and the PCG64 state after
plan().  The stochastic finite MDPs the cases run on are stored in the output, so the tests need nothing else.  Needs
the reference tree (oracle.ref_loader.REFERENCE_ROOT), so the output is committed and the tests only read it.  Writes
only golden_platypoos.json, reproducibly byte for byte.  The two budget-50 000 HighwayLite cases take about 40 s each.
Usage:  python tests/golden/make_golden_platypoos.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import envs  # noqa: E402
from oracle import ref_loader  # noqa: E402

ref_loader.load_reference()
from rl_agents.agents.tree_search import platypoos as ref_pl  # noqa: E402

CREATED = []
BASELINE = {"env_preprocessors": [{"method": "simplify"}], "gamma": 0.9, "budget": 2500, "max_depth": 4}


def _instrument():
    """Record node creation order and give the root the value 0.0 (sources stay unmodified)."""
    init = ref_pl.PlaTyPOOSNode.__init__

    def node_init(self, *a, **k):
        init(self, *a, **k)
        CREATED.append(self)
    ref_pl.PlaTyPOOSNode.__init__ = node_init
    reset = ref_pl.PlaTyPOOS.reset

    def planner_reset(self):
        del CREATED[:]
        reset(self)
        self.root.value = 0.0
    ref_pl.PlaTyPOOS.reset = planner_reset


_instrument()


def stochastic_mdps():
    """The stochastic tables of the cases, as JSON-ready lists."""
    rng = np.random.default_rng(2026)
    # dense "stochastic" MDP: 8 states, 4 actions, about 40 % zero entries per row, state 7 terminal
    p = rng.uniform(size=(8, 4, 8))
    p[p < 0.4] = 0.0
    p[:, :, 0] += 0.05
    p /= p.sum(axis=-1, keepdims=True)
    stoch8 = {"mode": "stochastic", "transition": p, "reward": rng.uniform(size=(8, 4)), "terminal": np.arange(8) == 7}
    # "sparse" garnet: 12 states, 3 actions, 4 successors, state 11 terminal
    gp, gn, gr = envs.garnet(12, 3, 4, seed=7)
    garnet = {"mode": "sparse", "transition": gp, "next": gn, "reward": gr, "terminal": np.arange(12) == 11}
    # a negative entry in the row (3, 2), reachable from the root
    bad = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in stoch8.items()}
    bad["transition"][3, 2] = 0.0
    bad["transition"][3, 2, :2] = [-0.25, 1.25]
    out = {"stoch8": stoch8, "garnet12": garnet, "stoch8_bad_row": bad}
    return {name: {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in m.items()}
            for name, m in out.items()}


def make_env(spec, m, tables):
    """The env a case runs on: {"name": "highway", "seed": s}; {"name": "garnet", ...} a deterministic
    oracle.envs.garnet; a deterministic MDP of finite_mdps.npz (optionally its first `actions` actions) or one of the
    stored stochastic tables; optionally with zero rewards, rooted at `state`."""
    n = spec["name"]
    if n == "highway":
        return envs.HighwayLite(seed=spec["seed"])
    if n == "garnet":
        T, R = envs.garnet(spec["states"], spec["actions"], 1, seed=spec["seed"], deterministic=True)
        return envs.FiniteMDPLite(T, R, state=spec.get("state", 0))
    if n in tables:
        t = tables[n]
        reward = np.zeros_like(np.array(t["reward"])) if spec.get("zero_rewards") else np.array(t["reward"])
        return envs.FiniteMDPLite(np.array(t["transition"]), reward, np.array(t["terminal"]), mode=t["mode"],
                                  nxt=None if "next" not in t else np.array(t["next"]), state=spec.get("state", 0))
    a = spec.get("actions", m[n + "_R"].shape[1])
    reward = np.zeros_like(m[n + "_R"][:, :a]) if spec.get("zero_rewards") else m[n + "_R"][:, :a]
    return envs.FiniteMDPLite(m[n + "_T"][:, :a], reward, m[n + "_term"], mode="deterministic",
                              state=spec.get("state", 0))


def dump_tree(root):
    assert CREATED[0] is root
    ids = {id(n): i for i, n in enumerate(CREATED)}
    out = {k: [] for k in ("parent", "action", "depth", "count", "done", "to_expand")}
    cum, val = [], []
    for n in CREATED:
        p = n.parent
        out["parent"].append(ids[id(p)] if p is not None else -1)
        out["action"].append(-1 if p is None else int(next(a for a, c in p.children.items() if c is n)))
        out["depth"].append(int(n.depth))
        out["count"].append(int(n.count))
        out["done"].append(int(bool(n.done)))
        out["to_expand"].append(int(bool(n.to_expand)))
        cum.append(float(n.cumulative_reward))
        val.append(float(n.value))
        kids = [ids[id(c)] for c in n.children.values()]
        assert kids == sorted(kids)
    out["cumulative_reward"] = np.array(cum, dtype=np.float64).tobytes().hex()
    out["value"] = np.array(val, dtype=np.float64).tobytes().hex()
    return out


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def make_agent(env, config, seed):
    agent = ref_pl.PlaTyPOOSAgent(envs.LegacyStepEnv(env), json.loads(json.dumps(config)))
    agent.planner.np_random, _ = ref_loader.legacy_np_random(seed)
    return agent


def run(m, tables, spec, config, seed=0):
    agent = make_agent(make_env(spec, m, tables), config, seed)
    planner = agent.planner
    planner.step_by_reset()
    plan = [int(a) for a in planner.plan(agent.env, None)]
    ids = {id(n): i for i, n in enumerate(CREATED)}
    out = {"env": spec, "config": config, "seed": seed, "horizon": planner.config["horizon"], "plan": plan,
           "openings": int(planner.openings), "candidates": [[int(p), ids[id(n)]] for p, n in planner.candidates.items()],
           "rng_state": rng_state(planner.np_random), "tree": dump_tree(planner.root)}
    print(spec, config, "horizon", out["horizon"], "nodes", len(CREATED), "openings", out["openings"], "plan", plan,
          flush=True)
    return out


def run_agent(m, tables, spec, config, seed, decisions):
    """`decisions` consecutive agent.plan() calls on one env: the receding horizon serves the rest of a plan."""
    agent = make_agent(make_env(spec, m, tables), config, seed)
    outs = [[int(a) for a in agent.plan(None)] for _ in range(decisions)]
    return {"env": spec, "config": config, "seed": seed, "decisions": outs,
            "rng_state": rng_state(agent.planner.np_random)}


def error_of(fn):
    try:
        fn()
    except Exception as e:              # noqa: BLE001 -- the reference's own exception is what is recorded
        return {"error": type(e).__name__, "message": str(e)}
    raise AssertionError("expected an error")


def main():
    m = np.load(os.path.join(HERE, "finite_mdps.npz"))
    tables = stochastic_mdps()
    trap_terminal = int(np.nonzero(m["trap_term"])[0][0])
    base = {k: v for k, v in BASELINE.items() if k != "env_preprocessors"}
    out = {"mdps": tables, "cases": {}, "agents": {}, "configs": {}, "errors": {}}
    cases = out["cases"]
    cases["hw3_baseline"] = run(m, tables, {"name": "highway", "seed": 3}, base, seed=0)
    cases["hw0_baseline"] = run(m, tables, {"name": "highway", "seed": 0}, base, seed=1)
    for budget in (10000, 50000):
        for gamma in (0.9, 0.7):
            cases["hw3_budget%d_gamma%s" % (budget, gamma)] = run(
                m, tables, {"name": "highway", "seed": 3}, {"budget": budget, "gamma": gamma}, seed=2)
    cases["large1_deterministic_budget10000"] = run(m, tables, {"name": "large1"}, {"budget": 10000, "gamma": 0.9},
                                                    seed=3)
    cases["stoch8_stochastic_budget10000"] = run(m, tables, {"name": "stoch8"}, {"budget": 10000, "gamma": 0.9},
                                                 seed=4)
    cases["stoch8_stochastic_budget50000_gamma0.7"] = run(m, tables, {"name": "stoch8"},
                                                          {"budget": 50000, "gamma": 0.7}, seed=5)
    cases["garnet12_sparse_budget10000"] = run(m, tables, {"name": "garnet12"}, {"budget": 10000, "gamma": 0.9},
                                               seed=6)
    cases["trap_terminal_root"] = run(m, tables, {"name": "trap", "state": trap_terminal},
                                      {"budget": 10000, "gamma": 0.9}, seed=7)
    cases["stoch8_terminal_root"] = run(m, tables, {"name": "stoch8", "state": 7}, {"budget": 10000, "gamma": 0.9},
                                        seed=8)
    # all rewards zero: every value ties, in the sort and among the candidates
    cases["stoch8_zero_rewards"] = run(m, tables, {"name": "stoch8", "zero_rewards": True},
                                       {"budget": 10000, "gamma": 0.9}, seed=9)
    cases["large1_zero_rewards"] = run(m, tables, {"name": "large1", "zero_rewards": True},
                                       {"budget": 10000, "gamma": 0.8}, seed=10)
    # two actions: the reference's range(1, n) expands action 1 only
    cases["trap_two_actions"] = run(m, tables, {"name": "trap"}, {"budget": 10000, "gamma": 0.9}, seed=11)
    cases["garnet1000_deterministic_budget200000"] = run(
        m, tables, {"name": "garnet", "states": 1000, "actions": 4, "seed": 0}, {"budget": 200000, "gamma": 0.9},
        seed=12)
    cases["stoch8_explicit_horizon"] = run(m, tables, {"name": "stoch8"}, {"horizon": 7, "gamma": 0.95}, seed=13)
    cases["hw1_explicit_horizon"] = run(m, tables, {"name": "highway", "seed": 1}, {"horizon": 4, "gamma": 0.8},
                                        seed=14)
    out["agents"]["stoch8_receding_horizon3"] = run_agent(
        m, tables, {"name": "stoch8"}, {"budget": 10000, "gamma": 0.9, "receding_horizon": 3}, seed=15, decisions=3)
    out["agents"]["hw2_receding_horizon3"] = run_agent(
        m, tables, {"name": "highway", "seed": 2}, {"budget": 10000, "gamma": 0.9, "receding_horizon": 3}, seed=16,
        decisions=3)

    def plan_with(config, spec):
        agent = make_agent(make_env(spec, m, tables), config, 0)
        return agent.planner.plan(agent.env, None)
    errs = out["errors"]
    errs["default_budget_highway"] = error_of(lambda: plan_with({}, {"name": "highway", "seed": 0}))
    errs["horizon_1"] = error_of(lambda: plan_with({"horizon": 1}, {"name": "stoch8"}))
    errs["one_action"] = error_of(lambda: plan_with({"budget": 10000}, {"name": "trap", "actions": 1}))
    errs["negative_budget"] = error_of(lambda: make_agent(make_env({"name": "stoch8"}, m, tables), {"budget": -10}, 0))
    errs["bad_row"] = error_of(lambda: plan_with({"budget": 10000, "gamma": 0.9}, {"name": "stoch8_bad_row"}))

    def subtree():
        agent = make_agent(make_env({"name": "garnet", "states": 1000, "actions": 4, "seed": 0}, m, tables),
                           {"budget": 10000, "step_strategy": "subtree"}, 0)
        for _ in range(2):
            agent.plan(None)
    errs["subtree_second_decision"] = error_of(subtree)

    # completed configs of the agent and its planner (the `__class__` key is left out)
    for name, cfg, spec in (("baseline_highway", BASELINE, {"name": "highway", "seed": 0}),
                            ("empty_finite", {}, {"name": "stoch8"}),
                            ("horizon_given", {"horizon": 5, "budget": 100, "gamma": 0.9}, {"name": "stoch8"}),
                            ("budget_200000_garnet", {"budget": 200000},
                             {"name": "garnet", "states": 1000, "actions": 4, "seed": 0})):
        agent = make_agent(make_env(spec, m, tables), cfg, 0)
        out["configs"][name] = {"config": cfg, "env": spec, "completed": json.loads(json.dumps(agent.config)),
                                "planner": json.loads(json.dumps(agent.planner.config))}
    with open(os.path.join(HERE, "golden_platypoos.json"), "w") as f:
        json.dump(out, f)
    print("PlaTyPOOS done")


if __name__ == "__main__":
    main()
