"""Generate tests/golden/golden_sparse_sampling.json by running the UNMODIFIED reference SparseSamplingAgent
(rl_agents/agents/tree_search/sparse_sampling.py) on the oracle env models, through the same shims as the BRUE and
MDP-GapE goldens (oracle.envs.LegacyStepEnv for the 4-tuple `step`, oracle.ref_loader.legacy_np_random for
`np_random.randint`).

The stochastic finite MDPs the cases run on are stored in the output, so the tests need nothing else.  Needs the
reference tree (oracle.ref_loader.REFERENCE_ROOT), so the output is committed and the tests only read it.  Writes only
golden_sparse_sampling.json, reproducibly byte for byte.  Usage:  python tests/golden/make_golden_sparse_sampling.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_loader  # noqa: E402
from oracle import envs  # noqa: E402
from oracle.sparse_sampling import tree_digest  # noqa: E402

ref_loader.load_reference()
from rl_agents.agents.tree_search import sparse_sampling as ref_ss  # noqa: E402

CREATED = []


def _instrument(cls):
    """Record node creation order at run time (sources stay unmodified)."""
    orig = cls.__init__

    def init(self, *a, **k):
        orig(self, *a, **k)
        CREATED.append(self)
    cls.__init__ = init


for _cls in (ref_ss.DecisionNode, ref_ss.ChanceNode):
    _instrument(_cls)


def stochastic_mdps():
    """The stochastic tables of the cases, as JSON-ready lists."""
    rng = np.random.default_rng(2024)
    # dense "stochastic" MDP: 8 states, 3 actions, about 40 % zero entries per row, state 7 terminal
    p = rng.uniform(size=(8, 3, 8))
    p[p < 0.4] = 0.0
    p[:, :, 0] += 0.05                      # no empty row
    p /= p.sum(axis=-1, keepdims=True)
    stoch8 = {"mode": "stochastic", "transition": p, "reward": rng.uniform(size=(8, 3)),
              "terminal": np.arange(8) == 7}
    # "sparse" garnet (oracle.envs.garnet): 12 states, 3 actions, 4 successors; the root's rows repeat a next state
    # and hold zero-probability entries, so first-visit merging and searchsorted's "right" side both matter
    gp, gn, gr = envs.garnet(12, 3, 4, seed=3)
    gn[0, 0] = [4, 4, 9, 1]
    gp[0, 0] = [0.25, 0.25, 0.0, 0.5]
    gn[0, 1] = [2, 7, 2, 7]
    gp[0, 1] = [0.0, 0.5, 0.0, 0.5]
    garnet = {"mode": "sparse", "transition": gp, "next": gn, "reward": gr, "terminal": np.zeros(12, bool)}
    # a bad probability row at the root (a negative entry) ...
    bad = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in stoch8.items()}
    bad["transition"][0, 1] = 0.0
    bad["transition"][0, 1, :2] = [-0.25, 1.25]
    # ... and a NaN row in a state no sample can reach (states 0-5 lead only to 0-5)
    blocked = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in stoch8.items()}
    blocked["transition"][:6, :, 6:] = 0.0
    blocked["transition"][:6, :, 0] += 0.1
    blocked["transition"][:6] /= blocked["transition"][:6].sum(axis=-1, keepdims=True)
    blocked["transition"][6, 0, :] = np.nan
    out = {"stoch8": stoch8, "garnet12": garnet, "stoch8_bad_root_row": bad, "stoch8_unreached_nan_row": blocked}
    return {name: {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in m.items()}
            for name, m in out.items()}


def dump_tree(root):
    """Creation-order dump: a chance node's key is its action; a decision node's key is the observed next state
    (int(str(obs))) on a finite MDP and -1 on HighwayLite and at the root.  Every node's children must be in
    creation order (dict insertion order)."""
    def top(n):
        while n.parent is not None:
            n = n.parent
        return n
    nodes = [n for n in CREATED if top(n) is root]
    assert nodes[0] is root
    ids = {id(n): i for i, n in enumerate(nodes)}
    out = {k: [] for k in ("parent", "kind", "key", "depth", "count", "value")}
    for n in nodes:
        chance = isinstance(n, ref_ss.ChanceNode)
        p = n.parent
        out["parent"].append(ids[id(p)] if p is not None else -1)
        out["kind"].append(1 if chance else 0)
        if p is None:
            key = -1
        else:
            key = next(k for k, c in p.children.items() if c is n)
            key = int(key) if chance or not isinstance(n.state.unwrapped, envs.HighwayLite) else -1
        out["key"].append(key)
        out["depth"].append(int(n.depth))
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


def run(m, tables, spec, config, seed=0, decisions=1):
    agent = ref_ss.SparseSamplingAgent(envs.LegacyStepEnv(make_env(spec, m, tables)), dict(config))
    agent.planner.np_random, _ = ref_loader.legacy_np_random(seed)
    plans = []
    for _ in range(decisions):
        del CREATED[:]
        plans.append([int(a) for a in agent.plan(None)])
    root = agent.planner.root
    n_actions = agent.env.action_space.n
    root_q = [None] * n_actions
    for a, c in root.children.items():
        root_q[int(a)] = float(c.value)
    tree = dump_tree(root)
    chance = sum(tree["kind"])
    out = {"env": spec, "config": config, "seed": seed, "plan": plans[-1], "root_q": root_q,
           "chance_nodes": chance, "samples": chance * config["C"], "rng_state": rng_state(agent.planner.np_random),
           "tree": tree_digest(tree)}
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
    with open(os.path.join(ref_loader.REFERENCE_ROOT, "scripts/configs/FiniteMDPEnv/agents/sparse_sampling.json")) as f:
        ss_json = json.load(f)
    shipped = {k: v for k, v in ss_json.items() if k != "__class__"}         # gamma 0.7, horizon 3, C 3
    stoch8 = {"name": "stoch8"}
    trap_terminal = int(np.nonzero(m["trap_term"])[0][0])

    out = {"mdps": tables, "cases": {}, "configs": {}, "errors": {}}
    cases = out["cases"]
    cases["stoch8_shipped"] = run(m, tables, stoch8, shipped)
    cases["garnet12_sparse_shipped"] = run(m, tables, {"name": "garnet12"}, shipped, seed=1)
    cases["large1_deterministic_shipped"] = run(m, tables, {"name": "large1"}, shipped, seed=2)
    cases["trap_deterministic_shipped"] = run(m, tables, {"name": "trap"}, shipped, seed=3)
    # `done` is ignored: a terminal root is planned through like any other state
    cases["trap_terminal_root_shipped"] = run(m, tables, {"name": "trap", "state": trap_terminal}, shipped, seed=4)
    cases["stoch8_terminal_root_shipped"] = run(m, tables, {"name": "stoch8", "state": 7}, shipped, seed=4)
    # all rewards zero: every root value ties and get_plan draws choice(indices)
    cases["stoch8_zero_rewards_shipped"] = run(m, tables, {"name": "stoch8", "zero_rewards": True}, shipped, seed=5)
    cases["stoch8_h1_c3_g0.9"] = run(m, tables, stoch8, {"gamma": 0.9, "horizon": 1, "C": 3}, seed=6)
    cases["stoch8_h3_c1_g0.9"] = run(m, tables, stoch8, {"gamma": 0.9, "horizon": 3, "C": 1}, seed=7)
    cases["stoch8_h4_c5_g0.9"] = run(m, tables, stoch8, {"gamma": 0.9, "horizon": 4, "C": 5}, seed=8)
    cases["garnet12_sparse_h4_c2_g0.95"] = run(m, tables, {"name": "garnet12", "state": 5},
                                               {"gamma": 0.95, "horizon": 4, "C": 2}, seed=9)
    cases["stoch8_unreached_nan_row_shipped"] = run(m, tables, {"name": "stoch8_unreached_nan_row"}, shipped, seed=10)
    for s in range(4):
        cases["hw%d_shipped" % s] = run(m, tables, {"name": "highway", "seed": s}, shipped, seed=20 + s)
    cases["hw1_h2_c2_g0.8"] = run(m, tables, {"name": "highway", "seed": 1}, {"gamma": 0.8, "horizon": 2, "C": 2},
                                  seed=24)
    # three consecutive decisions of one agent: the planner's np_random carries on
    cases["stoch8_three_decisions"] = run(m, tables, stoch8, dict(shipped, receding_horizon=3), seed=11, decisions=3)
    for k, c in cases.items():
        print(k, "plan", c["plan"], "nodes", c["tree"]["n_nodes"], "chance", c["chance_nodes"])

    def plan_with(config, spec=stoch8):
        agent = ref_ss.SparseSamplingAgent(envs.LegacyStepEnv(make_env(spec, m, tables)), config)
        agent.planner.np_random, _ = ref_loader.legacy_np_random(0)
        return agent.plan(None)
    errs = out["errors"]
    errs["horizon_zero"] = error_of(lambda: plan_with({"horizon": 0, "C": 3}))
    errs["horizon_negative"] = error_of(lambda: plan_with({"horizon": -1, "C": 1}))
    errs["c_zero"] = error_of(lambda: plan_with({"horizon": 2, "C": 0}))
    errs["missing_horizon"] = error_of(lambda: plan_with({"C": 3}))
    errs["missing_c"] = error_of(lambda: plan_with({"horizon": 3}))
    errs["bad_root_row"] = error_of(lambda: plan_with(dict(shipped), {"name": "stoch8_bad_root_row"}))
    # message of a RecursionError is platform text: keep its type only
    errs["horizon_negative"]["message"] = None

    # completed configs of the agent and its planner, as agent_factory builds them (the `__class__` key is left in)
    for name, cfg in (("empty", {}), ("sparse_sampling_json", ss_json)):
        agent = ref_ss.SparseSamplingAgent(make_env(stoch8, m, tables), json.loads(json.dumps(cfg)))
        completed = {k: v for k, v in agent.config.items() if k != "__class__"}
        planner = {k: v for k, v in agent.planner.config.items() if k != "__class__"}
        out["configs"][name] = {"config": cfg, "completed": json.loads(json.dumps(completed)),
                                "planner": json.loads(json.dumps(planner))}
    with open(os.path.join(HERE, "golden_sparse_sampling.json"), "w") as f:
        json.dump(out, f)
    print("sparse sampling done")


if __name__ == "__main__":
    main()
