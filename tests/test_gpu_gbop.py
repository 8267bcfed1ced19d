"""GPU parity tests of GBOP-T (b2_gbop_plan): the device planner against the reference's StateAwarePlanner
(golden vectors from the unmodified reference) and the oracle restatement -- plan, node order, leaves left
after pruning, state value table, bit for bit."""
import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import planners
from tests.util import load_golden, load_mdps

pytestmark = pytest.mark.gpu
G = load_golden("golden_finite.json")
M = load_mdps()


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def mdp(name="large1", terminal=None):
    from rl_agents_b200.envs.finite_mdp import FiniteMDP
    term = M[name + "_term"] if terminal is None else terminal
    return FiniteMDP("deterministic", M[name + "_T"], M[name + "_R"], term)


@pytest.mark.parametrize("key", sorted(G["gbopt"]))
def test_gbopt_matches_the_reference_goldens(key):
    import torch
    from rl_agents_b200.engine.gbop import GBOPEngine
    g = G["gbopt"][key]
    eng = GBOPEngine(1, 5, g["budget"], g["gamma"], mdp())
    eng.plan(torch.tensor([0], dtype=torch.int32, device="cuda"))
    plans, res = eng.finish([np_random(g["seed"])])
    assert plans[0] == g["plan"]
    d = eng.tree_dict(0)
    sv = eng.state_values(0)
    assert all(sv[int(k)] == v for k, v in g["state_values"].items())
    leaves = np.nonzero(d["leaf"])[0]
    assert len(leaves) == g["n_leaves"] == int(res[0, 1]) and len(set(d["obs"].tolist())) == g["n_states"]
    assert int(d["depth"][leaves].sum()) == g["leaf_depth_sum"]
    assert sum(float(d["lower"][l]) for l in leaves) == g["leaf_lower_sum"]      # python floats: 3.12's sum() compensates


@pytest.mark.parametrize("variant", [dict(), dict(backup_aggregated_nodes=False), dict(prune_suboptimal_leaves=False),
                                     dict(accuracy=0.05), dict(terminal_reward=0.3, terminal=True)])
def test_gbopt_batch_vs_oracle(variant):
    """A batch of roots, the config switches of state_aware.py:79-86 and terminal states, against the oracle."""
    import torch
    from rl_agents_b200.engine.gbop import GBOPEngine
    variant = dict(variant)
    term = None
    if variant.pop("terminal", False):
        term = M["large1_term"].copy()
        term[[3, 17, 66, 91]] = True
    tr = variant.pop("terminal_reward", 0.0)
    roots = [0, 7, 42, 99, 3]
    eng = GBOPEngine(len(roots), 5, 400, 0.85, mdp(terminal=term), terminal_reward=tr, **variant)
    eng.plan(torch.tensor(roots, dtype=torch.int32, device="cuda"))
    plans, res = eng.finish([np_random(1) for _ in roots])
    for i, r in enumerate(roots):
        env = oenvs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"] if term is None else term, state=r)
        plan, t, state_values, leaves = planners.state_aware_plan(env, r, 400, 0.85, np_random(1), terminal_reward=tr,
                                                                  **variant)
        d = eng.tree_dict(i)
        assert plans[i] == plan, (i, r)
        assert d["parent"].tolist() == t.parent and d["action"].tolist() == t.action and d["count"].tolist() == t.count
        assert d["obs"].tolist() == t.obs and np.array_equal(d["lower"], np.array(t.lower))
        assert sorted(np.nonzero(d["leaf"])[0].tolist()) == sorted(leaves)
        sv = eng.state_values(i)
        default = 1 / (1 - 0.85)
        assert all(sv[s] == state_values.get(s, default) for s in range(100))


def test_gbopt_agent_plugin_surface():
    from rl_agents_b200.agents.tree_search.state_aware import StateAwarePlannerAgent
    from rl_agents_b200.envs import FiniteMDPEnv
    g = G["gbopt"]["large1_b500_g0.9"]
    agent = StateAwarePlannerAgent(FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"]),
                                   {"budget": g["budget"], "gamma": g["gamma"]})
    agent.seed(g["seed"])
    assert agent.plan(0) == g["plan"]
    assert agent.config["prune_suboptimal_leaves"] is True and agent.config["accuracy"] == 0


# ------------------------------------------------------------------ GBOP-D (graph_based.py) ----
@pytest.mark.parametrize("key", sorted(G["gbopd"]))
def test_gbopd_matches_the_reference_and_the_oracle(key):
    """accuracy = 0: plan, node set and both bounds of every node equal the UNMODIFIED reference's (the fixed
    point does not depend on the order in which the reference's parent SETS are iterated); default accuracy: equal
    to the oracle restatement (parents in ascending state id), the reference's plan, its bounds within `accuracy`."""
    import torch
    from rl_agents_b200.engine.gbop import GBOPDEngine
    from rl_agents_b200.engine.mcts import pcg64_words
    g = G["gbopd"][key]
    eng = GBOPDEngine(1, 5, g["budget"], g["gamma"], mdp(), g["accuracy"], g["sampling_timeout"])
    rng = np_random(g["seed"])
    eng.plan(torch.tensor([0], dtype=torch.int32, device="cuda"), pcg64_words(rng).reshape(1, -1))
    plans, res, words = eng.finish()
    nodes = eng.nodes(0)
    ref = {int(k): v for k, v in g["nodes"].items()}
    assert plans[0] == g["plan"] and set(nodes) == set(ref)
    assert all(nodes[s]["expanded"] == ref[s][2] for s in ref)
    if g["accuracy"] == 0:
        assert all(nodes[s]["lower"] == ref[s][0] and nodes[s]["upper"] == ref[s][1] for s in ref)
    else:
        assert all(abs(nodes[s]["lower"] - ref[s][0]) <= 10 * g["accuracy"] and
                   abs(nodes[s]["upper"] - ref[s][1]) <= 10 * g["accuracy"] for s in ref)
    orng = np_random(g["seed"])
    env = oenvs.LegacyStepEnv(oenvs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"]))
    plan, onodes = planners.graph_based_plan(env, 0, g["budget"], g["gamma"], orng, g["accuracy"], g["sampling_timeout"])
    assert plans[0] == plan and nodes == onodes
    from rl_agents_b200.engine.mcts import set_pcg64_words
    set_pcg64_words(rng, words[0])
    assert rng.bit_generator.state["state"] == orng.bit_generator.state["state"]     # same RNG consumption


def test_gbopd_agent_plugin_surface():
    from rl_agents_b200.agents.tree_search.graph_based import GraphBasedPlannerAgent
    from rl_agents_b200.envs import FiniteMDPEnv
    g = G["gbopd"]["large1_b500_g0.9_default"]
    agent = GraphBasedPlannerAgent(FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"]),
                                   {"budget": g["budget"], "gamma": g["gamma"]})
    agent.seed(g["seed"])
    assert agent.plan(0) == g["plan"]
    assert agent.config["accuracy"] == 1e-2 and agent.config["sampling_timeout"] == 100


# ------------------------------------------------------------------ batches, ties, overflow, errors ----
GB = load_golden("golden_gbop.json")


def table_mdp(T, R, term=None):
    from rl_agents_b200.envs.finite_mdp import FiniteMDP
    T = np.asarray(T, dtype=np.int64)
    term = np.zeros(T.shape[0], dtype=bool) if term is None else np.asarray(term, dtype=bool)
    return FiniteMDP("deterministic", T, np.asarray(R, dtype=np.float64), term)


def named_tables(name):
    """(T, R, terminal) of an MDP of finite_mdps.npz, golden_gbop.json or a generated family:
    garnet<S>_<A>: deterministic garnet (half the rewards 0); quant<S>_<A>: rewards in {0, 0.5};
    large1_term: a quarter of large1's states terminal."""
    if name in GB["mdps"]:
        m = GB["mdps"][name]
        return np.asarray(m["T"]), np.asarray(m["R"], dtype=np.float64), np.asarray(m["term"], dtype=bool)
    if name + "_T" in M.files:
        return M[name + "_T"], M[name + "_R"], M[name + "_term"]
    if name == "large1_term":
        term = np.random.default_rng(11).uniform(size=100) < 0.25
        return M["large1_T"], M["large1_R"], term
    S, A = map(int, name.lstrip("garnetquant").split("_"))
    if name.startswith("garnet"):
        T, R = oenvs.garnet(S, A, 1, seed=S + A, deterministic=True)
    else:
        rng = np.random.default_rng(S * 10 + A)
        T, R = rng.integers(0, S, size=(S, A)), rng.choice([0.0, 0.5], size=(S, A))
    return T, R, np.zeros(S, dtype=bool)


def f64_bytes(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.float64)).tobytes()


def roots_for(S, n):
    return [int(r) for r in (np.arange(n) * 7919 + 3) % S]


N_BATCH = 66          # not a multiple of the kernels' 4 trees per CTA: the last CTA has idle warps


# (mdp, budget, gamma, engine keywords): every config switch, A in {1, 2, 3, 8}, S up to 1200, tie-heavy rewards
GBOPT_BATCHES = [
    ("loop", 300, 0.9, dict()),
    ("large2", 200, 0.85, dict(backup_aggregated_nodes=False)),
    ("garnet1000_1", 60, 0.9, dict()),
    ("garnet1200_2", 120, 0.8, dict(prune_suboptimal_leaves=False)),
    ("garnet1000_3", 150, 0.9, dict(accuracy=0.05)),
    ("garnet1100_8", 240, 0.85, dict()),
    ("quantized6", 90, 0.9, dict()),
    ("quant40_4", 160, 0.9, dict(backup_aggregated_nodes=False)),
    ("quant40_4", 160, 0.9, dict(accuracy=0.05)),
    ("large1_term", 300, 0.85, dict(terminal_reward=0.3)),
]


@pytest.mark.parametrize("case", GBOPT_BATCHES, ids=lambda c: "%s_b%d_%s" % (c[0], c[1], "_".join(sorted(c[3])) or "default"))
def test_gbopt_batches_vs_oracle(case):
    """One launch of 66 roots per MDP against the oracle, exactly: plan (ties broken by the host walks on each
    tree's own generator), node arrays, lower bounds and state values as float64 bytes, leaf set, expansions."""
    import torch
    from rl_agents_b200.engine.gbop import GBOPEngine
    name, budget, gamma, kw = case
    T, R, term = named_tables(name)
    S, A = R.shape
    roots = roots_for(S, N_BATCH)
    eng = GBOPEngine(len(roots), A, budget, gamma, table_mdp(T, R, term), **kw)
    eng.plan(torch.tensor(roots, dtype=torch.int32, device="cuda"))
    rngs = [np_random(100 + i) for i in range(len(roots))]
    plans, res = eng.finish(rngs)
    default = 1 / (1 - gamma)
    for i, r in enumerate(roots):
        orng = np_random(100 + i)
        plan, t, state_values, leaves = planners.state_aware_plan(oenvs.FiniteMDPLite(T, R, term, state=r), r, budget,
                                                                  gamma, orng, **kw)
        d = eng.tree_dict(i)
        assert plans[i] == plan, (i, r)
        assert rngs[i].bit_generator.state == orng.bit_generator.state, (i, r)
        for f in ("parent", "action", "count", "depth", "obs"):
            assert d[f].tolist() == getattr(t, f), (i, f)
        assert f64_bytes(d["lower"]) == f64_bytes(t.lower), i
        assert sorted(np.nonzero(d["leaf"])[0].tolist()) == sorted(leaves), i
        assert f64_bytes(eng.state_values(i)) == f64_bytes([state_values.get(s, default) for s in range(S)]), i
        assert int(res[i, 8]) == sum(1 for n in t.n_children if n > 0) == budget // A
        assert int(res[i, 1]) == len(leaves) and int(res[i, 0]) == len(t.parent)
    assert not res[:, 4].any() and not res[:, 7].any()
    if name.startswith("quant"):
        assert (res[:, 6] >= 0).sum() > len(roots) // 2          # most trees stopped at a get_plan tie


@pytest.mark.parametrize("name,budget", [("trap", 200), ("loop", 300), ("large1", 300), ("garnet400_8", 400)])
@pytest.mark.parametrize("accuracy", [0, 1e-2])
def test_gbopd_batches_vs_oracle(name, budget, accuracy):
    """66 roots, each on its own seed, against the oracle (parents pushed in ascending id, like the device):
    plan, node set, both bounds as float64 bytes, expanded flags, expansion count, PCG64 words after the search."""
    import torch
    from rl_agents_b200.engine.gbop import GBOPDEngine
    from rl_agents_b200.engine.mcts import pcg64_words, set_pcg64_words
    T, R, term = named_tables(name)
    S, A = R.shape
    gamma = 0.9
    roots = roots_for(S, N_BATCH)
    eng = GBOPDEngine(len(roots), A, budget, gamma, table_mdp(T, R, term), accuracy)
    words = np.stack([pcg64_words(np_random(1000 + i)) for i in range(len(roots))])
    eng.plan(torch.tensor(roots, dtype=torch.int32, device="cuda"), words)
    plans, res, words_after = eng.finish()
    draws = 0
    for i, r in enumerate(roots):
        orng = np_random(1000 + i)
        env = oenvs.LegacyStepEnv(oenvs.FiniteMDPLite(T, R, term, state=r))
        plan, onodes = planners.graph_based_plan(env, r, budget, gamma, orng, accuracy)
        nodes = eng.nodes(i)
        assert plans[i] == plan, (i, r)
        assert sorted(nodes) == sorted(onodes), i
        ids = sorted(onodes)
        for f in ("lower", "upper"):
            assert f64_bytes([nodes[s][f] for s in ids]) == f64_bytes([onodes[s][f] for s in ids]), (i, f)
        assert [nodes[s]["expanded"] for s in ids] == [onodes[s]["expanded"] for s in ids], i
        assert int(res[i, 1]) == sum(n["expanded"] for n in onodes.values()) and int(res[i, 0]) == len(onodes)
        dev = np_random(0)
        set_pcg64_words(dev, words_after[i])
        assert dev.bit_generator.state == orng.bit_generator.state, (i, r)
        draws += dev.bit_generator.state != np_random(1000 + i).bit_generator.state
    assert not res[:, 7].any()
    if name == "trap":
        assert draws == len(roots)            # every tree broke sampling ties on its stream


def test_gbopt_agent_plans_the_overflow_case_like_the_reference():
    """GBOP-T on loop at budget 1000: one backup needs more queue entries than 64 x node capacity (see
    test_gbop_oracle.py); the engine grows its queue, the plan equals the reference's, and the cached engine keeps
    the grown queue for the next decision."""
    from rl_agents_b200.agents.tree_search.state_aware import StateAwarePlannerAgent
    from rl_agents_b200.envs import FiniteMDPEnv
    g = GB["gbopt"]["loop_b1000_g0.9"]
    agent = StateAwarePlannerAgent(FiniteMDPEnv(*named_tables("loop")), dict(g["config"]))
    agent.seed(g["seed"])
    assert agent.plan(0) == g["plan"]
    eng = agent.planner.engine
    assert eng.relaunches >= 1 and eng.queue_capacity > 64 * eng.capacity
    sv = agent.planner.state_values
    assert all(sv[int(k)] == v for k, v in g["state_values"].items())
    d = eng.tree_dict(0)
    leaves = np.nonzero(d["leaf"])[0]
    assert len(leaves) == g["n_leaves"] and int(d["depth"][leaves].sum()) == g["leaf_depth_sum"]
    assert sum(float(d["lower"][l]) for l in leaves) == g["leaf_lower_sum"]
    relaunches, capacity = eng.relaunches, eng.queue_capacity
    agent.seed(g["seed"])
    assert agent.plan(0) == g["plan"]
    assert agent.planner.engine is eng and (eng.relaunches, eng.queue_capacity) == (relaunches, capacity)


def test_gbopd_agent_plans_the_overflow_case_like_the_reference():
    from rl_agents_b200.agents.tree_search.graph_based import GraphBasedPlannerAgent
    from rl_agents_b200.envs import FiniteMDPEnv
    g = GB["gbopd"]["loop_b500_g0.9_acc0"]
    agent = GraphBasedPlannerAgent(FiniteMDPEnv(*named_tables("loop")), dict(g["config"]))
    agent.seed(g["seed"])
    assert agent.plan(0) == g["plan"]
    eng = agent.planner.engine
    assert eng.relaunches >= 1 and eng.queue_capacity > 256 * eng.n_states
    nodes = eng.nodes(0)
    assert {str(s): [n["lower"], n["upper"], n["expanded"]] for s, n in sorted(nodes.items())} == g["nodes"]
    st = agent.planner.np_random.bit_generator.state
    assert str(st["state"]["state"]) == g["rng_state"]["state"] and str(st["state"]["inc"]) == g["rng_state"]["inc"]
    relaunches = eng.relaunches
    agent.seed(g["seed"])
    assert agent.plan(0) == g["plan"] and agent.planner.engine is eng and eng.relaunches == relaunches


@pytest.mark.parametrize("name,budget", [("trap", 500), ("loop", 500)])
def test_gbopd_golden_accuracy0(name, budget):
    """GBOP-D on trap (rewards -1: no range check) and loop against the reference at accuracy 0."""
    import torch
    from rl_agents_b200.engine.gbop import GBOPDEngine
    from rl_agents_b200.engine.mcts import pcg64_words, set_pcg64_words
    g = GB["gbopd"]["%s_b%d_g0.9_acc0" % (name, budget)]
    eng = GBOPDEngine(1, len(GB["mdps"][name]["R"][0]), budget, 0.9, table_mdp(*named_tables(name)), 0)
    rng = np_random(g["seed"])
    eng.plan(torch.tensor([0], dtype=torch.int32, device="cuda"), pcg64_words(rng).reshape(1, -1))
    plans, res, words = eng.finish()
    assert plans[0] == g["plan"]
    assert {str(s): [n["lower"], n["upper"], n["expanded"]] for s, n in sorted(eng.nodes(0).items())} == g["nodes"]
    set_pcg64_words(rng, words[0])
    assert str(rng.bit_generator.state["state"]["state"]) == g["rng_state"]["state"]


@pytest.mark.parametrize("key", sorted(GB["gbopt"]))
def test_gbopt_matches_the_new_reference_goldens(key):
    """Ties on quantized rewards (the planner RNG after both get_plan walks), terminal states with a terminal
    reward, and loop's overflowing backups, against the reference."""
    import torch
    from rl_agents_b200.engine.gbop import GBOPEngine
    g = GB["gbopt"][key]
    c = g["config"]
    T, R, term = named_tables(g["mdp"])
    eng = GBOPEngine(1, R.shape[1], c["budget"], c["gamma"], table_mdp(T, R, term), c.get("terminal_reward", 0.0))
    eng.plan(torch.tensor([0], dtype=torch.int32, device="cuda"))
    rng = np_random(g["seed"])
    plans, res = eng.finish([rng])
    assert plans[0] == g["plan"] and bool(res[0, 6] >= 0) == g["tied"]
    st = rng.bit_generator.state
    assert str(st["state"]["state"]) == g["rng_state"]["state"] and int(st["has_uint32"]) == g["rng_state"]["has_uint32"]
    sv = eng.state_values(0)
    assert all(sv[int(k)] == v for k, v in g["state_values"].items())
    d = eng.tree_dict(0)
    leaves = np.nonzero(d["leaf"])[0]
    assert len(leaves) == g["n_leaves"] == int(res[0, 1]) and len(set(d["obs"].tolist())) == g["n_states"]
    assert int(d["depth"][leaves].sum()) == g["leaf_depth_sum"]
    assert sum(float(d["lower"][l]) for l in leaves) == g["leaf_lower_sum"]


def test_small_queues_grow_to_the_default_engines_results():
    """queue_factor=1 forces overflows and relaunches; the grown engines equal the default-sized ones bit for bit,
    and a second search on the grown engine does not relaunch."""
    import torch
    from rl_agents_b200.engine.gbop import GBOPDEngine, GBOPEngine
    from rl_agents_b200.engine.mcts import pcg64_words
    T, R, term = named_tables("loop")          # budget 600: up to 1053 entries in one backup, 601 nodes
    roots = roots_for(4, N_BATCH)
    rt = torch.tensor(roots, dtype=torch.int32, device="cuda")
    out = []
    for qf in (64, 1):
        eng = GBOPEngine(len(roots), 3, 600, 0.9, table_mdp(T, R, term), queue_factor=qf)
        eng.plan(rt)
        plans, res = eng.finish([np_random(i) for i in range(len(roots))])
        trees = [eng.tree_dict(i) for i in range(len(roots))]
        out.append((plans, res, trees, [eng.state_values(i) for i in range(len(roots))], eng))
    (p0, r0, t0, s0, e0), (p1, r1, t1, s1, e1) = out
    assert e0.relaunches == 0 and e1.relaunches >= 1 and e1.queue_capacity > e1.capacity
    assert e1.ws_per_tree > 4 * e1.queue_capacity
    assert p0 == p1 and np.array_equal(r0[:, :9], r1[:, :9])         # the words the kernel writes
    for a, b, sa, sb in zip(t0, t1, s0, s1):
        assert all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in a)
        assert sa.tobytes() == sb.tobytes()
    n = e1.relaunches
    e1.plan(rt)
    assert e1.finish([np_random(i) for i in range(len(roots))])[0] == p0 and e1.relaunches == n

    T, R, term = named_tables("large1")
    roots = roots_for(100, N_BATCH)
    rt = torch.tensor(roots, dtype=torch.int32, device="cuda")
    words = np.stack([pcg64_words(np_random(50 + i)) for i in range(len(roots))])
    out = []
    for qf in (256, 1):
        eng = GBOPDEngine(len(roots), 5, 500, 0.9, table_mdp(T, R, term), 0, queue_factor=qf)
        eng.plan(rt, words)
        plans, res, w = eng.finish()
        out.append((plans, res[:, :8], w, eng.lower.cpu().numpy(), eng.upper.cpu().numpy(), eng.flags.cpu().numpy(),
                    eng))
    a, b = out
    assert a[-1].relaunches == 0 and b[-1].relaunches >= 1
    assert a[0] == b[0]
    for x, y in zip(a[1:-1], b[1:-1]):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes()
    n = b[-1].relaunches
    b[-1].plan(rt, words)
    assert b[-1].finish()[2].tobytes() == a[2].tobytes() and b[-1].relaunches == n


def test_gbopt_reward_range_error_only_when_reached():
    """The reference raises ValueError when an expansion meets a reward outside [0, 1]: on trap, and on large1
    with one reward 1.5 in a state the search expands, but not with it in a state the search never expands."""
    import torch
    from rl_agents_b200.engine.gbop import GBOPEngine
    e = GB["errors"]["gbopt_trap_b100_g0.9"]
    T, R, term = named_tables("trap")
    eng = GBOPEngine(1, 2, 100, 0.9, table_mdp(T, R, term))
    eng.plan(torch.tensor([0], dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError, match=e["message"].replace("[", r"\[").replace("]", r"\]")):
        eng.finish([np_random(0)])
    assert int(eng.result[0, 4]) == 1
    T, R, term = named_tables("large1")
    _, t, _, _ = planners.state_aware_plan(oenvs.FiniteMDPLite(T, R, term, state=0), 0, 100, 0.9, np_random(0))
    expanded = {t.obs[n] for n in range(len(t.parent)) if t.n_children[n] > 0}
    s_in, s_out = min(expanded - {0}), min(set(range(100)) - expanded)
    for s, raises in ((s_in, True), (s_out, False)):
        R2 = R.copy()
        R2[s, 2] = 1.5
        eng = GBOPEngine(1, 5, 100, 0.9, table_mdp(T, R2, term))
        eng.plan(torch.tensor([0], dtype=torch.int32, device="cuda"))
        if raises:
            with pytest.raises(ValueError):
                eng.finish([np_random(0)])
            with pytest.raises(ValueError):
                planners.state_aware_plan(oenvs.FiniteMDPLite(T, R2, term, state=0), 0, 100, 0.9, np_random(0))
        else:
            plan, _, _, _ = planners.state_aware_plan(oenvs.FiniteMDPLite(T, R2, term, state=0), 0, 100, 0.9,
                                                      np_random(0))
            assert eng.finish([np_random(0)])[0][0] == plan


def test_c_abi_argument_errors():
    import ctypes
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.gbop import GBOPDEngine, GBOPEngine
    T, R, term = named_tables("large1")
    rt = torch.tensor([0], dtype=torch.int32, device="cuda")
    eng = GBOPEngine(1, 5, 100, 0.9, table_mdp(T, R, term))
    lib = eng.lib

    def gbopt(**changes):
        cfg = _lib.GBOPConfig.from_buffer_copy(eng.cfg)
        for k, v in changes.items():
            if k.startswith("mdp_"):
                setattr(cfg.mdp, k[4:], v)
            else:
                setattr(cfg, k, v)
        return lib.b2_gbop_plan(ctypes.byref(cfg), _lib.ptr(rt), eng.tree, _lib.ptr(eng.workspace),
                                _lib.ptr(eng.plan_buf), _lib.ptr(eng.result), _lib.current_stream())

    for changes, msg in ((dict(n_actions=0), "n_actions must be in 1..8"), (dict(n_actions=9), "n_actions must be in 1..8"),
                         (dict(node_capacity=eng.capacity - 1), "node_capacity too small"),
                         (dict(mdp_transition=None), "finite MDP tables missing"),
                         (dict(mdp_reward=None), "finite MDP tables missing"),
                         (dict(queue_capacity=0), "capacities must be positive")):
        with pytest.raises(_lib.B2Error, match=msg):
            _lib.check(gbopt(**changes))
    cfg = _lib.GBOPConfig.from_buffer_copy(eng.cfg)
    cfg.queue_capacity = 0
    assert lib.b2_gbop_workspace_bytes(ctypes.byref(cfg)) < 0
    _lib.check(gbopt())                       # the unchanged config still launches
    eng.finish()

    deng = GBOPDEngine(1, 5, 100, 0.9, table_mdp(T, R, term))

    def gbopd(**changes):
        cfg = _lib.GBOPDConfig.from_buffer_copy(deng.cfg)
        for k, v in changes.items():
            if k.startswith("mdp_"):
                setattr(cfg.mdp, k[4:], v)
            else:
                setattr(cfg, k, v)
        return lib.b2_gbopd_plan(ctypes.byref(cfg), _lib.ptr(rt), _lib.ptr(deng.lower), _lib.ptr(deng.upper),
                                 _lib.ptr(deng.flags), _lib.ptr(deng.queue), _lib.ptr(deng.rng), _lib.ptr(deng.plan_buf),
                                 _lib.ptr(deng.result), _lib.current_stream())

    for changes, msg in ((dict(n_actions=0), "n_actions must be in 1..8"), (dict(n_actions=9), "n_actions must be in 1..8"),
                         (dict(mdp_transition=None), "finite MDP tables missing"),
                         (dict(mdp_n_actions=4), "finite MDP tables missing"),
                         (dict(rev_ptr=None), "reverse transition CSR missing"),
                         (dict(queue_capacity=0), "capacities must be positive"),
                         (dict(sampling_timeout=0), "bad batch / budget")):
        with pytest.raises(_lib.B2Error, match=msg):
            _lib.check(gbopd(**changes))


def test_queue_growth_stops_at_int32_indexing():
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.gbop import QUEUE_CAPACITY_MAX, grown_queue_capacity
    assert grown_queue_capacity(1000, "GBOP") == 2000
    assert grown_queue_capacity(2 ** 30 + 5, "GBOP") == QUEUE_CAPACITY_MAX == 2 ** 31 - 1
    with pytest.raises(_lib.B2Error, match="int32"):
        grown_queue_capacity(QUEUE_CAPACITY_MAX, "GBOP-D")


@pytest.mark.parametrize("agent_name", ["state_aware.StateAwarePlannerAgent", "graph_based.GraphBasedPlannerAgent"])
def test_gbop_agents_refuse_highway(agent_name):
    import importlib
    from rl_agents_b200.envs.highway_lite import HighwayLiteEnv
    mod, cls = agent_name.split(".")
    agent_cls = getattr(importlib.import_module("rl_agents_b200.agents.tree_search." + mod), cls)
    agent = agent_cls(HighwayLiteEnv(seed=0), {"budget": 50, "gamma": 0.8})
    with pytest.raises(TypeError):
        agent.plan(HighwayLiteEnv(seed=0))
