"""GPU tests of MCTS with double progressive widening (b2_mcts_dpw_plan, csrc/mcts_dpw.cu): the kernel against the
reference's goldens (tests/golden/golden_mcts_dpw.json) and against the oracle restatement (oracle/mcts_dpw.py), the
error paths, the agent surface and the batched evaluation branch.

Every comparison is exact: structure, keys, counts, the float64 bytes of every node's value (the digests hash them),
the plan, the env steps and the RNG stream position."""
import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import mcts_dpw as dpw
from oracle import ref_loader
from tests.test_mcts_dpw_oracle import G, M, case_env, completed_planner_config, rng_state

pytestmark = pytest.mark.gpu


def engine_for(env, cfg, n_trees):
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    from rl_agents_b200.engine.mcts_dpw import MCTSDPWEngine
    finite = isinstance(env, oenvs.FiniteMDPLite)
    return MCTSDPWEngine(_lib.ENV_FINITE if finite else _lib.ENV_HIGHWAY, n_trees, env.action_space.n, cfg["episodes"],
                         cfg["horizon"], cfg["gamma"], cfg["temperature"], cfg["k_action"], cfg["alpha_action"],
                         cfg["k_state"], cfg["alpha_state"], closed_loop=cfg["closed_loop"],
                         mdp=env.mdp if finite else None,
                         rollout_policy=MCTSAgent.policy_factory(cfg["rollout_policy"]))


def roots(envs_):
    import torch
    if isinstance(envs_[0], oenvs.FiniteMDPLite):
        return torch.tensor([e.mdp.state for e in envs_], dtype=torch.int32, device="cuda")
    return torch.from_numpy(np.stack([e.state.pack() for e in envs_]).astype(np.int32)).cuda()


def pcg64_of(seeds):
    from rl_agents_b200.engine.mcts import pcg64_words
    return np.stack([pcg64_words(ref_loader.legacy_np_random(s)[0]) for s in seeds])


def words_state(words):
    from rl_agents_b200.engine.mcts import set_pcg64_words
    g = np.random.Generator(np.random.PCG64(0))
    set_pcg64_words(g, words)
    return rng_state(g)


def device_digest(eng, i):
    d = eng.tree_dict(i)
    return dpw.tree_digest({f: d[f].tolist() for f in dpw.INT_FIELDS + dpw.FLOAT_FIELDS})


def run_batch_against_oracle(envs_, cfg, seeds):
    """One launch over all trees; every tree equals its own oracle run, value bytes included."""
    eng = engine_for(envs_[0], cfg, len(envs_))
    eng.plan(roots(envs_), pcg64_of(seeds))
    plans, res, words = eng.finish()
    for i, (env, s) in enumerate(zip(envs_, seeds)):
        rng = ref_loader.legacy_np_random(s)[0]
        action, t, steps = dpw.mcts_dpw_plan(env, cfg, rng)
        assert plans[i] == [action], i
        assert (int(res[i, 0]), int(res[i, 1]), int(res[i, 2])) == (len(t), cfg["episodes"], steps), i
        assert words_state(words[i]) == rng_state(rng), i
        assert device_digest(eng, i) == dpw.tree_digest(dpw.tree_dict(t)), i
    return res


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_kernel_matches_reference_golden(key):
    """Each golden case, consecutive decisions included: plan, node count, env steps, RNG position and the tree digest
    (integer fields and the float64 bytes of `value`) equal the reference's."""
    g = G["cases"][key]
    cfg = completed_planner_config(g["config"])
    env = case_env(g["env"])
    eng = engine_for(env, cfg, 1)
    words = pcg64_of([g["seed"]])
    plans = []
    for _ in range(len(g.get("plans", [g["plan"]]))):
        eng.plan(roots([env]), words)
        p, res, words = eng.finish()
        plans.append(p[0][0])
    assert plans == g.get("plans", [g["plan"]])
    assert (int(res[0, 0]), int(res[0, 1]), int(res[0, 2])) == (g["tree"]["n_nodes"], g["episodes"], g["steps"])
    assert (int(res[0, 3]), int(res[0, 4]), int(res[0, 5])) == (g["plan"], 0, -1)
    assert words_state(words[0]) == g["rng_state"]
    assert device_digest(eng, 0) == g["tree"]


def mixed_finite_mdp():
    """stoch8 ("stochastic"), garnet12 ("sparse"), large1's first three actions and trap's two plus a copy of its
    second (deterministic) side by side in one "sparse" table of width 8: next = arange for the stochastic rows,
    zero-probability padding for the garnet, probability one on the successor for the deterministic rows.
    -> (env factory by root state, state offsets)."""
    st, ga = G["mdps"]["stoch8"], G["mdps"]["garnet12"]
    parts_p, parts_n, parts_r, parts_t, offsets, base = [], [], [], [], [], 0
    sp = np.array(st["transition"])
    parts_p.append(sp)
    parts_n.append(np.broadcast_to(np.arange(8), sp.shape) + base)
    parts_r.append(np.array(st["reward"]))
    parts_t.append(np.array(st["terminal"]))
    offsets.append(base)
    base += 8
    gp, gn = np.array(ga["transition"]), np.array(ga["next"])
    parts_p.append(np.concatenate([gp, np.zeros(gp.shape[:2] + (4,))], axis=-1))
    parts_n.append(np.concatenate([gn, gn], axis=-1) + base)
    parts_r.append(np.array(ga["reward"]))
    parts_t.append(np.array(ga["terminal"]))
    offsets.append(base)
    base += 12
    for name in ("large1", "trap"):
        T, R = M[name + "_T"], M[name + "_R"]
        T, R = (T[:, :3], R[:, :3]) if T.shape[1] >= 3 else (T[:, [0, 1, 1]], R[:, [0, 1, 1]])
        p = np.zeros(T.shape + (8,))
        p[..., 0] = 1.0
        parts_p.append(p)
        parts_n.append(np.repeat(T[..., None], 8, axis=-1) + base)
        parts_r.append(R)
        parts_t.append(M[name + "_term"])
        offsets.append(base)
        base += T.shape[0]
    P, N, R, term = (np.concatenate(x) for x in (parts_p, parts_n, parts_r, parts_t))
    return (lambda s: oenvs.FiniteMDPLite(P, R, term, mode="sparse", nxt=N, state=s)), offsets


@pytest.mark.parametrize("config", [
    {"horizon": 6, "episodes": 120},
    {"horizon": 6, "episodes": 120, "closed_loop": True},
    {"horizon": 5, "episodes": 100, "closed_loop": True, "k_state": 2, "alpha_state": 0.5, "k_action": 1,
     "alpha_action": 0.5, "temperature": 2.5},
    {"horizon": 4, "episodes": 80, "closed_loop": True, "k_state": 0.5, "alpha_state": 0.2, "k_action": 10,
     "rollout_policy": {"type": "preference", "action": 2, "ratio": 3}},
], ids=["open", "closed", "closed_k2_a0.5", "closed_k0.5_a0.2_pref"])
def test_batch_of_256_mixed_finite_trees_equals_the_oracle(config):
    make, off = mixed_finite_mdp()
    starts = [off[0], off[0] + 7, off[1], off[1] + 5, off[2], off[2] + 37, off[3], off[3] + 2]
    envs_ = [make(starts[i % len(starts)]) for i in range(256)]
    res = run_batch_against_oracle(envs_, completed_planner_config(config), list(range(256)))
    assert len(set(res[:, 0].tolist())) > 5


def test_deterministic_mode_mdp_batch_equals_the_oracle():
    envs_ = [oenvs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"], state=s) for s in range(32)]
    run_batch_against_oracle(envs_, completed_planner_config({"horizon": 5, "episodes": 100, "closed_loop": True}),
                             list(range(32)))


def test_highway_batch_of_64_scenes_equals_the_oracle():
    cfg = completed_planner_config({"horizon": 5, "episodes": 30})
    run_batch_against_oracle([oenvs.HighwayLite(seed=s) for s in range(64)], cfg, [100 + s for s in range(64)])


def test_one_decision_at_budget_5000_equals_the_oracle():
    cfg = completed_planner_config({"budget": 5000})
    assert cfg["episodes"] * cfg["horizon"] <= 5000 and cfg["episodes"] > 100
    run_batch_against_oracle([oenvs.HighwayLite(seed=7)], cfg, [3])
    run_batch_against_oracle([case_env({"name": "stoch8"})], dict(cfg, closed_loop=True), [4])


def test_error_paths():
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPWAgent
    from rl_agents_b200.engine.mcts_dpw import MCTSDPWEngine
    from rl_agents_b200.envs import FiniteMDPEnv
    big = completed_planner_config({"horizon": 6, "episodes": 200})
    # a rejected probability row that a sample reaches: numpy's own ValueError, engine and agent alike
    bad = case_env({"name": "stoch8_bad_row"})
    eng = engine_for(bad, big, 1)
    eng.plan(roots([bad]), pcg64_of([0]))
    with pytest.raises(ValueError) as e:
        eng.finish()
    assert str(e.value) == G["errors"]["bad_row"]["message"]
    assert int(eng.result[0, 4].item()) == 2 and int(eng.result[0, 5].item()) == 5 * 3 + 0
    t = G["mdps"]["stoch8_bad_row"]
    agent = MCTSDPWAgent(FiniteMDPEnv(np.array(t["transition"]), np.array(t["reward"]), np.array(t["terminal"]),
                                      mode="stochastic"), {"horizon": 6, "episodes": 200})
    with pytest.raises(ValueError, match="non-negative"):
        agent.plan(0)
    # a NaN row that no sample reaches (state 8, probability 0 everywhere) plans as the oracle does
    st = G["mdps"]["stoch8"]
    P = np.zeros((9, 3, 9))
    P[:8, :, :8] = np.array(st["transition"])
    P[8] = np.nan
    R = np.concatenate([np.array(st["reward"]), np.zeros((1, 3))])
    term = np.concatenate([np.array(st["terminal"]), [False]])
    env = oenvs.FiniteMDPLite(P, R, term, mode="stochastic")
    run_batch_against_oracle([env], big, [1])
    # an exhausted node arena is a B2Error (it cannot happen at the engine's capacity of 1 + 2 * episodes)
    with pytest.raises(_lib.B2Error, match="exhausted"):
        eng._check(np.array([[3, 1, 5, -1, 1, -1, 0, 0]], dtype=np.int32))
    # the engine refuses what the reference cannot plan, before any device work
    with pytest.raises(ValueError, match="horizon"):
        MCTSDPWEngine(_lib.ENV_HIGHWAY, 1, 5, 10, 0, 0.9)
    with pytest.raises(ValueError, match="MiB"):
        MCTSDPWEngine(_lib.ENV_HIGHWAY, 1, 5, 5000, 4, 0.9)
    with pytest.raises(ZeroDivisionError):
        MCTSDPWEngine(_lib.ENV_HIGHWAY, 1, 5, 10, 4, 0.9, alpha_state=-1.0)
    with pytest.raises(NotImplementedError):
        MCTSDPWEngine(_lib.ENV_INTERSECTION, 1, 3, 10, 4, 0.9)
    # a decision node that can neither widen nor select (k_action < 0) raises the reference's message
    neg = completed_planner_config({"horizon": 3, "episodes": 4, "k_action": -1})
    env = case_env({"name": "stoch8"})
    eng = engine_for(env, neg, 1)
    eng.plan(roots([env]), pcg64_of([0]))
    with pytest.raises(ValueError, match="zero-size array"):
        eng.finish()
    # the C ABI refuses what the engine refuses
    eng = engine_for(env, big, 1)
    eng.cfg.env_kind = _lib.ENV_INTERSECTION
    with pytest.raises(_lib.B2Error, match="env_kind"):
        eng.plan(roots([env]), pcg64_of([0]))
    eng.cfg.env_kind, eng.cfg.node_capacity = _lib.ENV_FINITE, 2 * big["episodes"]
    with pytest.raises(_lib.B2Error, match="node_capacity"):
        eng.plan(roots([env]), pcg64_of([0]))
    eng.cfg.node_capacity, eng.cfg.horizon = 1 + 2 * big["episodes"], 0
    with pytest.raises(_lib.B2Error, match="horizon"):
        eng.plan(roots([env]), pcg64_of([0]))


def test_agent_surface_matches_reference():
    """On FiniteMDPEnv in all three modes and on HighwayLite: plans and RNG position equal the reference's planner;
    act returns an action; seed / reset as the reference's; consecutive decisions carry the planner's stream on."""
    from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPWAgent
    from rl_agents_b200.envs import FiniteMDPEnv, HighwayLiteEnv

    def finite_env(name):
        t = G["mdps"].get(name)
        if t is None:
            return FiniteMDPEnv(M[name + "_T"], M[name + "_R"], M[name + "_term"])
        return FiniteMDPEnv(np.array(t["transition"]), np.array(t["reward"]), np.array(t["terminal"]), mode=t["mode"],
                            nxt=None if "next" not in t else np.array(t["next"]))
    for key, name in (("stoch8_h6_e200", "stoch8"), ("garnet12_closed_loop_h6_e200", "garnet12"),
                      ("large1_deterministic_h6_e200", "large1"), ("stoch8_default", "stoch8")):
        g = G["cases"][key]
        agent = MCTSDPWAgent(finite_env(name), dict(g["config"]))
        assert agent.seed(g["seed"]) == [g["seed"]]
        assert agent.act(0) == g["plan"], key
        assert rng_state(agent.planner.np_random) == g["rng_state"], key
    # reset() keeps the RNG stream; seed() restarts it
    g = G["cases"]["stoch8_h6_e200"]
    agent = MCTSDPWAgent(finite_env("stoch8"), dict(g["config"]))
    agent.seed(g["seed"])
    first = agent.plan(0)
    agent.reset()
    second = agent.plan(0)
    agent.seed(g["seed"])
    assert agent.plan(0) == first == [g["plan"]] and len(second) == 1
    # receding_horizon 3 still replans at every call: three decisions equal the reference planner's three
    g = G["cases"]["stoch8_three_decisions"]
    agent = MCTSDPWAgent(finite_env("stoch8"), dict(g["config"], receding_horizon=3))
    agent.seed(g["seed"])
    assert [agent.act(0) for _ in range(3)] == g["plans"]
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    # HighwayLite through the env object, closed loop
    g = G["cases"]["hw1_closed_loop_h4_e40"]
    agent = MCTSDPWAgent(HighwayLiteEnv(seed=1), dict(g["config"]))
    agent.seed(g["seed"])
    assert agent.act(None) == g["plan"]
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    assert device_digest(agent.planner.last_tree, 0) == g["tree"]


def test_batched_evaluation_equals_per_episode_agents():
    from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPWAgent
    from rl_agents_b200.envs import HighwayLiteEnv
    from rl_agents_b200.evaluation import run_batched_episodes
    seeds = [0, 1, 2, 3]
    kw = {"closed_loop": True, "k_action": 2}
    out = run_batched_episodes("mcts_dpw", seeds, 60, 0.8, max_steps=6, planner_seed=50, **kw)
    for i, s in enumerate(seeds):
        env = HighwayLiteEnv(seed=s)
        agent = MCTSDPWAgent(env, dict(kw, budget=60, gamma=0.8))
        agent.seed(50 + i)
        total, steps = 0.0, 0
        for k in range(6):
            a = agent.act(None)
            assert a == out["actions"][i, k], (s, k)
            _, r, term, trunc, _ = env.step(a)
            total += float(np.float32(r))
            steps += 1
            if term or trunc:
                break
        assert steps == out["lengths"][i] and abs(total - out["returns"][i]) < 1e-9
