"""GPU tests of BRUE (b2_brue_plan, csrc/brue.cu): the kernel against the reference's goldens
(tests/golden/golden_brue.json) and against the oracle restatement (oracle/brue.py), the error paths, the agent surface
and the batched evaluation branch.

Every comparison is exact: structure, plan, rollouts, env steps, the RNG stream position, and the float64 bytes of
every node's value (the digests hash them)."""
import numpy as np
import pytest

from oracle import brue
from oracle import envs as oenvs
from oracle import ref_loader
from tests.test_brue_oracle import G, M, case_env, completed_planner_config, rng_state

pytestmark = pytest.mark.gpu


def engine_for(env, cfg, n_trees):
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.brue import BRUEEngine
    finite = isinstance(env, oenvs.FiniteMDPLite)
    return BRUEEngine(_lib.ENV_FINITE if finite else _lib.ENV_HIGHWAY, n_trees, env.action_space.n, cfg["budget"],
                      brue.brue_horizon(cfg, env.action_space.n), cfg["gamma"], mdp=env.mdp if finite else None)


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
    return brue.tree_digest({f: d[f].tolist() for f in brue.INT_FIELDS + brue.FLOAT_FIELDS})


def run_batch_against_oracle(envs_, cfg, seeds):
    """One launch over all trees; every tree equals its own oracle run, value bytes included."""
    eng = engine_for(envs_[0], cfg, len(envs_))
    eng.plan(roots(envs_), pcg64_of(seeds))
    plans, res, words = eng.finish()
    for i, (env, s) in enumerate(zip(envs_, seeds)):
        rng = ref_loader.legacy_np_random(s)[0]
        plan, t, rollouts = brue.brue_plan(oenvs.LegacyStepEnv(env), cfg, rng)
        assert (plans[i], int(res[i, 1]), int(res[i, 2])) == (plan, rollouts, cfg["budget"] - t.budget_left), i
        assert words_state(words[i]) == rng_state(rng), i
        assert device_digest(eng, i) == brue.tree_digest(brue.tree_dict(t)), i
    return res


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_kernel_matches_reference_golden(key):
    """Each golden case, consecutive decisions included: plan, rollouts, env steps, RNG position and the tree digest
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
        plans.append(p[0])
    assert eng.horizon == g["horizon"]
    assert plans == g.get("plans", [g["plan"]])
    assert (int(res[0, 1]), int(res[0, 2])) == (g["rollouts"], cfg["budget"] - g["budget_left"])
    assert int(res[0, 0]) == g["tree"]["n_nodes"]
    assert words_state(words[0]) == g["rng_state"]
    assert device_digest(eng, 0) == g["tree"]


def mixed_finite_mdp():
    """large1, large2 and trap side by side in one table (trap's two actions repeated over five), so that one launch
    holds trees on all three; -> (env factory by root state, state offsets)."""
    T = [M["large1_T"], M["large2_T"] + 100, M["trap_T"][:, [0, 1, 0, 1, 0]] + 200]
    R = [M["large1_R"], M["large2_R"], M["trap_R"][:, [0, 1, 0, 1, 0]]]
    term = np.concatenate([M["large1_term"], M["large2_term"], M["trap_term"]])
    T, R = np.concatenate(T), np.concatenate(R)
    return lambda s: oenvs.FiniteMDPLite(T, R, term, state=s)


def test_batch_of_256_finite_trees_with_mixed_rollout_counts_equals_the_oracle():
    make = mixed_finite_mdp()
    trap_terminal = 200 + int(np.nonzero(M["trap_term"])[0][0])
    starts = [0, 37, 100, 163, 200, 202, trap_terminal]
    envs_ = [make(starts[i % len(starts)]) for i in range(256)]
    cfg = completed_planner_config({"budget": 150, "gamma": 0.8})
    res = run_batch_against_oracle(envs_, cfg, list(range(256)))
    assert len(set(res[:, 1].tolist())) > 5 and (res[:, 1] == 150).any()      # terminal roots: one-step rollouts


def test_highway_batch_of_64_scenes_equals_the_oracle():
    cfg = completed_planner_config({"budget": 60, "gamma": 0.8, "horizon": 4})
    run_batch_against_oracle([oenvs.HighwayLite(seed=s) for s in range(64)], cfg, [100 + s for s in range(64)])


def test_one_highway_decision_at_budget_5000_equals_the_oracle():
    cfg = completed_planner_config({"budget": 5000, "gamma": 0.8})
    res = run_batch_against_oracle([oenvs.HighwayLite(seed=1)], cfg, [0])
    assert res[0, 2] >= 5000 and res[0, 0] > 5000


def test_error_paths():
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.brue import BRUEAgent
    from rl_agents_b200.engine.brue import BRUEEngine
    from rl_agents_b200.envs import FiniteMDPEnv, IntersectionLiteEnv
    fin = FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"])
    with pytest.raises(NotImplementedError):
        BRUEAgent(fin, {"step_strategy": "subtree"})
    with pytest.raises(NotImplementedError):
        BRUEAgent(IntersectionLiteEnv(seed=0), {})
    with pytest.raises(NotImplementedError):
        BRUEEngine(_lib.ENV_INTERSECTION, 1, 3, 10, 3, 0.8)
    # a stochastic finite MDP: the tree search needs deterministic transitions
    P = np.full((4, 2, 4), 0.25)
    stochastic = FiniteMDPEnv(P, np.zeros((4, 2)), None, mode="stochastic")
    with pytest.raises(ValueError):
        BRUEAgent(stochastic, {}).plan(0)
    # budget < 1 (the reference's empty-root ValueError) and horizon < 1 (its endless budget loop)
    with pytest.raises(ValueError, match="zero-size array"):
        BRUEAgent(fin, {"budget": 0}).plan(0)
    with pytest.raises(ValueError):
        BRUEAgent(fin, {"horizon": 0}).plan(0)
    for budget, horizon in ((0, 3), (10, 0)):
        with pytest.raises(ValueError):
            BRUEEngine(_lib.ENV_HIGHWAY, 1, 5, budget, horizon, 0.8)
    # the C ABI refuses what the engine refuses
    env = oenvs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"])
    eng = engine_for(env, completed_planner_config({"budget": 20}), 1)
    eng.cfg.env_kind = _lib.ENV_INTERSECTION
    with pytest.raises(_lib.B2Error, match="env_kind"):
        eng.plan(roots([env]), pcg64_of([0]))
    eng.cfg.env_kind, eng.cfg.budget = _lib.ENV_FINITE, 0
    with pytest.raises(_lib.B2Error, match="budget"):
        eng.plan(roots([env]), pcg64_of([0]))
    eng.cfg.budget, eng.cfg.node_capacity = 20, 10
    with pytest.raises(_lib.B2Error, match="node_capacity"):
        eng.plan(roots([env]), pcg64_of([0]))


def test_agent_surface_matches_reference():
    """Built from brue.json with `__class__` switched, as agent_factory builds it, on a finite MDP and on HighwayLite:
    one-action plans equal to the reference's, seed / reset as the reference's."""
    from rl_agents_b200.agents.tree_search.brue import BRUEAgent
    from rl_agents_b200.envs import FiniteMDPEnv, HighwayLiteEnv
    shipped = dict(G["configs"]["brue_json"]["config"], __class__="<class '%s.%s'>" % (BRUEAgent.__module__,
                                                                                          BRUEAgent.__name__))
    g = G["cases"]["large1_brue_json"]
    agent = BRUEAgent(FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"]), dict(shipped))
    assert agent.seed(g["seed"]) == [g["seed"]]
    assert agent.plan(0) == g["plan"] and agent.planner.available_budget == g["budget_left"]
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    assert device_digest(agent.planner.last_tree, 0) == g["tree"]
    # reset() keeps the RNG stream; seed() restarts it
    agent.reset()
    second = agent.plan(0)
    agent.seed(g["seed"])
    assert agent.plan(0) == g["plan"] and len(second) == 1
    # receding_horizon 3 still replans at every call: three decisions equal the reference's three
    g = G["cases"]["large1_receding3_three_decisions"]
    agent = BRUEAgent(FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"]), dict(g["config"]))
    agent.seed(g["seed"])
    assert [agent.plan(0) for _ in range(3)] == g["plans"]
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    assert device_digest(agent.planner.last_tree, 0) == g["tree"]
    # HighwayLite through the env object
    g = G["cases"]["hw0_brue_json"]
    agent = BRUEAgent(HighwayLiteEnv(seed=0), dict(shipped))
    agent.seed(g["seed"])
    assert agent.act(None) == g["plan"][0]
    assert device_digest(agent.planner.last_tree, 0) == g["tree"]


def test_batched_evaluation_equals_per_episode_agents():
    from rl_agents_b200.agents.tree_search.brue import BRUEAgent
    from rl_agents_b200.envs import HighwayLiteEnv
    from rl_agents_b200.evaluation import run_batched_episodes
    seeds = [0, 1, 2, 3]
    kw = {"horizon": 4}
    out = run_batched_episodes("brue", seeds, 60, 0.8, max_steps=6, planner_seed=50, **kw)
    for i, s in enumerate(seeds):
        env = HighwayLiteEnv(seed=s)
        agent = BRUEAgent(env, dict(kw, budget=60, gamma=0.8))
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
