"""GPU tests of MDP-GapE (b2_mdp_gape_plan, csrc/mdp_gape.cu): the kernel against the reference's goldens
(tests/golden/golden_mdp_gape.json) and against the oracle restatement (oracle/mdp_gape.py), the error paths, the
agent surface and the batched evaluation branch.

Structure, plan, episodes run and the RNG stream position are exact; the bounds agree within 1e-9 (CUDA's fp64
log / exp against the host's, <= 1 ulp each, as for OLOP)."""
import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import mdp_gape as gape
from oracle import ref_loader
from tests.test_mdp_gape_oracle import G, M, case_env, completed_planner_config, rng_state

pytestmark = pytest.mark.gpu
TOL = 1e-9


def engine_for(env, cfg, n_trees):
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mdp_gape import MDPGapEEngine
    episodes, horizon = gape.mdp_gape_allocation(cfg, env.action_space.n)
    finite = isinstance(env, oenvs.FiniteMDPLite)
    return MDPGapEEngine(_lib.ENV_FINITE if finite else _lib.ENV_HIGHWAY, n_trees, env.action_space.n, episodes,
                         horizon, cfg["gamma"], cfg["upper_bound"], cfg["accuracy"], cfg["confidence"],
                         cfg["continuation_type"], cfg["max_next_states_count"], mdp=env.mdp if finite else None)


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


def assert_device_tree(d, t, n=None):
    """Device tree `d` (engine.tree_dict) against the first `n` nodes (all by default) of a tree dump `t` in the
    form of oracle.mdp_gape.tree_dict; fields a node does not carry are None there."""
    if n is None:
        n = len(t["parent"])
        assert len(d["parent"]) == n
    for f in ("parent", "action", "kind", "count", "done"):
        assert d[f][:n].astype(int).tolist() == [int(x) for x in t[f][:n]], f
    for f in gape.FLOAT_FIELDS:
        ref = np.array([np.nan if x is None else float(x) for x in t[f][:n]])
        has = ~np.isnan(ref)
        np.testing.assert_allclose(d[f][:n][has], ref[has], rtol=0, atol=TOL, err_msg=f)


def run_batch_against_oracle(envs_, cfg, seeds):
    """One launch over all trees; every tree equals its own oracle run."""
    eng = engine_for(envs_[0], cfg, len(envs_))
    eng.plan(roots(envs_), pcg64_of(seeds))
    plans, res, words = eng.finish()
    for i, (env, s) in enumerate(zip(envs_, seeds)):
        rng = ref_loader.legacy_np_random(s)[0]
        plan, t, episodes_run = gape.mdp_gape_plan(oenvs.LegacyStepEnv(env), cfg, rng)
        assert (plans[i], int(res[i, 1]), words_state(words[i])) == (plan, episodes_run, rng_state(rng)), i
        assert (int(res[i, 4]), int(res[i, 5])) == (t.best, t.challenger), i
        assert_device_tree(eng.tree_dict(i), gape.tree_dict(t))
    return eng, res, words


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_kernel_matches_reference_golden(key):
    """Each golden case: the kernel equals the oracle run on the whole tree, and the reference's golden on the plan,
    episodes run, UGapE's best / challenger, the RNG position and the first nodes of the tree."""
    g = G["cases"][key]
    eng, res, words = run_batch_against_oracle([case_env(key)], completed_planner_config(g["config"]), [g["seed"]])
    assert (eng.episodes, eng.horizon) == (g["episodes"], g["horizon"])
    assert [int(res[0, 3])] == g["plan"] and int(res[0, 1]) == g["episodes_run"]
    assert (int(res[0, 4]) - 1, int(res[0, 5]) - 1) == (g["best_index"], g["challenger_index"])    # root children 1..A
    assert words_state(words[0]) == g["rng_state"]
    assert_golden_tree(eng.tree_dict(0), g["tree"])


def assert_golden_tree(d, digest):
    """Device tree against a golden digest: node count and the first nodes in full."""
    assert len(d["parent"]) == digest["n_nodes"]
    assert_device_tree(d, digest, n=min(gape.HEAD, digest["n_nodes"]))


def test_batch_of_256_finite_trees_with_mixed_stopping_points_equals_the_oracle():
    cfg = completed_planner_config({"budget": 1000, "gamma": 0.7, "accuracy": 3.0, "max_next_states_count": 2})
    envs_ = [oenvs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"], state=i % 100) for i in range(256)]
    _, res, _ = run_batch_against_oracle(envs_, cfg, list(range(256)))
    ran = res[:, 1]
    cap = gape.mdp_gape_allocation(cfg, 5)[0] + 2
    assert len(set(ran.tolist())) > 5 and ran.min() < cap


def test_highway_batch_with_mixed_stopping_points_equals_the_oracle():
    cfg = completed_planner_config({"budget": 300, "gamma": 0.7, "accuracy": 2.0, "confidence": 1,
                                    "upper_bound": {"threshold": "1*np.log(time)"}})
    seeds = [0, 1, 2, 3, 4, 5]
    _, res, _ = run_batch_against_oracle([oenvs.HighwayLite(seed=s) for s in seeds], cfg, [10 + s for s in seeds])
    assert len(set(res[:, 1].tolist())) > 1 and res[:, 1].max() < gape.mdp_gape_allocation(cfg, 5)[0] + 2


def test_one_highway_decision_at_budget_5000_equals_the_oracle():
    cfg = completed_planner_config({"budget": 5000, "gamma": 0.7, "accuracy": 2.0, "confidence": 1,
                                    "upper_bound": {"threshold": "1*np.log(time)"}})
    _, res, _ = run_batch_against_oracle([oenvs.HighwayLite(seed=1)], cfg, [0])
    assert res[0, 1] < gape.mdp_gape_allocation(cfg, 5)[0] + 2       # the stopping rule fired


def test_error_paths():
    from rl_agents_b200 import _lib
    cfg = completed_planner_config({"budget": 100})
    # rewards outside [0, 1] (the trap MDP's raw rewards): ValueError, as the reference raises
    env = oenvs.FiniteMDPLite(M["trap_T"], M["trap_R"], M["trap_term"])
    eng = engine_for(env, cfg, 2)
    eng.plan(roots([env, env]), pcg64_of([0, 1]))
    with pytest.raises(ValueError, match="normalized in"):
        eng.finish()
    # a single available action at the root: UGapE has no challenger (max() of an empty list)
    one = oenvs.FiniteMDPLite(np.zeros((3, 1), int), np.full((3, 1), 0.5), None)
    eng = engine_for(one, cfg, 1)
    eng.plan(roots([one]), pcg64_of([0]))
    with pytest.raises(ValueError):
        eng.finish()
    # env kinds the kernel does not run on are refused by the C ABI and by the engine
    fin = oenvs.FiniteMDPLite(M["large1_T"], M["large1_R"], M["large1_term"])
    eng = engine_for(fin, cfg, 1)
    eng.cfg.env_kind = _lib.ENV_INTERSECTION
    with pytest.raises(_lib.B2Error, match="env_kind"):
        eng.plan(roots([fin]), pcg64_of([0]))
    from rl_agents_b200.engine.mdp_gape import MDPGapEEngine
    with pytest.raises(NotImplementedError):
        MDPGapEEngine(_lib.ENV_INTERSECTION, 1, 3, 10, 3, 0.8, cfg["upper_bound"], 1.0, 0.9)
    with pytest.raises(NotImplementedError):
        MDPGapEEngine(_lib.ENV_HIGHWAY, 1, 5, 10, 3, 0.8, {"type": "hoeffding"}, 1.0, 0.9)
    # an exception of the threshold expression surfaces as the reference's would (confidence 1: 1/(1-1))
    with pytest.raises(ZeroDivisionError):
        MDPGapEEngine(_lib.ENV_HIGHWAY, 1, 5, 10, 3, 0.8, dict(cfg["upper_bound"]), 1.0, 1)


def finite_env(state=0):
    from rl_agents_b200.envs import FiniteMDPEnv
    return FiniteMDPEnv(M["large1_T"], M["large1_R"], M["large1_term"], state=state)


def test_agent_surface_matches_reference():
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapEAgent
    for key in ("large1_b200_g0.8_default", "large1_b2000_g0.7_acc3_K3_zeros_stop"):
        g = G["cases"][key]
        agent = MDPGapEAgent(finite_env(), dict(g["config"], receding_horizon=3))
        agent.seed(g["seed"])
        assert agent.plan(0) == g["plan"]
        assert agent.planner.budget_used == g["budget_used"]
        assert rng_state(agent.planner.np_random) == g["rng_state"]
        assert_golden_tree(agent.planner.last_tree.tree_dict(0), g["tree"])
        # a replan at every call whatever receding_horizon is; remaining_horizon counts down as in the reference
        remaining = [agent.remaining_horizon]
        for _ in range(3):
            assert len(agent.plan(0)) == 1
            remaining.append(agent.remaining_horizon)
        assert remaining == [2, 1, 0, 2]
        agent.record(0, g["plan"][0], 0.5, 17, False, {})
        assert agent.planner.next_observation == 17
    # HighwayLite through the env object, with the shipped baseline.json (simplify preprocessor included)
    from rl_agents_b200.envs import HighwayLiteEnv
    baseline = G["configs"]["baseline"]["config"]
    g = G["cases"]["hw0_baseline"]
    agent = MDPGapEAgent(HighwayLiteEnv(seed=0), dict(baseline, __class__="<class '%s'>" % MDPGapEAgent.__name__))
    agent.seed(g["seed"])
    assert agent.act(None) == g["plan"][0] and agent.planner.budget_used == g["budget_used"]
    assert_golden_tree(agent.planner.last_tree.tree_dict(0), g["tree"])


def test_batched_evaluation_equals_per_episode_agents():
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapEAgent
    from rl_agents_b200.envs import HighwayLiteEnv
    from rl_agents_b200.evaluation import run_batched_episodes
    seeds = [0, 1, 2, 3]
    kw = {"accuracy": 0.1, "confidence": 1, "upper_bound": {"threshold": "1*np.log(time)"}}
    out = run_batched_episodes("mdp_gape", seeds, 100, 0.8, max_steps=6, planner_seed=50, **kw)
    for i, s in enumerate(seeds):
        env = HighwayLiteEnv(seed=s)
        agent = MDPGapEAgent(env, dict(kw, budget=100, gamma=0.8))
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
