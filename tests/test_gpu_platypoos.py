"""GPU tests of PlaTyPOOS (b2_platypoos_plan, csrc/platypoos.cu): the kernel against the reference's goldens
(tests/golden/golden_platypoos.json) and against the oracle restatement (oracle/platypoos.py), the error paths, the agent
surface and the batched evaluation branch.

Every comparison is exact: structure, counts, flags, the float64 bytes of every node's cumulative reward and value, the
openings, the candidates, the plan and the RNG stream position."""
import json

import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import platypoos as opl
from oracle import ref_loader
from tests.test_platypoos_oracle import G, M, assert_tree_equals_golden, case_env, completed_planner_config, rng_state

pytestmark = pytest.mark.gpu


def engine_for(env, cfg, n_trees, **kw):
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.platypoos import PlaTyPOOSEngine
    finite = isinstance(env, oenvs.FiniteMDPLite)
    return PlaTyPOOSEngine(_lib.ENV_FINITE if finite else _lib.ENV_HIGHWAY, n_trees, env.action_space.n,
                           cfg["horizon"], cfg["gamma"], mdp=env.mdp if finite else None, **kw)


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


def assert_tree_equals_oracle(d, t):
    o = opl.tree_dict(t)
    for f in opl.INT_FIELDS:
        assert [int(x) for x in d[f]] == o[f], f
    for f in opl.FLOAT_FIELDS:
        assert np.asarray(d[f], dtype=np.float64).tobytes() == np.array(o[f], dtype=np.float64).tobytes(), f


def run_batch_against_oracle(envs_, cfg, seeds):
    """One launch over all trees; every tree equals its own oracle run, float bytes included."""
    eng = engine_for(envs_[0], cfg, len(envs_))
    eng.plan(roots(envs_), pcg64_of(seeds))
    plans, res, words = eng.finish()
    for i, (env, s) in enumerate(zip(envs_, seeds)):
        rng = ref_loader.legacy_np_random(s)[0]
        plan, t, openings, candidates = opl.platypoos_plan(env, cfg, rng)
        assert plans[i] == plan, i
        assert (int(res[i, 0]), int(res[i, 1]), int(res[i, 2]), int(res[i, 3])) == (len(t), openings, len(plan), 0), i
        assert words_state(words[i]) == rng_state(rng), i
        d = eng.tree_dict(i)
        assert d["candidates"] == [tuple(c) for c in candidates], i
        assert_tree_equals_oracle(d, t)
    return res


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_kernel_matches_reference_golden(key):
    g = G["cases"][key]
    env = case_env(g["env"])
    cfg = completed_planner_config(g["config"], env)
    assert cfg["horizon"] == g["horizon"]
    eng = engine_for(env, cfg, 1)
    eng.plan(roots([env]), pcg64_of([g["seed"]]))
    plans, res, words = eng.finish()
    assert plans[0] == g["plan"]
    assert (int(res[0, 1]), int(res[0, 2]), int(res[0, 3]), int(res[0, 4])) == (g["openings"], len(g["plan"]), 0, -1)
    assert words_state(words[0]) == g["rng_state"]
    d = eng.tree_dict(0)
    assert [list(c) for c in d["candidates"]] == g["candidates"]
    assert_tree_equals_golden(d, g)


@pytest.mark.parametrize("budget,gamma", [(2500, 0.9), (20000, 0.8), (200000, 0.9)])
def test_batch_of_256_mixed_finite_trees_equals_the_oracle(budget, gamma):
    """256 trees in one launch on one "sparse" table holding stochastic, sparse and deterministic rows side by side
    (tests/test_gpu_mcts_dpw.py::mixed_finite_mdp), rooted in each part; at budget 200 000 (h_max 115) the stochastic
    and sparse children are seeded thousands of draws into the stream."""
    from tests.test_gpu_mcts_dpw import mixed_finite_mdp
    make, off = mixed_finite_mdp()
    starts = [off[0], off[0] + 7, off[1], off[1] + 5, off[2], off[2] + 37, off[3], off[3] + 2]
    envs_ = [make(starts[i % len(starts)]) for i in range(256)]
    cfg = completed_planner_config({"budget": budget, "gamma": gamma}, envs_[0])
    res = run_batch_against_oracle(envs_, cfg, list(range(256)))
    assert len(set(res[:, 0].tolist())) > 3


def test_batch_of_garnet_trees_at_budget_200000_equals_the_oracle():
    T, R = oenvs.garnet(1000, 4, 1, seed=0, deterministic=True)
    envs_ = [oenvs.FiniteMDPLite(T, R, state=s) for s in range(0, 1000, 40)]
    envs_ += [oenvs.FiniteMDPLite(T, R, mode="deterministic", state=s) for s in (1, 2)]
    cfg = completed_planner_config({"budget": 200000, "gamma": 0.9}, envs_[0])
    res = run_batch_against_oracle(envs_, cfg, list(range(len(envs_))))
    assert cfg["horizon"] == 90 and res[:, 0].max() > 500


def test_finite_mdp_with_40_actions_equals_the_oracle():
    """39 expanded actions per node: cross-validation updates more children than one warp has lanes."""
    rng = np.random.default_rng(3)
    P = rng.uniform(size=(30, 40, 30))
    P /= P.sum(axis=-1, keepdims=True)
    R = rng.uniform(size=(30, 40))
    envs_ = [oenvs.FiniteMDPLite(P, R, mode="stochastic", state=s) for s in (0, 11, 29)]
    cfg = completed_planner_config({"budget": 200000, "gamma": 0.9}, envs_[0])
    res = run_batch_against_oracle(envs_, cfg, [5, 6, 7])
    assert (res[:, 0] > 1000).all()


def test_horizon_above_127_equals_the_oracle():
    """An explicit horizon of 150: trees 149 layers deep at most, plans as long as their best candidate is deep."""
    envs_ = [case_env({"name": "stoch8", "state": s}) for s in (0, 3)]
    cfg = completed_planner_config({"horizon": 150, "gamma": 0.95}, envs_[0])
    res = run_batch_against_oracle(envs_, cfg, [8, 9])
    assert (res[:, 0] > 1000).all()


def test_batch_of_16_highway_scenes_at_budget_10000_equals_the_oracle():
    envs_ = [oenvs.HighwayLite(seed=s) for s in range(16)]
    cfg = completed_planner_config({"budget": 10000, "gamma": 0.9}, envs_[0])
    res = run_batch_against_oracle(envs_, cfg, list(range(100, 116)))
    assert (res[:, 2] >= 2).any()


def test_error_paths():
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOSAgent
    from rl_agents_b200.engine.platypoos import PlaTyPOOSEngine
    from rl_agents_b200.envs import FiniteMDPEnv, HighwayLiteEnv
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv
    e = G["errors"]
    # horizon < 2: the default budget on HighwayLite gives h_max 0
    with pytest.raises(ValueError, match="max\\(\\) iterable argument is empty"):
        PlaTyPOOSAgent(HighwayLiteEnv(seed=0), {}).act(None)
    with pytest.raises(ValueError, match="horizon >= 2"):
        PlaTyPOOSAgent(HighwayLiteEnv(seed=0), {"horizon": 1}).act(None)
    # one finite action: the root gets no child
    with pytest.raises(ValueError, match="max\\(\\) iterable argument is empty"):
        PlaTyPOOSAgent(FiniteMDPEnv(M["trap_T"][:, :1], M["trap_R"][:, :1]), {"budget": 10000}).act(None)
    # a reached row that Generator.choice rejects raises numpy's own ValueError, only when reached
    bad = case_env({"name": "stoch8_bad_row"})
    cfg = completed_planner_config({"budget": 10000, "gamma": 0.9}, bad)
    eng = engine_for(bad, cfg, 2)
    eng.plan(roots([bad, case_env({"name": "stoch8_bad_row", "state": 7})]), pcg64_of([0, 1]))
    with pytest.raises(ValueError, match=e["bad_row"]["message"]):
        eng.finish()
    assert eng.result[1, 3].item() == 0            # the terminal root never steps the bad row
    # a root whose tree never reaches the bad row plans normally
    unreached = case_env({"name": "stoch8_bad_row", "state": 7})
    run_batch_against_oracle([unreached], cfg, [3])
    # an arena smaller than the tree: error 1, a B2Error
    env = case_env({"name": "large1"})
    cfg = completed_planner_config({"budget": 10000, "gamma": 0.9}, env)
    for kw in ({"node_capacity": 20}, {"layer_capacity": 3}):
        small = engine_for(env, cfg, 1, **kw)
        small.plan(roots([env]), pcg64_of([0]))
        with pytest.raises(_lib.B2Error, match="exhausted"):
            small.finish()
        assert small.result[0, 3].item() == 1
    with pytest.raises(ValueError):
        PlaTyPOOSEngine(_lib.ENV_FINITE, 1, 4, 6, 0.9, mdp=env.mdp, node_capacity=2 ** 31)
    # "subtree" and IntersectionLite
    with pytest.raises(NotImplementedError):
        PlaTyPOOSAgent(HighwayLiteEnv(seed=0), {"budget": 10000, "step_strategy": "subtree"})
    with pytest.raises(NotImplementedError):
        PlaTyPOOSAgent(IntersectionLiteEnv(seed=0), {"budget": 10000})
    with pytest.raises(NotImplementedError):
        PlaTyPOOSEngine(_lib.ENV_INTERSECTION, 1, 3, 6, 0.9)
    assert torch.cuda.is_available()


def finite_env(name, state=0):
    from rl_agents_b200.envs import FiniteMDPEnv
    return case_env({"name": name, "state": state}, finite_cls=FiniteMDPEnv)


def test_agent_surface_matches_reference():
    """Plans, openings and RNG position equal the reference planner's on FiniteMDPEnv in every mode and on HighwayLite;
    the receding horizon serves multi-action plans as the reference agent does; seed / reset as the reference's."""
    from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOSAgent
    from rl_agents_b200.envs import HighwayLiteEnv
    for key in ("stoch8_stochastic_budget10000", "garnet12_sparse_budget10000", "large1_deterministic_budget10000",
                "hw3_budget10000_gamma0.9", "stoch8_explicit_horizon"):
        g = G["cases"][key]
        spec = g["env"]
        env = HighwayLiteEnv(seed=spec["seed"]) if spec["name"] == "highway" else finite_env(spec["name"])
        agent = PlaTyPOOSAgent(env, dict(g["config"]))
        assert agent.seed(g["seed"]) == [g["seed"]]
        assert agent.plan(None) == g["plan"], key
        assert agent.planner.openings == g["openings"]
        assert [list(c) for c in agent.planner.candidates] == g["candidates"]
        assert rng_state(agent.planner.np_random) == g["rng_state"], key
    for key, a in G["agents"].items():
        spec = a["env"]
        env = HighwayLiteEnv(seed=spec["seed"]) if spec["name"] == "highway" else finite_env(spec["name"])
        agent = PlaTyPOOSAgent(env, dict(a["config"]))
        agent.seed(a["seed"])
        assert [agent.plan(None) for _ in a["decisions"]] == a["decisions"], key
        assert rng_state(agent.planner.np_random) == a["rng_state"], key
    # the shipped baseline.json, `__class__` switched, with its "simplify" preprocessor: the golden's plan
    c = G["configs"]["baseline_highway"]
    g = G["cases"]["hw0_baseline"]
    agent = PlaTyPOOSAgent(HighwayLiteEnv(seed=0), dict(
        json.loads(json.dumps(c["config"])), __class__="<class 'rl_agents_b200.agents.tree_search.platypoos."
                                                       "PlaTyPOOSAgent'>"))
    agent.seed(g["seed"])
    assert agent.act(None) == g["plan"][0]
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    # reset() keeps the stream; seed() restarts it
    g = G["cases"]["stoch8_stochastic_budget10000"]
    agent = PlaTyPOOSAgent(finite_env("stoch8"), dict(g["config"]))
    agent.seed(g["seed"])
    first = agent.plan(None)
    agent.reset()
    agent.plan(None)
    agent.seed(g["seed"])
    agent.reset()
    assert agent.plan(None) == first == g["plan"]


def test_batched_evaluation_equals_per_episode_agents():
    from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOSAgent
    from rl_agents_b200.envs import HighwayLiteEnv
    from rl_agents_b200.evaluation import run_batched_episodes
    seeds = [0, 1, 2, 3]
    out = run_batched_episodes("platypoos", seeds, 10000, 0.8, max_steps=5, planner_seed=50)
    for i, s in enumerate(seeds):
        env = HighwayLiteEnv(seed=s)
        agent = PlaTyPOOSAgent(env, {"budget": 10000, "gamma": 0.8})
        agent.seed(50 + i)
        total, steps = 0.0, 0
        for k in range(5):
            a = agent.act(None)
            assert a == out["actions"][i, k], (s, k)
            _, r, term, trunc, _ = env.step(a)
            total += float(np.float32(r))
            steps += 1
            if term or trunc:
                break
        assert steps == out["lengths"][i] and abs(total - out["returns"][i]) < 1e-9
