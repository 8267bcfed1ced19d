"""GPU tests of MCTS and OLOP on IntersectionLite (b2_mcts_plan / b2_olop_plan with B2_ENV_INTERSECTION): the kernels
and the agents against the reference goldens (tests/golden/golden_intersection_planners.json), the Python oracle on
batches, and the C oracle at C3 size.  MCTS is bit-exact; OLOP's mu_ucb and value_upper are compared within the
tolerance of test_olop_finite_golden (the KL Newton solve uses log())."""
import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import intersection as oit
from oracle import planners, ref_loader
from tests.util import assert_tree_matches, canonical_tree, load_golden

pytestmark = pytest.mark.gpu
G = load_golden("golden_intersection_planners.json")
KL = {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)"}


def case_state(spec):
    st = oit.make_intersection_state(spec["seed"])
    if "speed_index" in spec:
        st.speed_index = int(spec["speed_index"])
    return st


def case_words(spec):
    return case_state(spec).pack()


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def golden_words(rs):
    """A golden rng_state -> the 6 PCG64 words the kernel advances."""
    m = (1 << 64) - 1
    s, inc = int(rs["state"]), int(rs["inc"])
    return [s >> 64, s & m, inc >> 64, inc & m, rs["has_uint32"], rs["uinteger"]]


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def scenes(words):
    import torch
    return torch.tensor(np.stack(words), dtype=torch.int32, device="cuda")


def policy(c, key):
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    return MCTSAgent.policy_factory(c.get(key, {"type": "random_available"}))


def mcts_engine(n, episodes, horizon, gamma, temperature, config=None):
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import MCTSEngine
    c = config or {}
    return MCTSEngine(_lib.ENV_INTERSECTION, n, 3, episodes, horizon, gamma, temperature,
                      rollout_policy=policy(c, "rollout_policy"), prior_policy=policy(c, "prior_policy"))


def olop_engine(n, episodes, horizon, gamma, ub, continuation):
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.olop import OLOPEngine
    return OLOPEngine(_lib.ENV_INTERSECTION, n, 3, episodes, horizon, gamma, ub, continuation)


def assert_mcts_tree_equals_oracle(d, t):
    assert d["parent"].tolist() == t.parent and d["action"].tolist() == t.action and d["count"].tolist() == t.count
    assert np.array_equal(d["value"], np.array(t.value)) and np.array_equal(d["prior"], np.array(t.prior))


# ------------------------------------------------------------------------------------------------- kernels ---
@pytest.mark.parametrize("key", sorted(G["mcts"]))
def test_mcts_kernel_equals_reference(key):
    from rl_agents_b200.engine.mcts import pcg64_words
    g = G["mcts"][key]
    eng = mcts_engine(1, g["episodes"], g["horizon"], g["config"]["gamma"], g["temperature"], g["config"])
    eng.plan(scenes([case_words(g["env"])]), pcg64_words(np_random(g["seed"])).reshape(1, -1))
    plans, res, words = eng.finish()
    assert plans[0] == g["plan"]
    assert_tree_matches(eng.tree_dict(0), g["tree"], ["value", "prior"])
    assert words[0].tolist() == golden_words(g["rng_state"])


@pytest.mark.parametrize("key", sorted(G["olop"]))
def test_olop_kernel_equals_reference(key):
    from rl_agents_b200.engine.mcts import pcg64_words
    g = G["olop"][key]
    c = g["config"]
    eng = olop_engine(1, g["episodes"], g["horizon"], c["gamma"], c["upper_bound"], c["continuation_type"])
    eng.plan(scenes([case_words(g["env"])]), pcg64_words(ref_loader.legacy_np_random(g["seed"])[0]).reshape(1, -1))
    if "error" in g:
        with pytest.raises(KeyError):
            eng.finish()
        return
    plans, res, words = eng.finish()
    assert plans[0] == g["plan"]
    assert_tree_matches(eng.tree_dict(0), g["tree"], ["cumulative_reward", "mu_ucb", "upper"], exact=False,
                        rtol=1e-9, atol=1e-12)
    assert words[0].tolist() == golden_words(g["rng_state"])


def test_mcts_odd_batch_with_an_idle_half_warp_equals_the_oracle():
    from rl_agents_b200.engine.mcts import pcg64_words
    specs = [{"seed": 20}, {"seed": 21, "speed_index": 2}, {"seed": 22, "speed_index": 0}]
    eng = mcts_engine(len(specs), 50, 6, 0.85, 10.0)
    eng.plan(scenes([case_words(s) for s in specs]), np.stack([pcg64_words(np_random(i + 1)) for i in range(3)]))
    plans, res, words = eng.finish()
    for i, s in enumerate(specs):
        rng = np_random(i + 1)
        plan, t = planners.mcts_plan(oit.IntersectionLite(case_state(s)), 50, 6, 0.85, 10.0, rng)
        assert plans[i] == plan
        assert_mcts_tree_equals_oracle(eng.tree_dict(i), t)
        assert words[i].tolist() == pcg64_words(rng).tolist()


def test_olop_odd_batch_with_an_idle_half_warp_equals_the_oracle():
    from rl_agents_b200.engine.mcts import pcg64_words
    specs = [{"seed": 30}, {"seed": 31, "speed_index": 2}, {"seed": 32, "speed_index": 0}]
    eng = olop_engine(len(specs), 14, 5, 0.8, KL, "uniform")
    eng.plan(scenes([case_words(s) for s in specs]),
             np.stack([pcg64_words(ref_loader.legacy_np_random(7 + i)[0]) for i in range(3)]))
    plans, res, words = eng.finish()
    for i, s in enumerate(specs):
        rng, _ = ref_loader.legacy_np_random(7 + i)
        plan, t = planners.olop_plan(oenvs.LegacyStepEnv(oit.IntersectionLite(case_state(s))), 0, 0.8, rng,
                                     upper_bound=KL, continuation_type="uniform", episodes=14, horizon=5)
        d = eng.tree_dict(i)
        assert plans[i] == plan
        assert d["parent"].tolist() == t.parent and d["count"].tolist() == t.count and d["action"].tolist() == t.action
        assert d["done"].tolist() == t.done
        assert np.array_equal(d["cumulative_reward"], np.array(t.cumulative_reward, dtype=np.float64))
        np.testing.assert_allclose(d["upper"], np.array(t.upper), rtol=1e-9, atol=1e-12)
        assert words[i].tolist() == pcg64_words(rng).tolist()


def test_mixed_batch_on_one_launch_equals_the_oracle():
    """Nine scenes in one launch: every root speed index (three or two actions available), a horizon past DURATION,
    each tree on its own stream, with the preference policies (whose table rows depend on each tree's available
    actions)."""
    from rl_agents_b200.engine.mcts import pcg64_words
    specs = [{"seed": s, "speed_index": s % 3} for s in range(40, 49)]
    config = {"prior_policy": {"type": "preference", "action": 0, "ratio": 3},
              "rollout_policy": {"type": "preference", "action": 2, "ratio": 2}}
    eng = mcts_engine(len(specs), 64, 15, 0.9, 4.0, config)
    eng.plan(scenes([case_words(s) for s in specs]), np.stack([pcg64_words(np_random(100 + i)) for i in range(9)]))
    plans, res, words = eng.finish()
    for i, s in enumerate(specs):
        rng = np_random(100 + i)
        plan, t = planners.mcts_plan(oit.IntersectionLite(case_state(s)), 64, 15, 0.9, 4.0, rng,
                                     prior_policy=config["prior_policy"], rollout_policy=config["rollout_policy"])
        assert plans[i] == plan, i
        assert_mcts_tree_equals_oracle(eng.tree_dict(i), t)
        assert words[i].tolist() == pcg64_words(rng).tolist()


def test_mcts_c3_size_equals_the_c_oracle():
    """C3's search size (4 096 episodes x horizon 20) on three scenes in one launch against the C statement: every
    node statistic, the env steps and the RNG words."""
    from oracle import c_mcts_intersection
    from rl_agents_b200.engine.mcts import pcg64_words
    specs = [{"seed": 3}, {"seed": 11, "speed_index": 2}, {"seed": 17}]
    eng = mcts_engine(len(specs), 4096, 20, 0.8, 10.0)
    rng_words = np.stack([pcg64_words(np_random(50 + i)) for i in range(3)])
    eng.plan(scenes([case_words(s) for s in specs]), rng_words)
    plans, res, words = eng.finish()
    for i, s in enumerate(specs):
        c, c_words = c_mcts_intersection.mcts_intersection_plan(case_words(s), 4096, 20, 0.8, 10.0, rng_words[i])
        d = eng.tree_dict(i)
        assert int(res[i, 0]) == len(c["parent"]) and int(res[i, 2]) == c["env_steps"]
        for f in ("parent", "action", "count", "first_child", "n_children"):
            assert np.array_equal(d[f], c[f]), f
        assert np.array_equal(d["value"], c["value"]) and np.array_equal(d["prior"], c["prior"])
        assert words[i].tolist() == c_words.tolist()


# -------------------------------------------------------------------------------------------------- agents ---
def il_env(spec):
    from rl_agents_b200.envs import IntersectionLiteEnv
    return IntersectionLiteEnv(words=case_words(spec))


@pytest.mark.parametrize("key", sorted(G["mcts"]))
def test_mcts_agent_equals_reference(key):
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    g = G["mcts"][key]
    agent = MCTSAgent(il_env(g["env"]), dict(g["config"]))
    agent.seed(g["seed"])
    assert agent.plan(None) == g["plan"]
    assert_tree_matches(agent.planner.last_tree.tree_dict(0), g["tree"], ["value", "prior"])
    assert rng_state(agent.planner.np_random) == g["rng_state"]


@pytest.mark.parametrize("key", sorted(G["olop"]))
def test_olop_agent_equals_reference(key):
    from rl_agents_b200.agents.tree_search.olop import OLOPAgent
    g = G["olop"][key]
    agent = OLOPAgent(il_env(g["env"]), dict(g["config"]))
    agent.seed(g["seed"])
    assert (agent.planner.config["episodes"], agent.planner.config["horizon"]) == (g["episodes"], g["horizon"])
    if "error" in g:
        with pytest.raises(KeyError):
            agent.plan(None)
        return
    assert agent.plan(None) == g["plan"]
    assert_tree_matches(agent.planner.last_tree.tree_dict(0), g["tree"], ["cumulative_reward", "mu_ucb", "upper"],
                        exact=False, rtol=1e-9, atol=1e-12)
    assert rng_state(agent.planner.np_random) == g["rng_state"]


def test_mcts_agent_closed_loop_equals_reference():
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    g = G["closed_loop"]
    agent = MCTSAgent(il_env(g["env"]), dict(g["config"]))
    agent.seed(g["seed"])
    assert agent.plan(None) == g["plan_actions"]
    d = agent.planner.last_tree.tree_dict(0)
    fc, n = int(d["first_child"][0]), int(d["n_children"][0])
    assert [[int(d["action"][c]), int(d["count"][c]), float(d["value"][c])] for c in range(fc, fc + n)] == g["root"]
    assert int(d["count"][0]) == g["root_count"] and float(d["value"][0]) == g["root_value"]
    assert rng_state(agent.planner.np_random) == g["rng_state"]


def test_mcts_agent_subtree_strategy_equals_reference():
    """Three decisions, the sub-tree under the executed action kept (host re-rooting, kernel resume), the env
    stepped by the CUDA transition between them."""
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    g = G["subtree"]
    env = il_env(g["env"])
    agent = MCTSAgent(env, dict(g["config"]))
    agent.seed(g["seed"])
    for k in range(3):
        assert env.words.tolist() == g["words"][k], k
        plan = agent.plan(None)
        assert plan == g["plans"][k], k
        d = agent.planner.last_tree.tree_dict(0)
        got = canonical_tree(d["first_child"], d["n_children"], [d["count"].tolist(), d["value"].tolist(),
                                                                 d["prior"].tolist()])
        assert got == g["trees"][k], k
        env.step(plan[0])
    assert rng_state(agent.planner.np_random) == g["rng_state"]


def test_agents_receding_horizon_equal_reference():
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    from rl_agents_b200.agents.tree_search.olop import OLOPAgent
    for key, g in G["agents"].items():
        cls = MCTSAgent if key.startswith("mcts") else OLOPAgent
        agent = cls(il_env(g["env"]), dict(g["config"]))
        agent.seed(g["seed"])
        assert [agent.plan(None) for _ in range(len(g["decisions"]))] == g["decisions"], key
        assert rng_state(agent.planner.np_random) == g["rng_state"], key


def test_mcts_agent_root_parallel():
    """"root_parallel": R trees of episodes/R episodes from the same root: reproducible for a planner seed, every
    episode accounted for in the merged root statistics, and each replica equal to the oracle on its spawned stream."""
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    cfg = {"episodes": 256, "horizon": 8, "gamma": 0.8, "root_parallel": 8}
    plans = []
    for _ in range(2):
        agent = MCTSAgent(il_env({"seed": 2}), dict(cfg))
        agent.seed(7)
        plans.append(agent.plan(None))
        counts = agent.planner.root_statistics["counts"]
        assert counts.sum() == 8 * (256 // 8 - 1)          # the expanding episode of each tree selects no child
        assert counts[plans[-1][0]] == counts.max()
    assert plans[0] == plans[1]
    eng = agent.planner.last_tree
    for r, gen in enumerate(np_random(7).spawn(8)):
        _, t = planners.mcts_plan(oit.IntersectionLite(case_state({"seed": 2})), 32, 8, 0.8, 10.0, gen)
        assert_mcts_tree_equals_oracle(eng.tree_dict(r), t)


@pytest.mark.parametrize("planner", ["mcts", "olop"])
def test_batched_episodes_equal_per_scene_agents(planner):
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    from rl_agents_b200.agents.tree_search.olop import OLOPAgent
    from rl_agents_b200.envs import IntersectionLiteEnv
    from rl_agents_b200.evaluation import run_batched_episodes
    seeds = [0, 1, 2, 3, 4]
    out = run_batched_episodes(planner, seeds, 150, 0.8, max_steps=14, planner_seed=100, env="intersection")
    for i, s in enumerate(seeds):
        env = IntersectionLiteEnv(seed=s)
        if planner == "mcts":
            agent = MCTSAgent(env, {"budget": 150, "gamma": 0.8})
        else:
            agent = OLOPAgent(env, {"budget": 150, "gamma": 0.8, "upper_bound": KL, "continuation_type": "uniform"})
        agent.seed(100 + i)
        total, steps, crashed = 0.0, 0, False
        for k in range(14):
            a = agent.act(None)
            assert a == out["actions"][i, k], (s, k)
            _, r, term, trunc, _ = env.step(a)
            total += r
            steps += 1
            crashed = bool(env.words[48] & 2)
            if term or trunc:
                break
        assert steps == out["lengths"][i] and abs(total - out["returns"][i]) < 1e-9
        assert crashed == out["crashed"][i]


# ------------------------------------------------------------------------------------------------- refusals ---
def test_the_other_planners_still_refuse_intersection_lite():
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.brue import BRUEAgent
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPWAgent
    from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapEAgent
    from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOSAgent
    from rl_agents_b200.agents.tree_search.sparse_sampling import SparseSamplingAgent
    from rl_agents_b200.engine.brue import BRUEEngine
    from rl_agents_b200.evaluation import run_batched_episodes
    for cls, cfg in ((BRUEAgent, {}), (MDPGapEAgent, {}), (SparseSamplingAgent, {"horizon": 2, "C": 2}),
                     (MCTSDPWAgent, {}), (PlaTyPOOSAgent, {"budget": 10000})):
        with pytest.raises(NotImplementedError):
            cls(il_env({"seed": 0}), cfg)
    with pytest.raises(NotImplementedError):
        BRUEEngine(_lib.ENV_INTERSECTION, 1, 3, 50, 4, 0.8)
    # wavefront MCTS is HighwayLite and finite MDPs only
    agent = MCTSAgent(il_env({"seed": 0}), {"episodes": 64, "horizon": 5, "wavefront": 16})
    with pytest.raises(_lib.B2Error, match="env_kind 2"):
        agent.plan(None)
    for planner in ("opd", "brue", "mdp_gape", "mcts_dpw", "platypoos", "vi"):
        with pytest.raises(NotImplementedError):
            run_batched_episodes(planner, [0], 100, 0.8, max_steps=1, env="intersection")


def test_c_abi_refuses_other_action_counts_for_intersection_lite():
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import MCTSEngine, pcg64_words
    from rl_agents_b200.engine.olop import OLOPEngine
    root = scenes([case_words({"seed": 0})])
    words = pcg64_words(np_random(0)).reshape(1, -1)
    for n_actions in (2, 5):
        with pytest.raises(_lib.B2Error, match="IntersectionLite has 3 actions"):
            MCTSEngine(_lib.ENV_INTERSECTION, 1, n_actions, 10, 4, 0.8, 10.0).plan(root, words)
        with pytest.raises(_lib.B2Error, match="IntersectionLite has 3 actions"):
            OLOPEngine(_lib.ENV_INTERSECTION, 1, n_actions, 10, 4, 0.8, KL).plan(root, words)
