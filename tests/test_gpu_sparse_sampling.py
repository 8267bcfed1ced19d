"""GPU tests of sparse sampling (b2_sparse_sampling_plan, csrc/sparse_sampling.cu): the kernel against the reference's
goldens (tests/golden/golden_sparse_sampling.json) and against the oracle restatement (oracle/sparse_sampling.py), the
error paths, the agent surface and the batched evaluation branch.

Every comparison is exact: structure, plan, node and sample counts, the RNG stream position, the root's chance values
and the float64 bytes of every node's value (the digests hash them)."""
import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import ref_loader
from oracle import sparse_sampling as ss
from tests.test_sparse_sampling_oracle import G, M, case_env, completed_planner_config, golden_root_q, rng_state

pytestmark = pytest.mark.gpu


def engine_for(env, cfg, n_trees, record=True, **kw):
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.sparse_sampling import SparseSamplingEngine
    finite = isinstance(env, oenvs.FiniteMDPLite)
    return SparseSamplingEngine(_lib.ENV_FINITE if finite else _lib.ENV_HIGHWAY, n_trees, env.action_space.n,
                                cfg["horizon"], cfg["C"], cfg["gamma"], mdp=env.mdp if finite else None,
                                record_tree=record, **kw)


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
    return ss.tree_digest({f: d[f].tolist() for f in ss.INT_FIELDS + ss.FLOAT_FIELDS})


def run_batch_against_oracle(envs_, cfg, seeds):
    """One launch over all trees; every tree equals its own oracle run, value bytes included."""
    eng = engine_for(envs_[0], cfg, len(envs_))
    eng.plan(roots(envs_), pcg64_of(seeds))
    plans, res, words = eng.finish()
    root_q = eng.root_q.cpu().numpy()
    for i, (env, s) in enumerate(zip(envs_, seeds)):
        rng = ref_loader.legacy_np_random(s)[0]
        plan, t, q = ss.sparse_sampling_plan(oenvs.LegacyStepEnv(env), cfg, rng)
        assert plans[i] == plan, i
        assert (int(res[i, 0]), int(res[i, 1]), int(res[i, 2])) == (len(t), sum(t.kind), cfg["C"] * sum(t.kind)), i
        assert words_state(words[i]) == rng_state(rng), i
        assert np.array_equal(root_q[i], q, equal_nan=True), i
        assert device_digest(eng, i) == ss.tree_digest(ss.tree_dict(t)), i
    return res


@pytest.mark.parametrize("key", sorted(G["cases"]))
def test_kernel_matches_reference_golden(key):
    """Each golden case, consecutive decisions included: plan, node and sample counts, RNG position, the root's chance
    values and the tree digest (integer fields and the float64 bytes of `value`) equal the reference's."""
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
    assert plans == g.get("plans", [g["plan"]])
    assert (int(res[0, 0]), int(res[0, 1]), int(res[0, 2])) == (g["tree"]["n_nodes"], g["chance_nodes"], g["samples"])
    assert (int(res[0, 3]), int(res[0, 4]), int(res[0, 5])) == (g["plan"][0], 0, -1)
    assert words_state(words[0]) == g["rng_state"]
    assert np.array_equal(eng.root_q[0].cpu().numpy(), golden_root_q(g), equal_nan=True)
    assert device_digest(eng, 0) == g["tree"]


def mixed_finite_mdp():
    """stoch8 ("stochastic"), garnet12 ("sparse"), large1's first three actions and loop (deterministic) side by side
    in one "sparse" table of width 8: next = arange for the stochastic rows, zero-probability padding for the garnet,
    probability one on the successor for the deterministic rows.  -> (env factory by root state, state offsets)."""
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
    for name in ("large1", "loop"):
        T = M[name + "_T"][:, :3]
        p = np.zeros(T.shape + (8,))
        p[..., 0] = 1.0
        parts_p.append(p)
        parts_n.append(np.repeat(T[..., None], 8, axis=-1) + base)
        parts_r.append(M[name + "_R"][:, :3])
        parts_t.append(M[name + "_term"])
        offsets.append(base)
        base += T.shape[0]
    P, N, R, term = (np.concatenate(x) for x in (parts_p, parts_n, parts_r, parts_t))
    return (lambda s: oenvs.FiniteMDPLite(P, R, term, mode="sparse", nxt=N, state=s)), offsets


def test_batch_of_256_mixed_finite_trees_equals_the_oracle():
    make, off = mixed_finite_mdp()
    starts = [off[0], off[0] + 7, off[1], off[1] + 5, off[2], off[2] + 37, off[3], off[3] + 2]
    envs_ = [make(starts[i % len(starts)]) for i in range(256)]
    cfg = completed_planner_config({"gamma": 0.7, "horizon": 3, "C": 3})
    res = run_batch_against_oracle(envs_, cfg, list(range(256)))
    assert len(set(res[:, 0].tolist())) > 5


def test_highway_batch_of_64_scenes_equals_the_oracle():
    cfg = completed_planner_config({"gamma": 0.8, "horizon": 3, "C": 2})
    run_batch_against_oracle([oenvs.HighwayLite(seed=s) for s in range(64)], cfg, [100 + s for s in range(64)])


def test_one_stochastic_decision_at_horizon_5_equals_the_oracle():
    cfg = completed_planner_config({"gamma": 0.9, "horizon": 5, "C": 3})
    res = run_batch_against_oracle([case_env({"name": "stoch8"})], cfg, [3])
    assert res[0, 0] > 15000


def test_error_paths():
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.tree_search.sparse_sampling import SparseSamplingAgent
    from rl_agents_b200.engine.sparse_sampling import SparseSamplingEngine
    from rl_agents_b200.envs import FiniteMDPEnv
    shipped = completed_planner_config({"gamma": 0.7, "horizon": 3, "C": 3})
    # a rejected probability row that the search samples: numpy's own ValueError, engine and agent alike
    bad = case_env({"name": "stoch8_bad_root_row"})
    eng = engine_for(bad, shipped, 1)
    eng.plan(roots([bad]), pcg64_of([0]))
    with pytest.raises(ValueError) as e:
        eng.finish()
    assert str(e.value) == G["errors"]["bad_root_row"]["message"]
    assert int(eng.result[0, 4].item()) == 2 and int(eng.result[0, 5].item()) == 0 * 3 + 1
    t = G["mdps"]["stoch8_bad_root_row"]
    agent = SparseSamplingAgent(FiniteMDPEnv(np.array(t["transition"]), np.array(t["reward"]), np.array(t["terminal"]),
                                             mode="stochastic"), {"horizon": 3, "C": 3})
    with pytest.raises(ValueError, match="non-negative"):
        agent.plan(0)
    # a NaN row that no sample reaches plans normally (the golden case checks the plan itself)
    t = G["mdps"]["stoch8_unreached_nan_row"]
    agent = SparseSamplingAgent(FiniteMDPEnv(np.array(t["transition"]), np.array(t["reward"]), np.array(t["terminal"]),
                                             mode="stochastic"), {"horizon": 3, "C": 3})
    assert len(agent.plan(0)) == 1
    # the tree dump's capacity is checked
    env = case_env({"name": "stoch8"})
    eng = engine_for(env, shipped, 2, capacity=50)
    eng.plan(roots([env, env]), pcg64_of([0, 1]))
    with pytest.raises(RuntimeError, match="capacity"):
        eng.finish()
    assert (eng.result[:, 4].cpu().numpy() == 1).all()
    # the engine refuses what the reference cannot plan
    with pytest.raises(ValueError, match="zero-size array"):
        SparseSamplingEngine(_lib.ENV_HIGHWAY, 1, 5, 0, 3, 0.8)
    for horizon, C in ((-1, 3), (3, 0)):
        with pytest.raises(ValueError):
            SparseSamplingEngine(_lib.ENV_HIGHWAY, 1, 5, horizon, C, 0.8)
    with pytest.raises(NotImplementedError):
        SparseSamplingEngine(_lib.ENV_INTERSECTION, 1, 3, 3, 3, 0.8)
    # the C ABI refuses what the engine refuses
    eng = engine_for(env, shipped, 1, record=False)
    eng.cfg.env_kind = _lib.ENV_INTERSECTION
    with pytest.raises(_lib.B2Error, match="env_kind"):
        eng.plan(roots([env]), pcg64_of([0]))
    eng.cfg.env_kind, eng.cfg.C = _lib.ENV_FINITE, 0
    with pytest.raises(_lib.B2Error, match="C must be"):
        eng.plan(roots([env]), pcg64_of([0]))
    eng.cfg.C, eng.cfg.horizon = 3, 0
    with pytest.raises(_lib.B2Error, match="horizon"):
        eng.plan(roots([env]), pcg64_of([0]))


def test_plan_without_the_tree_dump_is_the_same_plan():
    env = case_env({"name": "garnet12"})
    cfg = completed_planner_config({"gamma": 0.7, "horizon": 3, "C": 3})
    out = []
    for record in (True, False):
        eng = engine_for(env, cfg, 4, record=record)
        eng.plan(roots([env] * 4), pcg64_of([0, 1, 2, 3]))
        plans, res, words = eng.finish()
        out.append((plans, res.tolist(), words.tolist(), eng.root_q.cpu().numpy().tobytes()))
    assert out[0] == out[1]


def test_agent_surface_matches_reference():
    """Built from sparse_sampling.json with `__class__` switched, as agent_factory builds it, on FiniteMDPEnv in all
    three modes and on HighwayLite: plans, RNG position and root values equal the reference's; seed / reset as the
    reference's; consecutive decisions carry the planner's stream on."""
    from rl_agents_b200.agents.tree_search.sparse_sampling import SparseSamplingAgent
    from rl_agents_b200.envs import FiniteMDPEnv, HighwayLiteEnv
    shipped = dict(G["configs"]["sparse_sampling_json"]["config"],
                   __class__="<class '%s.%s'>" % (SparseSamplingAgent.__module__, SparseSamplingAgent.__name__))

    def finite_env(name):
        t = G["mdps"].get(name)
        if t is None:
            return FiniteMDPEnv(M[name + "_T"], M[name + "_R"], M[name + "_term"])
        return FiniteMDPEnv(np.array(t["transition"]), np.array(t["reward"]), np.array(t["terminal"]), mode=t["mode"],
                            nxt=None if "next" not in t else np.array(t["next"]))
    for key, name in (("stoch8_shipped", "stoch8"), ("garnet12_sparse_shipped", "garnet12"),
                      ("large1_deterministic_shipped", "large1")):
        g = G["cases"][key]
        agent = SparseSamplingAgent(finite_env(name), dict(shipped))
        assert agent.seed(g["seed"]) == [g["seed"]]
        assert agent.plan(0) == g["plan"], key
        assert rng_state(agent.planner.np_random) == g["rng_state"], key
        assert np.array_equal(agent.planner.root_values, golden_root_q(g), equal_nan=True), key
    # reset() keeps the RNG stream; seed() restarts it
    g = G["cases"]["stoch8_shipped"]
    agent = SparseSamplingAgent(finite_env("stoch8"), dict(shipped))
    agent.seed(g["seed"])
    first = agent.plan(0)
    agent.reset()
    second = agent.plan(0)
    agent.seed(g["seed"])
    assert agent.plan(0) == first == g["plan"] and len(second) == 1
    # receding_horizon 3 still replans at every call: three decisions equal the reference's three
    g = G["cases"]["stoch8_three_decisions"]
    agent = SparseSamplingAgent(finite_env("stoch8"), dict(g["config"]))
    agent.seed(g["seed"])
    assert [agent.plan(0) for _ in range(3)] == g["plans"]
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    # HighwayLite through the env object
    g = G["cases"]["hw0_shipped"]
    agent = SparseSamplingAgent(HighwayLiteEnv(seed=0), dict(shipped))
    agent.seed(g["seed"])
    assert agent.act(None) == g["plan"][0]
    assert rng_state(agent.planner.np_random) == g["rng_state"]
    assert np.array_equal(agent.planner.root_values, golden_root_q(g), equal_nan=True)


def test_batched_evaluation_equals_per_episode_agents():
    from rl_agents_b200.agents.tree_search.sparse_sampling import SparseSamplingAgent
    from rl_agents_b200.envs import HighwayLiteEnv
    from rl_agents_b200.evaluation import run_batched_episodes
    seeds = [0, 1, 2, 3]
    kw = {"horizon": 2, "C": 2}
    out = run_batched_episodes("sparse_sampling", seeds, 0, 0.8, max_steps=6, planner_seed=50, **kw)
    for i, s in enumerate(seeds):
        env = HighwayLiteEnv(seed=s)
        agent = SparseSamplingAgent(env, dict(kw, gamma=0.8))
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
