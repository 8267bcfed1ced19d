"""GPU tests of the device re-root of MCTS trees, b2_mcts_reroot (csrc/mcts_reroot.cu), and of the closed-loop episodes
that keep their trees across decisions with it (evaluation.run_batched_episodes("mcts", ..., step_strategy="subtree")).

The kernel is checked bit for bit against its specification engine/mcts.py::reroot_arrays on trees from real batched
searches; the batched episodes against one MCTSAgent per episode with step_strategy "subtree"."""
import copy

import numpy as np
import pytest

from tests.test_gpu_eval_finite import ENV_SEED, GAMMA, N, PLANNER_SEED, STEPS, make_env, mdp_spec, words_of

pytestmark = pytest.mark.gpu
UNWRITTEN = -7
FIELDS = ("parent", "first_child", "count", "meta", "value", "prior")


def planner_rng(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def searched(kind, n=256, capacity=None):
    """-> (engine, its number of actions) after one batched search of n trees on `kind`."""
    import torch
    from oracle import envs as oenvs
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import MCTSEngine
    from rl_agents_b200.envs import highway_lite, intersection_lite
    dev = torch.device("cuda")
    env_words = None
    if kind == "garnet_sparse":
        P, nxt, R = oenvs.garnet(200, 4, 3, seed=0)
        mdp = oenvs.FiniteMDPLite(P, R, None, mode="sparse", nxt=nxt).mdp
        E, A, roots = _lib.ENV_FINITE, 4, torch.arange(n, dtype=torch.int32, device=dev) % 200
        env_words = np.stack([words_of(planner_rng(10 ** 6 + i)) for i in range(n)])
    elif kind == "garnet_deterministic":
        T, R = oenvs.garnet(200, 3, 3, seed=1, deterministic=True)
        mdp = oenvs.FiniteMDPLite(T, R, None).mdp
        E, A, roots = _lib.ENV_FINITE, 3, torch.arange(n, dtype=torch.int32, device=dev) % 200
    elif kind == "highway":
        mdp, E, A = None, _lib.ENV_HIGHWAY, 5
        roots = torch.from_numpy(np.stack([highway_lite.make_scene(s) for s in range(n)])).to(dev)
    else:
        mdp, E, A = None, _lib.ENV_INTERSECTION, intersection_lite.N_ACTIONS
        roots = torch.from_numpy(np.stack([intersection_lite.make_scene(s) for s in range(n)])).to(dev)
    eng = MCTSEngine(E, n, A, 60, 6, 0.8, 10.0, mdp=mdp, device=dev, capacity=capacity)
    eng.plan(roots, np.stack([words_of(planner_rng(i)) for i in range(n)]), None, env_words)
    eng.finish()
    assert eng.sampled == (kind == "garnet_sparse")
    return eng, A


def host_trees(eng):
    res = eng.result.cpu().numpy()
    arrays = {k: getattr(eng, k).cpu().numpy() for k in FIELDS}
    return [{k: arrays[k][i, :res[i, 0]] for k in FIELDS} for i in range(eng.n_trees)]


def device_reroot(eng, actions, sources=None, n_dst=None, capacity=None, reserve=0):
    """b2_mcts_reroot from eng's arena into a new sentinel-filled one -> (kept, destination arrays as numpy)."""
    import torch
    from rl_agents_b200 import _lib
    n_dst = eng.n_trees if n_dst is None else n_dst
    capacity = eng.capacity if capacity is None else capacity
    dst = {k: torch.full((n_dst, capacity), UNWRITTEN, device=eng.device, dtype=getattr(eng, k).dtype) for k in FIELDS}
    act = torch.as_tensor(np.asarray(actions, np.int32), device=eng.device)
    src = None if sources is None else torch.as_tensor(np.asarray(sources, np.int32), device=eng.device)
    kept = torch.full((n_dst,), UNWRITTEN, dtype=torch.int32, device=eng.device)
    _lib.check(eng.lib.b2_mcts_reroot(eng.tree, eng.n_trees, eng.capacity, _lib.ptr(eng.result), _lib.MCTS_RESULT_WORDS,
                                      _lib.MCTSTree(*[dst[k].data_ptr() for k in FIELDS]), n_dst, capacity,
                                      _lib.ptr(src), _lib.ptr(act), reserve, _lib.ptr(kept), _lib.current_stream()))
    return kept.cpu().numpy(), {k: v.cpu().numpy() for k, v in dst.items()}


def assert_equals_spec(trees, kept, dst, actions, sources, capacity, reserve=0):
    """Every destination tree against reroot_arrays; -> the kept counts the specification gives."""
    from rl_agents_b200.engine.mcts import reroot_arrays
    expected = []
    for j, a in enumerate(actions):
        s = j if sources is None else sources[j]
        if not 0 <= s < len(trees):
            assert kept[j] == -1, j
            for k in FIELDS:
                assert (dst[k][j] == UNWRITTEN).all(), (j, k)           # the destination is untouched
            expected.append(-1)
            continue
        out, k_ = reroot_arrays(trees[s], len(trees[s]["parent"]), int(a))
        if k_ + reserve > capacity:
            k_ = 0
        assert kept[j] == k_, (j, s, a)
        for f in FIELDS if k_ else ():
            assert dst[f][j, :k_].tobytes() == out[f].tobytes(), (j, f)
        expected.append(k_)
    return np.array(expected)


@pytest.mark.parametrize("kind", ["garnet_sparse", "garnet_deterministic", "highway", "intersection"])
def test_kernel_equals_reroot_arrays(kind):
    eng, A = searched(kind)
    trees = host_trees(eng)
    n = eng.n_trees
    rng = np.random.default_rng(3)
    seen = set()
    for a in range(-1, A + 1):                  # every root action, -1 and one beyond the action set
        actions = np.full(n, a)
        kept, dst = device_reroot(eng, actions)
        got = assert_equals_spec(trees, kept, dst, actions, None, eng.capacity)
        seen.update(np.sign(got).tolist())
    assert {0, 1} <= seen                       # unexpanded actions and kept sub-trees both occur
    actions = rng.integers(-1, A, n)
    for sources in (rng.permutation(n), rng.integers(0, n, n), np.zeros(n, int)):    # permuted and repeated sources
        kept, dst = device_reroot(eng, actions, sources)
        assert_equals_spec(trees, kept, dst, actions, sources, eng.capacity)
    # a smaller destination arena gathers a subset, as the finite harness does when episodes end
    sources = np.sort(rng.choice(n, n // 3, replace=False))
    kept, dst = device_reroot(eng, actions[sources], sources, n_dst=len(sources))
    assert_equals_spec(trees, kept, dst, actions[sources], sources, eng.capacity)


@pytest.mark.parametrize("kind", ["garnet_sparse", "highway"])
def test_capacity_fallback_and_bad_sources(kind):
    eng, A = searched(kind)
    trees = host_trees(eng)
    n = eng.n_trees
    rng = np.random.default_rng(5)
    actions = rng.integers(0, A, n)
    full, _ = device_reroot(eng, actions)
    big = np.sort(full[full > 0])
    assert big.size > 10
    # kept + reserve > capacity -> 0: a reserve that lets about half of the kept sub-trees fit
    capacity = eng.capacity
    reserve = capacity - int(big[big.size // 2])
    kept, dst = device_reroot(eng, actions, reserve=reserve)
    got = assert_equals_spec(trees, kept, dst, actions, None, capacity, reserve)
    assert (got == 0).sum() > (full == 0).sum() and (got > 0).any()
    # a smaller destination capacity: the same rule against it
    small = int(big[big.size // 2]) + 4
    kept, dst = device_reroot(eng, actions, capacity=small, reserve=4)
    assert_equals_spec(trees, kept, dst, actions, None, small, 4)
    # out-of-range sources: -1, the destination untouched; the others re-rooted as usual
    sources = np.arange(n)
    sources[::7], sources[3::11] = -1, n
    sources[5] = 2 ** 31 - 1
    kept, dst = device_reroot(eng, actions, sources)
    got = assert_equals_spec(trees, kept, dst, actions, sources, capacity)
    assert (got == -1).sum() == ((sources < 0) | (sources >= n)).sum()
    # the identity mapping over more destination trees than source trees
    kept, dst = device_reroot(eng, np.concatenate([actions, actions[:5]]), n_dst=n + 5)
    assert (kept[n:] == -1).all()
    assert_equals_spec(trees, kept[:n], {k: v[:n] for k, v in dst.items()}, actions, None, capacity)


def test_source_node_count_out_of_range_is_reported():
    """A source whose node count word is outside [1, capacity] is not read: -1, the destination untouched."""
    eng, A = searched("garnet_deterministic", n=64)
    trees = host_trees(eng)
    res = eng.result.clone()
    eng.result[1, 0], eng.result[2, 0], eng.result[3, 0] = 0, -5, eng.capacity + 1
    kept, dst = device_reroot(eng, np.zeros(64, int))
    eng.result.copy_(res)
    assert kept[1:4].tolist() == [-1, -1, -1]
    for k in FIELDS:
        assert (dst[k][1:4] == UNWRITTEN).all()
    keep = [0] + list(range(4, 64))
    assert_equals_spec([trees[i] for i in keep], kept[keep], {k: v[keep] for k, v in dst.items()},
                       np.zeros(len(keep), int), None, eng.capacity)


def test_engine_reroot_in_place_swaps_the_spare_arena():
    """MCTSEngine.reroot: the re-rooted trees are the engine's arena afterwards (tree_dict and the plan kernel read
    them), and a resumed search grows them."""
    from rl_agents_b200.agents.tree_search.mcts import subtree_capacity
    from rl_agents_b200.engine.mcts import pcg64_words, reroot_arrays
    from rl_agents_b200.envs import highway_lite
    n = 32
    eng, A = searched("highway", n=n, capacity=subtree_capacity(60, 6, 5))
    trees = host_trees(eng)
    before = eng.tree.parent
    actions = [int(p) for p in eng.plan_buf[:, 0].cpu().numpy()]
    kept = eng.reroot(actions)
    assert eng.tree.parent != before and eng.tree.parent == eng.parent.data_ptr()
    assert (kept >= 1).all() and (kept > 1).sum() > n // 2
    for i in range(n):
        out, k = reroot_arrays(trees[i], len(trees[i]["parent"]), actions[i])
        assert kept[i] == k
        d = eng.tree_dict(i)
        for f in FIELDS:
            assert getattr(eng, f)[i, :k].cpu().numpy().tobytes() == out[f].tobytes(), (i, f)
        assert d["parent"][:k].tolist() == out["parent"].tolist()
    # a resumed search continues from the kept nodes: the root keeps its visits and gains the new episodes'
    scenes = eng.torch.from_numpy(np.stack([highway_lite.make_scene(s) for s in range(n)])).to(eng.device)
    root_counts = eng.count[:, 0].cpu().numpy().copy()
    eng.plan(scenes, np.stack([pcg64_words(planner_rng(i)) for i in range(n)]), kept)
    res = eng.finish()[1]
    assert (eng.count[:, 0].cpu().numpy() == root_counts + 60).all()
    assert (res[:, 0] >= kept).all() and (res[:, 0] > kept).any()
    eng.reroot(actions)
    assert eng.tree.parent == before                             # the first arena served as the spare


def test_refusals_launch_no_kernel():
    import torch
    from rl_agents_b200 import _lib
    eng, A = searched("garnet_deterministic", n=4)
    lib = eng.lib
    other = {k: torch.empty_like(getattr(eng, k)) for k in FIELDS}
    dst = _lib.MCTSTree(*[other[k].data_ptr() for k in FIELDS])
    act = torch.zeros(4, dtype=torch.int32, device=eng.device)
    kept = torch.empty(4, dtype=torch.int32, device=eng.device)
    base = dict(src=eng.tree, n_src=4, src_cap=eng.capacity, nodes=_lib.ptr(eng.result), stride=_lib.MCTS_RESULT_WORDS,
                dst=dst, n_dst=4, dst_cap=eng.capacity, src_tree=None, action=_lib.ptr(act), reserve=0,
                kept=_lib.ptr(kept))

    def call(**over):
        a = dict(base, **over)
        kept.fill_(UNWRITTEN)
        rc = lib.b2_mcts_reroot(a["src"], a["n_src"], a["src_cap"], a["nodes"], a["stride"], a["dst"], a["n_dst"],
                                a["dst_cap"], a["src_tree"], a["action"], a["reserve"], a["kept"],
                                _lib.current_stream())
        torch.cuda.synchronize()
        return rc

    assert call() == 0 and (kept != UNWRITTEN).all()              # the accepted call launched and wrote kept

    def with_field(tree, field, value):
        t = _lib.MCTSTree.from_buffer_copy(tree)
        setattr(t, field, value)
        return t

    cases = [(dict(src=None), "null pointer"), (dict(dst=None), "null pointer"), (dict(nodes=None), "null pointer"),
             (dict(action=None), "null pointer"), (dict(kept=None), "null pointer")]
    cases += [(dict(src=with_field(eng.tree, f, None)), "null pointer") for f in FIELDS]
    cases += [(dict(dst=with_field(dst, f, None)), "null pointer") for f in FIELDS]
    cases += [(dict(n_dst=0), "n_dst must be >= 1"), (dict(n_dst=-3), "n_dst must be >= 1")]
    cases += [(dict(**{k: 0}), "n_src, capacities and src_nodes_stride must be >= 1")
              for k in ("n_src", "src_cap", "dst_cap", "stride")]
    cases += [(dict(dst=eng.tree), "must not share an array"),
              (dict(dst=with_field(dst, "value", eng.tree.value)), "must not share an array"),
              (dict(dst=with_field(dst, "count", eng.tree.meta)), "must not share an array")]
    cases += [(dict(reserve=-1), "reserve must be >= 0")]
    for over, msg in cases:
        assert call(**over) == 1, over                           # B2_ERR_INVALID
        assert msg in lib.b2_last_error().decode(), over
        assert (kept == UNWRITTEN).all(), over                   # no kernel ran
    assert call(src_tree=_lib.ptr(torch.arange(4, dtype=torch.int32, device=eng.device))) == 0


# -- closed-loop episodes with step_strategy "subtree" ----------------------------------------------------------------

SUBTREE = {"step_strategy": "subtree"}


def finite_agent_episodes(name, starts, budget):
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    out = {"actions": [], "rewards": [], "final_states": [], "planner_words": [], "env_words": []}
    for i, s0 in enumerate(starts):
        env = make_env(name, int(s0), seed=ENV_SEED + i)
        agent = MCTSAgent(env, dict(SUBTREE, budget=budget, gamma=GAMMA))
        agent.seed(PLANNER_SEED + i)
        acts, rews = [], []
        for _ in range(STEPS):
            a = int(agent.act(env.mdp.state))
            s2, r, done, _, _ = env.step(a)
            acts.append(a)
            rews.append(r)
            if done:
                break
        out["actions"].append(acts)
        out["rewards"].append(rews)
        out["final_states"].append(env.mdp.state)
        out["planner_words"].append(words_of(agent.planner.np_random))
        out["env_words"].append(words_of(env.np_random))
    return out


@pytest.mark.parametrize("name", ["large1", "trap", "loop", "garnet50", "dense6", "dup20", "term40"])
def test_finite_subtree_episodes_equal_per_episode_agents(name):
    from rl_agents_b200.evaluation import run_batched_episodes
    budget = 40
    S = mdp_spec(name)[2].shape[0]
    starts = np.arange(N) % S
    expected = finite_agent_episodes(name, starts, budget)
    out = run_batched_episodes("mcts", list(range(N)), budget, GAMMA, max_steps=STEPS, env="finite",
                               planner_seed=PLANNER_SEED, mdp=make_env(name), start_states=starts, env_seed=ENV_SEED,
                               **copy.deepcopy(SUBTREE))
    reset = run_batched_episodes("mcts", list(range(N)), budget, GAMMA, max_steps=STEPS, env="finite",
                                 planner_seed=PLANNER_SEED, mdp=make_env(name), start_states=starts, env_seed=ENV_SEED)
    for i in range(N):
        k = len(expected["actions"][i])
        assert out["lengths"][i] == k, i
        assert out["actions"][i, :k].tolist() == expected["actions"][i], i
        assert out["rewards"][i, :k].tobytes() == np.array(expected["rewards"][i], np.float64).tobytes(), i
        assert out["final_states"][i] == expected["final_states"][i], i
        assert (out["env_words"][i] == expected["env_words"][i]).all(), i
        assert (out["planner_words"][i] == expected["planner_words"][i]).all(), i
    assert out["resumed"].sum() > 0                             # sub-trees were kept and searched on
    assert "resumed" not in reset
    # a resumed tree draws differently from a fresh one: the planner streams show the re-root was followed
    assert any((out["planner_words"][i] != reset["planner_words"][i]).any() for i in range(N))
    if name in ("term40", "trap"):
        assert len(set(out["lengths"].tolist())) > 1            # episodes end at different steps: the gather path


@pytest.mark.parametrize("env_name", ["highway", "intersection"])
def test_scene_subtree_episodes_equal_per_scene_agents(env_name):
    from rl_agents_b200.agents.tree_search.mcts import MCTSAgent
    from rl_agents_b200.envs import HighwayLiteEnv, IntersectionLiteEnv
    from rl_agents_b200.evaluation import run_batched_episodes
    seeds, steps, budget = [0, 1, 2, 3], 8, 150
    out = run_batched_episodes("mcts", seeds, budget, 0.8, max_steps=steps, planner_seed=100, env=env_name,
                               step_strategy="subtree")
    make = HighwayLiteEnv if env_name == "highway" else IntersectionLiteEnv
    for i, s in enumerate(seeds):
        env = make(seed=s)
        agent = MCTSAgent(env, {"budget": budget, "gamma": 0.8, "step_strategy": "subtree"})
        agent.seed(100 + i)
        total, n_steps = 0.0, 0
        for k in range(steps):
            a = agent.act(None)
            assert a == out["actions"][i, k], (s, k)
            _, r, term, trunc, _ = env.step(a)
            total += float(np.float32(r)) if env_name == "highway" else r
            n_steps += 1
            if term or trunc:
                break
        assert n_steps == out["lengths"][i] and abs(total - out["returns"][i]) < 1e-9, s
    assert out["resumed"].sum() > 0
    assert out["lengths"].max() >= 6
