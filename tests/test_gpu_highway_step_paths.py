"""hw::step (csrc/highway_lite.cuh) against the oracle on the scene families of tests/highway_scenes.py: more than 8
MOBIL deciders per sub-step, absent slots with stale words, exact x ties at entry and later, collisions between
vehicles that are not x-neighbours, the abort rule and the kinematic edges -- in the full-warp mode of the batched
step and the OPD kernels (two scenes per warp, one mask) and in the per-group mode of the one-tree-per-group planners
(each 16-lane half steps on its own), and through every kernel that calls the step.  Every comparison is exact."""
import numpy as np
import pytest

from oracle import c_oracle
from oracle import envs as oenvs
from oracle import planners
from tests import highway_scenes as hs

pytestmark = pytest.mark.gpu


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def all_runs():
    """(name, oracle trajectory, meets a tie) for every scene of every family"""
    out = []
    for name in hs.FAMILY_NAMES:
        for run, tie in zip(hs.family_trajectories(name), hs.scene_ties(name)):
            out.append(("%s[%d]" % (name, len(out)), run, tie))
    return out


def odd(xs):
    return xs if len(xs) % 2 else xs[:-1]


def batch_orders():
    """tie_with_free: every tie scene shares its warp (scenes 2g, 2g + 1) with a tie-free scene; free_only: tie-free
    scenes paired together, in another order.  Both odd, so the last warp has an idle group."""
    runs = all_runs()
    tie = [r for r in runs if r[2]]
    free = [r for r in runs if not r[2]]
    assert len(tie) >= 20 and len(free) > len(tie)
    mixed = []
    for i, f in enumerate(free):
        mixed += [tie[i], f] if i < len(tie) else [f]
    return {"tie_with_free": odd(mixed), "free_only": odd(free[::-1])}


@pytest.mark.parametrize("order", ["tie_with_free", "free_only"])
def test_full_warp_step_equals_the_oracle_on_every_family(order):
    import torch
    from rl_agents_b200 import _lib
    lib = _lib.load()
    runs = batch_orders()[order]
    n = len(runs)
    st = torch.tensor(np.stack([r[1][1][0] for r in runs]), dtype=torch.int32, device="cuda")
    rew = torch.empty(n, dtype=torch.float32, device="cuda")
    flg = torch.empty(n, dtype=torch.int32, device="cuda")
    avail = torch.empty(n, dtype=torch.int32, device="cuda")
    for k in range(hs.N_DECISIONS):
        act = torch.tensor([r[1][0][k] for r in runs], dtype=torch.int32, device="cuda")
        _lib.check(lib.b2_highway_step(_lib.ptr(st), _lib.ptr(act), _lib.ptr(rew), _lib.ptr(flg), _lib.ptr(avail), n,
                                       _lib.current_stream()))
        got, r_got, f_got, a_got = st.cpu().numpy(), rew.cpu().numpy(), flg.cpu().numpy(), avail.cpu().numpy()
        for i, (name, (acts, words, rews, flags, av), _) in enumerate(runs):
            assert np.array_equal(got[i], words[k + 1]), (name, k, np.nonzero(got[i] != words[k + 1])[0])
            assert r_got[i].view(np.int32) == rews[k].view(np.int32), (name, k)
            assert f_got[i] == flags[k] and a_got[i] == av[k], (name, k)


def test_half_warp_step_equals_the_oracle_on_every_family():
    """Per-group mode (HighwayEnv::step, gmask = 0xFFFF << (lane & 16)): the two scenes of a warp take different numbers
    of decisions, so after the shorter one returns the other steps alone; every intermediate state is compared."""
    import torch
    from rl_agents_b200 import _lib
    lib = _lib.load()
    runs = batch_orders()["tie_with_free"]
    n, m = len(runs), hs.N_DECISIONS
    # scenes 2g and 2g + 1 share a warp: 1 + a and m - a decisions (never equal for even m)
    n_steps = np.array([1 + (3 * (i // 2)) % m if i % 2 == 0 else m - (3 * (i // 2)) % m for i in range(n)], np.int32)
    assert all(n_steps[g] != n_steps[g + 1] for g in range(0, n - 1, 2)) and n_steps.max() == m
    roots = torch.tensor(np.stack([r[1][1][0] for r in runs]), dtype=torch.int32, device="cuda")
    acts = torch.tensor(np.stack([r[1][0] for r in runs]), dtype=torch.int32, device="cuda")
    trace = torch.full((n, m, 136), -1, dtype=torch.int32, device="cuda")
    rew = torch.zeros((n, m), dtype=torch.float32, device="cuda")
    flg = torch.full((n, m), -1, dtype=torch.int32, device="cuda")
    _lib.check(lib.b2_selftest_highway_step_groups(_lib.ptr(roots), _lib.ptr(acts),
                                                   _lib.ptr(torch.from_numpy(n_steps).cuda()), _lib.ptr(trace),
                                                   _lib.ptr(rew), _lib.ptr(flg), n, m, _lib.current_stream()))
    trace, rew, flg = trace.cpu().numpy(), rew.cpu().numpy(), flg.cpu().numpy()
    for i, (name, (_, words, rews, flags, av), _) in enumerate(runs):
        for k in range(n_steps[i]):
            assert np.array_equal(trace[i, k], words[k + 1]), (name, k, np.nonzero(trace[i, k] != words[k + 1])[0])
            assert rew[i, k].view(np.int32) == rews[k].view(np.int32), (name, k)
            assert flg[i, k] == flags[k] | (av[k] << 2), (name, k)
        assert (trace[i, n_steps[i]:] == -1).all() and (flg[i, n_steps[i]:] == -1).all()


# --------------------------------------------------------------------------------------- every caller of the step ----
SPECIAL = [("entry_ties", 0), ("late_ties", 0), ("absent", 0), ("entry_ties", 8), ("late_ties", 1), ("absent", 3),
           ("adapter", 0), ("entry_ties", 2), ("late_ties", 2), ("absent", 6), ("entry_ties", 9), ("late_ties", 3),
           ("adapter", 4), ("absent", 9), ("entry_ties", 10), ("late_ties", 5)]
ORDINARY = [("sync_timers", 0), ("kinematic", 0), ("jam", 0), ("sync_timers", 1), ("kinematic", 1), ("adapter", 9),
            ("sync_timers", 2), ("kinematic", 3), ("jam", 1), ("sync_timers", 5), ("kinematic", 6), ("adapter", 11),
            ("sync_timers", 6), ("kinematic", 8), ("jam", 4), ("sync_timers", 7)]


def roots(n):
    """n root scenes, tie and absent-slot scenes alternating with ordinary ones (so they share warps)"""
    picks = [p for pair in zip(SPECIAL, ORDINARY) for p in pair][:n]
    return [hs.family(name)[i] for name, i in picks]


def words_of(states):
    return [s.pack() for s in states]


def assert_opd_tree(d, t, res_row=None):
    for k in ("parent", "action", "count", "depth", "first_child", "n_children"):
        assert np.array_equal(np.asarray(d[k], dtype=np.int64), t[k].astype(np.int64)), k
    assert np.array_equal(d["done"], t["done"].astype(bool))
    for k in ("reward", "lower", "upper"):
        assert np.array_equal(d[k], t[k]), k
    if res_row is not None:
        assert res_row[0] == len(t["parent"]) and res_row[1] == t["n_leaves"]


@pytest.mark.parametrize("n_trees", [7, 24])
def test_opd_kernels_equal_the_c_oracle(n_trees):
    """7 trees: one tree per CTA (opd_highway_kernel); 24 trees: the batch kernel (opd_highway_multi_kernel)."""
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDEngine
    words = words_of(roots(n_trees))
    budget = 500 if n_trees < 16 else 300
    eng = OPDEngine(_lib.ENV_HIGHWAY, n_trees, 5, budget, 0.8)
    eng.plan(torch.tensor(np.stack(words), dtype=torch.int32, device="cuda"))
    plans, res = eng.finish([np_random(0) for _ in words])
    for i, w in enumerate(words):
        assert_opd_tree(eng.tree_dict(i), c_oracle.opd_plan(w, budget, 0.8), res[i])


def test_opd_wavefront_and_speculative_equal_their_specifications():
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDSpeculativeEngine, OPDWaveEngine
    wave = OPDWaveEngine(_lib.ENV_HIGHWAY, 5, 600, 0.8, 16)
    spec = OPDSpeculativeEngine(_lib.ENV_HIGHWAY, 5, 600, 0.8, 16)
    for w in words_of(roots(8)):
        wave.plan(torch.tensor(w, dtype=torch.int32, device="cuda"))
        _, res = wave.finish([np_random(0)])
        c = c_oracle.opd_plan_wave(w, 600, 0.8, 16)
        assert_opd_tree(wave.tree_dict(0), c, res[0])
        assert int(res[0, 7]) == c["n_waves"]
        spec.plan(torch.tensor(w, dtype=torch.int32, device="cuda"))
        spec.finish([np_random(0)])
        assert_opd_tree(spec.tree_dict(0), c_oracle.opd_plan(w, 600, 0.8))
    # the C strict tree is the Python restatement's (on one tie scene; test_c_oracle pins the rest)
    s = hs.family("late_ties")[0]
    _, tp = planners.opd_plan(oenvs.HighwayLite(s), 60, 0.8, np_random=np_random(0))
    tc = c_oracle.opd_plan(s.pack(), 60, 0.8)
    assert tc["parent"].tolist() == tp.parent and np.array_equal(tc["upper"], np.array(tp.upper))


def test_mcts_kernel_equals_the_c_oracle():
    from oracle.pcg64 import PCG64
    from rl_agents_b200 import _lib
    from tests.test_gpu_engines import run_mcts
    words = words_of(roots(24))
    eng, plans, res, rng_words, _ = run_mcts(_lib.ENV_HIGHWAY, words, 100, 6, 0.8, 10.0, list(range(1, 25)))
    for i, w in enumerate(words):
        t, rw = c_oracle.mcts_plan(w, 100, 6, 0.8, 10.0, PCG64.from_numpy(np_random(i + 1)).words())
        d = eng.tree_dict(i)
        assert res[i, 0] == len(t["parent"]), i
        for k in ("parent", "action", "count", "first_child", "n_children"):
            assert np.array_equal(np.asarray(d[k], dtype=np.int64), t[k].astype(np.int64)), (i, k)
        assert np.array_equal(d["value"], t["value"]) and np.array_equal(d["prior"], t["prior"]), i
        assert rng_words[i].tolist() == rw.tolist(), i


def test_mcts_wavefront_kernel_equals_the_c_specification():
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import MCTSWaveEngine
    eng = MCTSWaveEngine(_lib.ENV_HIGHWAY, 5, 200, 6, 0.8, 10.0, 16)
    for seed, w in enumerate(words_of(roots(8))):
        eng.plan(torch.tensor(w, dtype=torch.int32, device="cuda"), seed)
        c = c_oracle.mcts_plan_wave(w, 200, 6, 0.8, 10.0, 16, seed)
        _, res = eng.finish()
        d = eng.tree_dict()
        for k in ("parent", "first_child", "n_children", "count", "vsum"):
            assert np.array_equal(d[k], c[k]), (seed, k)
        assert np.array_equal(d["value"], c["value"])
        used = c["parent"] != -2
        assert np.array_equal(d["action"][used], c["action"][used]) and int(res[2]) == c["env_steps"]


def test_olop_kernel_equals_the_oracle():
    import torch
    from oracle import ref_loader
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.mcts import pcg64_words
    from rl_agents_b200.engine.olop import OLOPEngine
    ub = {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)"}
    states = roots(16)
    eng = OLOPEngine(_lib.ENV_HIGHWAY, len(states), 5, 12, 4, 0.8, ub, "uniform")
    eng.plan(torch.tensor(np.stack(words_of(states)), dtype=torch.int32, device="cuda"),
             np.stack([pcg64_words(np_random(7 + i)) for i in range(len(states))]))
    plans, _, _ = eng.finish()
    for i, s in enumerate(states):
        rng, _ = ref_loader.legacy_np_random(7 + i)
        plan, t = planners.olop_plan(oenvs.LegacyStepEnv(oenvs.HighwayLite(s.copy())), 0, 0.8, rng, upper_bound=ub,
                                     continuation_type="uniform", episodes=12, horizon=4)
        d = eng.tree_dict(i)
        assert plans[i] == plan, i
        assert d["parent"].tolist() == t.parent and d["count"].tolist() == t.count and d["action"].tolist() == t.action
        np.testing.assert_array_equal(d["cumulative_reward"], np.array(t.cumulative_reward, dtype=float))
        # upper bounds go through the KL solve's log(), whose device and numpy results may differ by an ulp
        np.testing.assert_allclose(d["upper"], np.array(t.upper), rtol=1e-9)


def test_brue_kernel_equals_the_oracle():
    from tests.test_brue_oracle import completed_planner_config
    from tests.test_gpu_brue import run_batch_against_oracle
    cfg = completed_planner_config({"budget": 60, "gamma": 0.8, "horizon": 4})
    run_batch_against_oracle([oenvs.HighwayLite(s) for s in roots(16)], cfg, list(range(200, 216)))


def test_mdp_gape_kernel_equals_the_oracle():
    from tests.test_gpu_mdp_gape import run_batch_against_oracle
    from tests.test_mdp_gape_oracle import completed_planner_config
    cfg = completed_planner_config({"budget": 100, "gamma": 0.7, "accuracy": 2.0, "confidence": 1,
                                    "upper_bound": {"threshold": "1*np.log(time)"}})
    run_batch_against_oracle([oenvs.HighwayLite(s) for s in roots(8)], cfg, list(range(300, 308)))


def test_sparse_sampling_kernel_equals_the_oracle():
    from tests.test_gpu_sparse_sampling import run_batch_against_oracle
    from tests.test_sparse_sampling_oracle import completed_planner_config
    cfg = completed_planner_config({"gamma": 0.8, "horizon": 4, "C": 1})
    run_batch_against_oracle([oenvs.HighwayLite(s) for s in roots(4)], cfg, [400, 401, 402, 403])


def test_mcts_dpw_kernel_equals_the_oracle():
    from tests.test_gpu_mcts_dpw import run_batch_against_oracle
    from tests.test_mcts_dpw_oracle import completed_planner_config
    cfg = completed_planner_config({"horizon": 5, "episodes": 30})
    run_batch_against_oracle([oenvs.HighwayLite(s) for s in roots(16)], cfg, list(range(500, 516)))
