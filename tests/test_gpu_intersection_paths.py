"""il::step (csrc/intersection_lite.cuh) and the OPD kernels on IntersectionLite against the C and Python statements of
the spec, on the scene families of tests/intersection_scenes.py: arrivals (and crashes in the same step), full slots,
blocked spawns at the clear distance, exact front ties, threshold positions, crossing collisions, the spawn counter's
wrap, stale absent slots -- with the two scenes of a warp spawning on different sub-steps, so that the spawn branch
runs on one 16-lane group while the other skips it.  Trees from a few hundred nodes to the full C5 size (budget 1e6)
are compared whole.  Every comparison is exact."""
import concurrent.futures

import numpy as np
import pytest

from oracle import c_oracle
from oracle import intersection as oit
from oracle import planners
from tests import intersection_scenes as its

pytestmark = pytest.mark.gpu

GAMMA = 0.9


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def all_roots():
    """(name, seed of its action stream, start words) for every scene of every family"""
    out = []
    for name in its.FAMILY_NAMES:
        for i, s in enumerate(its.family(name)):
            out.append(("%s[%d]" % (name, i), i, s.pack()))
    return out


def warp_order(roots):
    """Pairs every scene with one whose spawn clock gives different spawn sub-steps at the first decision (the clocks
    of two scenes keep their difference, so the pair stays divergent), where one is left."""
    left, out = list(roots), []
    while left:
        a = left.pop(0)
        out.append(a)
        if not left:
            break
        j = next((j for j, b in enumerate(left) if its.spawn_substeps(b[2][130]) != its.spawn_substeps(a[2][130])), 0)
        out.append(left.pop(j))
    return out


def step_batch_against_c(roots, n_decisions=its.N_DECISIONS):
    """Steps the batch through b2_intersection_step and the C oracle in lock step, with each scene's ActionStream over
    the C states; compares all 136 words, the reward, the flags and the mask.  Returns the C words per decision."""
    import torch
    from rl_agents_b200 import _lib
    lib = _lib.load()
    n = len(roots)
    w = np.stack([r[2] for r in roots])
    st = torch.tensor(w, dtype=torch.int32, device="cuda")
    rew = torch.empty(n, dtype=torch.float32, device="cuda")
    flg = torch.empty(n, dtype=torch.int32, device="cuda")
    avail = torch.empty(n, dtype=torch.int32, device="cuda")
    picks = [its.ActionStream(r[1]) for r in roots]
    trace = [w]
    for k in range(n_decisions):
        acts = [picks[i](oit.IntersectionLiteState.unpack(w[i])) for i in range(n)]
        _lib.check(lib.b2_intersection_step(_lib.ptr(st), _lib.ptr(torch.tensor(acts, dtype=torch.int32, device="cuda")),
                                            _lib.ptr(rew), _lib.ptr(flg), _lib.ptr(avail), n, _lib.current_stream()))
        w, r_c, f_c = c_oracle.il_step_batch(w, acts)
        got, r_got, f_got, a_got = st.cpu().numpy(), rew.cpu().numpy(), flg.cpu().numpy(), avail.cpu().numpy()
        for i, (name, _, _) in enumerate(roots):
            assert np.array_equal(got[i], w[i]), (name, k, np.nonzero(got[i] != w[i])[0])
            assert r_got[i].view(np.int32) == r_c[i].view(np.int32) and f_got[i] == f_c[i], (name, k)
            assert a_got[i] == its.avail_mask(oit.IntersectionLiteState.unpack(w[i])), (name, k)
        trace.append(w)
    return np.stack(trace, axis=1)


@pytest.mark.parametrize("size", ["all_odd", "partial_cta"])
def test_batched_step_equals_the_c_oracle_on_every_family(size):
    """All families in one batch (odd: the last warp has an idle group), and a batch that leaves its last CTA (8
    scenes) partly empty, in another order; the warps' two scenes spawn on different sub-steps."""
    roots = warp_order(all_roots())
    if size == "all_odd":
        roots = roots if len(roots) % 2 else roots[:-1]
    else:
        roots = warp_order(all_roots()[::-1])
        roots = roots[:len(roots) - (len(roots) % 8) - 3]
        assert len(roots) % 8 == 5
    words = step_batch_against_c(roots)
    pairs = its.divergent_pairs(words)
    print(size, len(roots), "scenes,", pairs, "divergent warps")
    assert pairs >= len(roots) // 4


def test_single_scene_batches_equal_the_c_oracle():
    """Batch size 1 (one live group, the warp's other group idle) on the arrival, full and wrap scenes."""
    for name in ("arrival", "full", "wrap"):
        for i, s in enumerate(its.family(name)[:6]):
            step_batch_against_c([("%s[%d]" % (name, i), i, s.pack())])


def test_env_step_on_an_arrival_scene():
    """IntersectionLiteEnv.step (n = 1, no mask buffer) through an arrival in the second decision: reward 1,
    terminated."""
    from rl_agents_b200.envs import IntersectionLiteEnv
    s = its.family("arrival")[5]
    env = IntersectionLiteEnv(words=s.pack())
    w = s.pack()[None]
    arrived = False
    for k in range(3):
        _, r, term, trunc, _ = env.step(oit.A_IDLE)
        w, r_c, f_c = c_oracle.il_step_batch(w, [oit.A_IDLE])
        assert np.array_equal(env.words, w[0]) and np.float32(r) == r_c[0], k
        assert term == bool(f_c[0] & 1) and trunc == bool(f_c[0] & 2), k
        arrived = arrived or (r == 1.0 and term)
    assert arrived and env.words[132] == 1


# ------------------------------------------------------------------------------------------------- OPD kernels ----
ROOTS = [("arrival", 0), ("arrival", 13), ("full", 1), ("full", 4), ("ties", 2), ("ties", 7)]


def root_words(name, i):
    return its.family(name)[i].pack()


def tree_of(c):
    t = planners.Tree()
    for k in ("parent", "action", "depth", "count", "first_child", "n_children"):
        setattr(t, k, c[k].tolist())
    return t


def assert_opd_tree(d, c, res_row=None):
    for k in ("parent", "action", "count", "depth", "first_child", "n_children"):
        assert np.array_equal(np.asarray(d[k], dtype=np.int64), c[k].astype(np.int64)), k
    assert np.array_equal(d["done"], c["done"].astype(bool))
    for k in ("reward", "lower", "upper"):
        assert np.array_equal(d[k], c[k]), k
    if res_row is not None:
        assert res_row[0] == len(c["parent"]) and res_row[1] == c["n_leaves"]


@pytest.mark.parametrize("width", [1, 16, 64])
def test_wavefront_opd_equals_the_python_specification(width):
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDWaveEngine
    eng = OPDWaveEngine(_lib.ENV_INTERSECTION, 3, 240, GAMMA, width)
    for name, i in ROOTS:
        s = its.family(name)[i]
        eng.plan(torch.tensor(s.pack(), dtype=torch.int32, device="cuda"))
        plans, res = eng.finish([np_random(0)])
        plan, t = planners.opd_plan_wavefront(oit.IntersectionLite(s.copy()), 240, GAMMA, width, np_random=np_random(0))
        d = eng.tree_dict(0)
        assert plans[0] == plan, (name, i)
        assert d["parent"].tolist() == t.parent and d["action"].tolist() == t.action and d["count"].tolist() == t.count
        assert np.array_equal(d["reward"], np.array(t.reward)) and np.array_equal(d["lower"], np.array(t.lower))
        assert np.array_equal(d["upper"], np.array(t.upper)) and d["done"].tolist() == t.done, (name, i)
        assert int(res[0, 1]) == t.n_leaves and int(res[0, 7]) == len(t.waves), (name, i)


@pytest.mark.parametrize("width", [16, 64])
def test_speculative_opd_equals_the_c_strict_tree(width):
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDSpeculativeEngine
    eng = OPDSpeculativeEngine(_lib.ENV_INTERSECTION, 3, 900, GAMMA, width)
    for name, i in ROOTS:
        w = root_words(name, i)
        eng.plan(torch.tensor(w, dtype=torch.int32, device="cuda"))
        plans, _ = eng.finish([np_random(0)])
        c = c_oracle.il_opd_plan(w, 900, GAMMA)
        assert_opd_tree(eng.tree_dict(0), c)
        assert plans[0] == planners.greedy_plan(tree_of(c), c["lower"], np_random(0)), (name, i)


def wave_against_c(words, budget, width):
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDWaveEngine
    with concurrent.futures.ThreadPoolExecutor(1) as pool:        # the C tree is built while the GPU searches
        fut = pool.submit(c_oracle.il_opd_plan_wave, words, budget, GAMMA, width)
        eng = OPDWaveEngine(_lib.ENV_INTERSECTION, 3, budget, GAMMA, width)
        eng.plan(torch.tensor(words, dtype=torch.int32, device="cuda"))
        plans, res = eng.finish([np_random(0)])
        d = eng.tree_dict(0)
        c = fut.result()
    assert_opd_tree(d, c, res[0])
    assert int(res[0, 7]) == c["n_waves"]
    assert plans[0] == planners.greedy_plan(tree_of(c), c["lower"], np_random(0))
    return d, c


@pytest.mark.parametrize("budget", [24000, 30000])
def test_wavefront_opd_equals_c_around_one_tile(budget):
    """24 000: the largest tree whose frontier keys stay resident in one shared-memory tile (24 576); 30 000: just
    past it, the first size with distributed selection."""
    from rl_agents_b200.envs.intersection_lite import make_scene
    for w in (make_scene(0), root_words("arrival", 13)):
        wave_against_c(w, budget, 256)


@pytest.mark.parametrize("width", [256, 1024])
def test_distributed_selection_equals_c(width):
    """Budget 1e5 (100 000 nodes, four tiles of frontier keys): the selection is distributed over the CTAs."""
    from rl_agents_b200.envs.intersection_lite import make_scene
    wave_against_c(make_scene(0), 100000, width)


def spawn_phase_divergent_waves(c, root_clock):
    """Waves of the C tree in which the two children of some warp (work items 2g, 2g + 1: children wave_start + 2g and
    + 2g + 1) spawn on different sub-steps: a child's spawn clock is its parent's depth's, root_clock + 15 * depth."""
    n, start = 0, 1
    for end in c["wave_end"]:
        kids = np.arange(start, end)
        a, b = kids[0:len(kids) - 1:2], kids[1::2]
        ca = (root_clock + 15 * c["depth"][c["parent"][a]]) % oit.SPAWN_PERIOD
        cb = (root_clock + 15 * c["depth"][c["parent"][b]]) % oit.SPAWN_PERIOD
        n += any(its.spawn_substeps(x) != its.spawn_substeps(y) for x, y in zip(ca, cb))
        start = end
    return n


@pytest.mark.parametrize("width", [1024, 4096])
def test_c5_decision_at_full_size_equals_c(width):
    """BASELINE C5 as bench.py times it: make_scene(0), budget 1e6 (333 333 expansions), gamma 0.9, widths 1024 and
    4096 -- the whole tree, the plan, the frontier size and the wave count against the C statement."""
    from rl_agents_b200.envs.intersection_lite import make_scene
    words = make_scene(0)
    d, c = wave_against_c(words, 1000000, width)
    n = len(c["parent"])
    assert (d["n_children"] > 0).sum() == 1000000 // 3
    assert d["count"][0] == n and (d["parent"][1:] < np.arange(1, n)).all()
    assert (d["lower"] <= d["upper"] + 1e-12).all() and d["upper"][0] <= 1 / (1 - GAMMA) + 1e-9
    assert np.array_equal(np.bincount(d["parent"][1:], minlength=n)[:n], d["n_children"])
    assert c["depth"].max() > oit.DURATION                 # past t = DURATION: truncated nodes expand on
    assert spawn_phase_divergent_waves(c, int(words[130])) > 0
