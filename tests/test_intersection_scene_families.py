"""The IntersectionLite scene families (tests/intersection_scenes.py) on the CPU: each reaches the step paths it is built
for (census floors), the C statement of the spec (oracle/c/intersection_lite.c) equals the numpy statement on every
family bit for bit, and the C strict and wavefront OPD equal the Python planners on family roots -- so the C oracle
can stand in for the numpy one where the GPU tests need speed (a C5-sized tree is about a million steps)."""
import numpy as np
import pytest

from oracle import c_oracle
from oracle import intersection as oit
from oracle import planners
from tests import intersection_scenes as its

# per family: the paths it exists for, and how often its trajectories (13 decisions per scene) must reach each
FLOORS = {
    "phases": {"spawn": 60, "blocked": 40, "box_crossing_hit": 20, "ego_crash": 5},
    "arrival": {"arrival": 15, "arrive_crash": 4, "box_crossing_hit": 5},
    "full": {"spawn_full": 10, "spawn_freed": 4, "spawn": 20},
    "blocked": {"blocked": 20, "clear_edge": 4, "spawn": 20},
    "ties": {"front_tie": 16, "lane_hit": 200},
    "boundaries": {"arrival": 3, "box_lane_pair": 200, "box_crossing_hit": 200, "depart_left": 10,
                   "depart_straight": 10, "depart_right": 10},
    "crossing": {"box_crossing_hit": 100, "box_lane_pair": 10, "crossing_hit": 500},
    "wrap": {"seq_wrap": 6},
    "stale": {"spawn": 15, "blocked": 15, "ego_crash": 3},
}
ALL_FAMILIES_FLOORS = {"odd_action": 10, "yield": 100}


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def test_every_family_has_a_floor():
    assert set(FLOORS) == set(its.FAMILY_NAMES)
    assert all(set(f) <= set(its.PATHS) for f in FLOORS.values())


@pytest.mark.parametrize("name", its.FAMILY_NAMES)
def test_family_reaches_its_paths(name):
    counts = its.census(name)
    print(name, dict(counts))
    for path, floor in {**ALL_FAMILIES_FLOORS, **FLOORS[name]}.items():
        assert counts[path] >= floor, (name, path, counts[path], floor)


@pytest.mark.parametrize("name", its.FAMILY_NAMES)
def test_family_scenes_stay_in_the_state_domain(name):
    for s in its.family(name):
        w = s.pack()
        assert s.flags[0] & 1 and s.route[0] == oit.EGO_ROUTE and np.isfinite(w[:32].view(np.float32)).all()
        assert ((s.route >= 0) & (s.route < oit.N_ROUTES)).all() and ((s.flags >= 0) & (s.flags <= 3)).all()
        assert 0 <= s.speed_index <= 2 and 0 <= s.spawn_clock < oit.SPAWN_PERIOD and 0 <= s.spawn_seq <= its.SEQ_MAX
        assert s.arrived == 0 and (w[64:128] == 0).all() and (w[133:] == 0).all()


def test_phases_pairs_spawn_on_different_substeps():
    words = np.stack([r[1] for r in its.family_trajectories("phases")])
    assert its.divergent_pairs(words) == len(words) // 2
    assert sorted(s.spawn_clock for s in its.family("phases")) == list(range(oit.SPAWN_PERIOD))


def test_blocked_scenes_straddle_the_entry_clear_distance():
    """At the first sub-step the spawn is blocked one ulp below ENTRY_CLEAR and goes ahead at and above it."""
    for i, s in enumerate(its.family("blocked")):
        spawns = []
        oit.intersection_step(s.copy(), oit.A_IDLE, on_substep=lambda spawn, **_: spawns.append(spawn))
        assert spawns[0] is not None and spawns[0]["clear"] == (i % 3 != 0), i


def test_observer_leaves_the_step_unchanged():
    for name in ("full", "arrival", "crossing"):
        for s in its.family(name)[:4]:
            a, b = s.copy(), s.copy()
            ra = oit.intersection_step(a, oit.A_FASTER)
            rb = oit.intersection_step(b, oit.A_FASTER, on_substep=lambda **kw: None)
            assert ra == rb and np.array_equal(a.pack(), b.pack())


@pytest.mark.parametrize("name", its.FAMILY_NAMES)
def test_c_step_equals_numpy_step(name):
    runs = its.family_trajectories(name)
    assert len(runs[0][0]) >= 13
    w = np.stack([r[1][0] for r in runs])
    for k in range(len(runs[0][0])):
        w, rew, flg = c_oracle.il_step_batch(w, [r[0][k] for r in runs])
        for i, r in enumerate(runs):
            assert np.array_equal(w[i], r[1][k + 1]), (name, i, k, np.nonzero(w[i] != r[1][k + 1])[0])
            assert rew[i].view(np.int32) == r[2][k].view(np.int32) and flg[i] == r[3][k], (name, i, k)


def test_unavailable_and_out_of_range_actions_leave_the_speed_index():
    for si, a in ((0, oit.A_SLOWER), (2, oit.A_FASTER), (1, 7), (0, 7), (2, -1)):
        s = its.family("phases")[0]
        s.speed_index = si
        w, _, _ = c_oracle.il_step_batch(s.pack()[None], [a])
        ref = s.copy()
        oit.intersection_step(ref, a)
        assert ref.speed_index == si and np.array_equal(w[0], ref.pack())


# roots of the planner comparisons: an arrival root whose tree contains arrivals, a crash-and-arrive root, a full
# scene, a tie scene, a blocked scene and one of each spawn phase pair
PLANNER_ROOTS = [("arrival", 0), ("arrival", 13), ("full", 1), ("ties", 2), ("blocked", 1), ("phases", 3)]


def root_state(name, i):
    return its.family(name)[i]


def assert_c_tree_equals(c, t):
    for k in ("parent", "action", "depth", "count", "first_child", "n_children"):
        assert c[k].tolist() == list(getattr(t, k)), k
    assert c["done"].astype(bool).tolist() == [bool(x) for x in t.done]
    for k in ("reward", "lower", "upper"):
        assert np.array_equal(c[k], np.array(getattr(t, k), dtype=np.float64)), k
    assert c["n_leaves"] == t.n_leaves


@pytest.mark.parametrize("name,i", PLANNER_ROOTS)
def test_c_strict_opd_equals_the_python_planner(name, i):
    s = root_state(name, i)
    _, t = planners.opd_plan(oit.IntersectionLite(s.copy()), 120, 0.9, np_random=np_random(0))
    c = c_oracle.il_opd_plan(s.pack(), 120, 0.9)
    assert_c_tree_equals(c, t)
    if name == "arrival":                      # arrivals (reward 1), or arrivals that crash (reward 0), end the tree
        assert c["done"].any() and (c["reward"] == 1.0).any() == (i == 0)


@pytest.mark.parametrize("name,i", PLANNER_ROOTS[:4])
@pytest.mark.parametrize("width", [4, 16])
def test_c_wavefront_opd_equals_the_python_specification(name, i, width):
    s = root_state(name, i)
    _, t = planners.opd_plan_wavefront(oit.IntersectionLite(s.copy()), 150, 0.9, width, np_random=np_random(0))
    c = c_oracle.il_opd_plan_wave(s.pack(), 150, 0.9, width)
    assert_c_tree_equals(c, t)
    assert c["n_waves"] == len(t.waves)
    ends = np.cumsum([sum(t.n_children[leaf] for leaf in wave) for wave in t.waves]) + 1
    assert c["wave_end"].tolist() == ends.tolist()


def test_c_opd_keeps_the_highway_capacity():
    """The env descriptor's action count sets the capacity: 1 + (budget // 3) * 3 nodes here, 5 on highway."""
    c = c_oracle.il_opd_plan(root_state("phases", 0).pack(), 31, 0.9)
    assert (c["n_children"] > 0).sum() == 10 and len(c["parent"]) <= 31
