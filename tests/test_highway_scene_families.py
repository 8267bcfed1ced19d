"""The HighwayLite scene families (tests/highway_scenes.py) on the CPU: each reaches the step paths it is built for
(census floors), and the C statement of the spec equals the numpy statement on every family, bit for bit -- so the
C oracle can stand in for the numpy one where the GPU tests need speed."""
import numpy as np
import pytest

from oracle import c_oracle
from oracle import envs as oenvs
from tests import highway_scenes as hs

# per family: the paths it exists for, and how often its trajectories (8 decisions per scene) must reach each
FLOORS = {
    "adapter": {"absent_ranked": 500, "deciders_gt8": 10, "far_collision": 3, "abort": 2, "recount": 20},
    "sync_timers": {"deciders_gt4": 40, "deciders_gt8": 40, "deciders_gt12": 40, "recount": 20},
    "absent": {"absent_ranked": 800, "far_collision": 5, "recount": 10},
    "entry_ties": {"entry_tie": 12, "scan_to_ranked": 12, "far_collision": 20, "recount": 40},
    "late_ties": {"late_tie": 8, "scan_to_ranked": 8, "absent_ranked": 400, "recount": 20},
    "jam": {"far_collision": 1000, "abort": 5, "ego_crash": 5, "recount": 100},
    "kinematic": {"clamp": 30, "wrap": 100, "abort": 5, "recount": 40},
}


def test_every_family_has_a_floor():
    assert set(FLOORS) == set(hs.FAMILY_NAMES)
    assert all(set(f) <= set(hs.PATHS) for f in FLOORS.values())


@pytest.mark.parametrize("name", hs.FAMILY_NAMES)
def test_family_reaches_its_paths(name):
    counts = hs.census(name)
    print(name, dict(counts))
    for path, floor in FLOORS[name].items():
        assert counts[path] >= floor, (name, path, counts[path], floor)


@pytest.mark.parametrize("name", hs.FAMILY_NAMES)
def test_family_scenes_stay_in_the_state_domain(name):
    for s in hs.family(name):
        w = s.pack()
        f = w[:96].view(np.float32)
        assert s.flags[0] & 1 and np.isfinite(f).all() and (w[130:] == 0).all()
        assert ((s.tgt_lane >= 0) & (s.tgt_lane <= 3)).all() and ((s.flags >= 0) & (s.flags <= 3)).all()
        assert (np.abs(s.v) <= 46).all() and (np.abs(s.x) < 1000).all() and 0 <= s.speed_index <= 2


def test_late_ties_appear_after_the_first_substep():
    """The tie of each late-tie scene is absent at entry and exact at its sub-step."""
    for s in hs.family("late_ties"):
        p = (s.flags & 1) != 0
        assert np.unique(s.x[p]).size == p.sum()
        xs = []
        oenvs.highway_step(s.copy(), oenvs.A_IDLE, on_substep=lambda sub, x, present, **_: xs.append(x.copy()))
        assert any(np.unique(x[p]).size < p.sum() for x in xs[1:])


def test_observer_leaves_the_step_unchanged():
    for name in ("jam", "kinematic"):
        for s in hs.family(name)[:4]:
            a, b = s.copy(), s.copy()
            ra = oenvs.highway_step(a, oenvs.A_LEFT)
            rb = oenvs.highway_step(b, oenvs.A_LEFT, on_substep=lambda **kw: None)
            assert ra == rb and np.array_equal(a.pack(), b.pack())


@pytest.mark.parametrize("name", hs.FAMILY_NAMES)
def test_c_oracle_equals_numpy_oracle(name):
    runs = hs.family_trajectories(name)
    assert len(runs[0][0]) >= 8
    w = np.stack([r[1][0] for r in runs])
    for k in range(len(runs[0][0])):
        w, rew, flg = c_oracle.step_batch(w, [r[0][k] for r in runs])
        for i, r in enumerate(runs):
            assert np.array_equal(w[i], r[1][k + 1]), (name, i, k)
            assert rew[i] == r[2][k] and flg[i] == r[3][k], (name, i, k)
