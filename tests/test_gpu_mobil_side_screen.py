"""hw::step's per-side MOBIL own-gain screen (own_gain_shut) against the oracle, on scenes at the edges of the screen.

A decider's side is served only when the side lane exists and the screen cannot prove that the own term fails the gain
test.  The scenes put deciders where that proof changes its answer:
- a side front at the last and first fp32 positions where the screen shuts the side (the sign of fma(k, D, -|gap|)
  flips), and at the last and first positions where the side's gain test flips (the screen must leave both served);
- a side front so much faster than the decider that its gap (D0 + v TAU + v (v - vf) / 2 sqrt(ab)) is negative;
- deciders on lanes 0 and 3, with a front on their only side lane;
- five deciders in one group with both sides served: ten pairs, so the server takes a second pass;
- a decider whose free-road term overflows to -inf (target speed 0 at 5e7 m/s), so self_a = -inf and the gain
  a_free - self_a is NaN: the screen must not shut its sides.
Each scene is stepped through the batched step, the per-group step and both OPD kernels (one tree per CTA, batch) and
compared bit for bit with the numpy and C oracles."""
import numpy as np
import pytest

from oracle import c_oracle
from oracle import envs as oenvs
from tests import highway_scenes as hs
from tests.test_gpu_step_gating import first_step_record, trajectory

f32 = np.float32
I = oenvs.A_IDLE
N_DECISIONS = 4
K_SHUT = f32(float.fromhex("0x1.55aaaap-2"))


def _base():
    s = hs.blank()
    hs.put(s, 0, -200.0, 12.0, 25.0, timer=0.0)
    return s


def _boundary_scene(x_side):
    """slot 1 decides on lane 1 (x 200, v = ts = 25) 40 m behind slot 2 (same speed); slot 3 is the front of its left
    lane at x_side; the right lane is blocked by slot 4 close ahead and slower"""
    s = _base()
    hs.put(s, 1, 200.0, 4.0, 25.0, timer=1.05)
    hs.put(s, 2, 240.0, 4.0, 25.0, timer=0.0)
    hs.put(s, 3, x_side, 0.0, 25.0, timer=0.0)
    hs.put(s, 4, 215.0, 8.0, 20.0, timer=0.0)
    return s


def _left_side(x_side):
    """(shut by the screen, goes left) for slot 1 of _boundary_scene(x_side), in fp32 as the step computes them
    (the screen's k from numpy's square root; the device's approximate one may move its edge by an ulp of k)"""
    s = _boundary_scene(x_side)
    v, ts, x = s.v[[1]], s.tgt_speed[[1]], s.x[[1]]
    a_free = oenvs._idm(v, ts, np.array([False]), x, x, v)[0]
    self_a = oenvs._idm(v, ts, np.array([True]), x, s.x[[2]], s.v[[2]])[0]
    pred = oenvs._idm(v, ts, np.array([True]), x, s.x[[3]], s.v[[3]])[0]
    k = np.sqrt(f32(f32(f32(a_free - self_a) - oenvs.MOBIL_MIN_GAIN) * K_SHUT))
    assert (k >= f32(2.0 ** -8)) and f32(f32(a_free - f32(oenvs.COMFORT_ACC_MAX * f32(k * k))) - self_a) < 0.2
    g = abs(f32(f32(oenvs.D0 + f32(v[0] * oenvs.TAU)) + f32(f32(v[0] * f32(v[0] - s.v[3])) / oenvs.TWO_SQRT_AB)))
    dist = max(abs(f32(s.x[3] - x[0])), oenvs.EPS)
    shut = float(k) * float(dist) - float(g) < 0.0
    return shut, not (f32(pred - self_a) < oenvs.MOBIL_MIN_GAIN)


def _edge(pred, lo, hi):
    """the largest fp32 x in [lo, hi) with pred(x) true, pred monotone (true below the edge)"""
    lo, hi = f32(lo), f32(hi)
    assert pred(lo) and not pred(hi)
    while hs.ulp_step(lo, 1) < hi:
        mid = f32((float(lo) + float(hi)) / 2.0)
        if mid <= lo or mid >= hi:
            mid = hs.ulp_step(lo, 1)
        if pred(mid):
            lo = mid
        else:
            hi = mid
    return lo


SHUT_EDGE = _edge(lambda x: _left_side(x)[0], 230.0, 250.0)
GO_EDGE = _edge(lambda x: not _left_side(x)[1], 230.0, 250.0)


def side_front_at(x_side):
    def scene():
        return _boundary_scene(x_side), [I] * N_DECISIONS
    return scene


def negative_gap():
    """slot 1 decides behind a close front on lane 2; its left front runs 20 m/s faster (gap < 0), its right one
    slower and close"""
    s = _base()
    hs.put(s, 1, 200.0, 8.0, 25.0, timer=1.05)
    hs.put(s, 2, 225.0, 8.0, 25.0, timer=0.0)
    hs.put(s, 3, 210.0, 4.0, 45.0, ts=45.0, timer=0.0)
    hs.put(s, 4, 212.0, 12.0, 20.0, timer=0.0)
    return s, [I] * N_DECISIONS


def outer_deciders():
    """deciders on lane 0 and lane 3 behind slower fronts, each with a front on its only side lane: one closer
    (shut), one far ahead (served)"""
    s = _base()
    hs.put(s, 1, 200.0, 0.0, 25.0, timer=1.05)
    hs.put(s, 2, 230.0, 0.0, 20.0, timer=0.0)
    hs.put(s, 3, 215.0, 4.0, 20.0, timer=0.0)
    hs.put(s, 4, 400.0, 12.0, 25.0, timer=1.02)
    hs.put(s, 5, 430.0, 12.0, 20.0, timer=0.0)
    hs.put(s, 6, 600.0, 8.0, 25.0, timer=0.0)
    return s, [I] * N_DECISIONS


def ten_pairs():
    """five deciders on lane 1, 50 m apart at one speed, with both side lanes empty ahead: ten served pairs"""
    s = _base()
    for j in range(5):
        hs.put(s, 1 + j, 100.0 + 50.0 * j, 4.0, 25.0, timer=1.01 + 0.01 * j)
    hs.put(s, 6, 350.0, 4.0, 25.0, timer=0.0)
    return s, [I] * N_DECISIONS


def infinite_self_a():
    """slot 1 at 5e7 m/s with target speed 0: a_free = self_a = -inf; fronts on its own lane and both side lanes"""
    s = _base()
    hs.put(s, 1, 200.0, 4.0, 5e7, ts=0.0, timer=1.05)
    hs.put(s, 2, 300.0, 4.0, 5e7, ts=5e7, timer=0.0)
    hs.put(s, 3, 250.0, 0.0, 25.0, timer=0.0)
    hs.put(s, 4, 260.0, 8.0, 25.0, timer=0.0)
    return s, [I] * N_DECISIONS


SCENES = {"shut_edge_in": side_front_at(SHUT_EDGE), "shut_edge_out": side_front_at(hs.ulp_step(SHUT_EDGE, 1)),
          "go_edge_stay": side_front_at(GO_EDGE), "go_edge_go": side_front_at(hs.ulp_step(GO_EDGE, 1)),
          "negative_gap": negative_gap, "outer_deciders": outer_deciders, "ten_pairs": ten_pairs,
          "infinite_self_a": infinite_self_a}


def all_scenes():
    return [(name, *make()) for name, make in SCENES.items()]


def test_scenes_reach_the_screen_edges():
    """On the oracle: each scene reaches the case its name promises (at the first sub-step)."""
    assert SHUT_EDGE < GO_EDGE
    assert _left_side(SHUT_EDGE) == (True, False) and _left_side(hs.ulp_step(SHUT_EDGE, 1)) == (False, False)
    assert _left_side(GO_EDGE) == (False, False) and _left_side(hs.ulp_step(GO_EDGE, 1)) == (False, True)
    with np.errstate(all="ignore"):
        rec = {name: first_step_record(*make()[:1], I)[0] for name, make in SCENES.items()}
    assert rec["go_edge_stay"]["new_tgt"][1] == 1 and rec["go_edge_go"]["new_tgt"][1] == 0
    s = negative_gap()[0]
    assert f32(oenvs.D0 + s.v[1] * oenvs.TAU) + f32(s.v[1] * (s.v[1] - s.v[3])) / oenvs.TWO_SQRT_AB < 0
    assert rec["negative_gap"]["decide"][1]
    r = rec["outer_deciders"]
    assert r["decide"][1] and r["decide"][4] and r["new_tgt"][1] == 0 and r["new_tgt"][4] == 2
    r = rec["ten_pairs"]
    assert r["decide"][1:6].all() and (r["new_tgt"][1:6] != 1).all()
    s = infinite_self_a()[0]
    with np.errstate(all="ignore"):
        a_free = oenvs._idm(s.v[[1]], s.tgt_speed[[1]], np.array([False]), s.x[[1]], s.x[[1]], s.v[[1]])[0]
        self_a = oenvs._idm(s.v[[1]], s.tgt_speed[[1]], np.array([True]), s.x[[1]], s.x[[2]], s.v[[2]])[0]
        assert a_free == -np.inf and self_a == -np.inf and np.isnan(a_free - self_a)
    assert rec["infinite_self_a"]["decide"][1]


def _runs():
    scenes = all_scenes()
    with np.errstate(all="ignore"):
        return scenes, [trajectory(s, acts) for _, s, acts in scenes]


@pytest.mark.gpu
def test_full_warp_step_on_screen_edges():
    import torch
    from rl_agents_b200 import _lib
    lib = _lib.load()
    scenes, runs = _runs()
    n = len(runs)
    st = torch.tensor(np.stack([r[1][0] for r in runs]), dtype=torch.int32, device="cuda")
    rew = torch.empty(n, dtype=torch.float32, device="cuda")
    flg = torch.empty(n, dtype=torch.int32, device="cuda")
    avail = torch.empty(n, dtype=torch.int32, device="cuda")
    for k in range(N_DECISIONS):
        act = torch.tensor([r[0][k] for r in runs], dtype=torch.int32, device="cuda")
        _lib.check(lib.b2_highway_step(_lib.ptr(st), _lib.ptr(act), _lib.ptr(rew), _lib.ptr(flg), _lib.ptr(avail), n,
                                       _lib.current_stream()))
        got, r_got, f_got, a_got = st.cpu().numpy(), rew.cpu().numpy(), flg.cpu().numpy(), avail.cpu().numpy()
        for i, (acts, words, rews, flags, av) in enumerate(runs):
            name = scenes[i][0]
            assert np.array_equal(got[i], words[k + 1]), (name, k, np.nonzero(got[i] != words[k + 1])[0])
            assert r_got[i].view(np.int32) == rews[k].view(np.int32), (name, k)
            assert f_got[i] == flags[k] and a_got[i] == av[k], (name, k)


@pytest.mark.gpu
def test_half_warp_step_on_screen_edges():
    """Per-group mode: the two scenes of a warp take different numbers of decisions."""
    import torch
    from rl_agents_b200 import _lib
    lib = _lib.load()
    scenes, runs = _runs()
    n, m = len(runs), N_DECISIONS
    n_steps = np.array([m if i % 2 == 0 else 1 + (i // 2) % (m - 1) for i in range(n)], np.int32)
    roots = torch.tensor(np.stack([r[1][0] for r in runs]), dtype=torch.int32, device="cuda")
    acts = torch.tensor(np.stack([r[0] for r in runs]), dtype=torch.int32, device="cuda")
    trace = torch.full((n, m, 136), -1, dtype=torch.int32, device="cuda")
    rew = torch.zeros((n, m), dtype=torch.float32, device="cuda")
    flg = torch.full((n, m), -1, dtype=torch.int32, device="cuda")
    _lib.check(lib.b2_selftest_highway_step_groups(_lib.ptr(roots), _lib.ptr(acts),
                                                   _lib.ptr(torch.from_numpy(n_steps).cuda()), _lib.ptr(trace),
                                                   _lib.ptr(rew), _lib.ptr(flg), n, m, _lib.current_stream()))
    trace, rew, flg = trace.cpu().numpy(), rew.cpu().numpy(), flg.cpu().numpy()
    for i, (_, words, rews, flags, av) in enumerate(runs):
        name = scenes[i][0]
        for k in range(n_steps[i]):
            assert np.array_equal(trace[i, k], words[k + 1]), (name, k, np.nonzero(trace[i, k] != words[k + 1])[0])
            assert rew[i, k].view(np.int32) == rews[k].view(np.int32), (name, k)
            assert flg[i, k] == flags[k] | (av[k] << 2), (name, k)


@pytest.mark.gpu
@pytest.mark.parametrize("n_trees", [8, 24])
def test_opd_kernels_on_screen_edges(n_trees):
    """8 trees: one tree per CTA (opd_highway_kernel); 24 trees: the batch kernel.  The scenes repeat to fill them."""
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDEngine
    from tests.test_gpu_highway_step_paths import assert_opd_tree, np_random
    words = [s.pack() for _, s, _ in all_scenes()]
    words = (words * 3)[:n_trees]
    eng = OPDEngine(_lib.ENV_HIGHWAY, len(words), 5, 200, 0.8)
    eng.plan(torch.tensor(np.stack(words), dtype=torch.int32, device="cuda"))
    _, res = eng.finish([np_random(0) for _ in words])
    for i, w in enumerate(words):
        assert_opd_tree(eng.tree_dict(i), c_oracle.opd_plan(w, 200, 0.8), res[i])
