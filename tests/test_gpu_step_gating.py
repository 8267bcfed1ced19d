"""hw::step's gated blocks against the oracle on scenes built to sit on the edges of their gates.

The lane-change block (lane-entering masks, abort rule, front on the target lane, IDM behind it) runs only while an IDM
vehicle changes lanes, and the MOBIL server only for deciders that could move (|v| >= 1 and a_free - self_a >= 0.2).
The scenes below put the work those gates skip next to work they must not skip: an IDM vehicle that aborts because
the ego enters its target lane ahead of it, crashed vehicles changing lanes (one of them the only vehicle between
lanes), a vehicle that crashes while changing lanes, deciders whose gain a_free - self_a is the largest fp32 value
below 0.2 and 0.20000008 (the nearest above that the front positions tried gave; none gave exactly 0.2), deciders on
the outer lanes, deciders slower than 1 m/s and at exactly 1 m/s.  Each scene is
also run with an exact x tie added, which sends every sub-step to the scan path.  Every comparison is exact: the
batched step (two scenes per warp), the per-group step and the OPD batch kernel against the numpy and C oracles."""
import numpy as np
import pytest

from oracle import c_oracle
from oracle import envs as oenvs
from tests import highway_scenes as hs

f32 = np.float32
L, I, R = oenvs.A_LEFT, oenvs.A_IDLE, oenvs.A_RIGHT
N_DECISIONS = 4

# front positions that put a decider at x = 200, v = ts = 25 (a_free = 0) on either side of a gain of 0.2 behind a
# front at the same speed: fl(a_free - self_a) = 0.19999999 and 0.20000008
FRONT_BELOW, FRONT_ABOVE = f32(383.9667), f32(383.96667)


def _base():
    s = hs.blank()
    hs.put(s, 0, -200.0, 0.0, 25.0, timer=0.0)
    hs.put(s, 5, -120.0, 8.0, 22.0, ts=24.0, timer=0.1)
    hs.put(s, 6, 600.0, 12.0, 24.0, ts=24.0, timer=0.2)
    return s


def ego_enters_ahead():
    """slot 1 moves 1 -> 2; the ego, 10 m ahead, moves 3 -> 2 (LEFT): slot 1 aborts, the ego is the only other changer"""
    s = _base()
    hs.put(s, 0, 110.0, 12.0, 25.0, timer=0.0)
    hs.put(s, 1, 100.0, 4.0, 25.0, timer=0.2, tgt=2)
    return s, [L, I, R, I]


def crashed_enters_ahead():
    """slot 1 moves 3 -> 2; crashed slot 2, 10 m ahead, is moving 1 -> 2: slot 1 aborts"""
    s = _base()
    hs.put(s, 1, 100.0, 12.0, 25.0, timer=0.2, tgt=2)
    hs.put(s, 2, 110.0, 4.0, 3.0, timer=0.2, tgt=2, crashed=True)
    return s, [I, R, I, I]


def crashed_only_changer():
    """crashed slot 2 is the only vehicle whose lane differs from its target"""
    s = _base()
    hs.put(s, 1, 20.0, 0.0, 24.0, timer=0.3)
    hs.put(s, 2, 60.0, 4.0, 8.0, timer=0.4, tgt=2, crashed=True)
    hs.put(s, 3, 30.0, 8.0, 23.0, timer=0.5)
    return s, [I, I, I, I]


def crash_while_changing():
    """slot 1 moves 1 -> 2 and overlaps slot 2 at the start: it crashes after the first sub-step"""
    s = _base()
    hs.put(s, 1, 100.0, 4.0, 25.0, timer=0.2, tgt=2)
    hs.put(s, 2, 103.0, 5.5, 24.0, timer=0.2, tgt=1)
    return s, [I, I, I, I]


def decider(front_x):
    """slot 1 decides at the first sub-step (lane 1, x 200) behind slot 2; both side lanes are empty ahead"""
    def scene():
        s = _base()
        hs.put(s, 0, 0.0, 12.0, 25.0, timer=0.0)
        hs.put(s, 1, 200.0, 4.0, 25.0, timer=1.05)
        hs.put(s, 2, front_x, 4.0, 25.0, timer=0.0)
        return s, [I, I, I, I]
    return scene


def outer_deciders():
    """deciders on lane 0 and lane 3 close behind a slower front: each can only go inwards"""
    s = _base()
    hs.put(s, 1, 200.0, 0.0, 25.0, timer=1.05)
    hs.put(s, 2, 230.0, 0.0, 18.0, timer=0.0)
    hs.put(s, 3, 300.0, 12.0, 25.0, timer=1.02)
    hs.put(s, 4, 330.0, 12.0, 18.0, timer=0.0)
    return s, [I, I, I, I]


def slow_deciders():
    """deciders at |v| = 0.5 (never moves), v = -0.5 and v = 1.0 (may move) close behind a stopped front"""
    s = _base()
    hs.put(s, 1, 200.0, 4.0, 0.5, ts=25.0, timer=1.05)
    hs.put(s, 2, 212.0, 4.0, 0.0, timer=0.0)
    hs.put(s, 3, 300.0, 8.0, -0.5, ts=25.0, timer=1.05)
    hs.put(s, 4, 312.0, 8.0, 0.0, timer=0.0)
    hs.put(s, 7, 400.0, 4.0, 1.0, ts=25.0, timer=1.05)
    hs.put(s, 8, 412.0, 4.0, 0.0, timer=0.0)
    return s, [I, I, I, I]


SCENES = {"ego_enters_ahead": ego_enters_ahead, "crashed_enters_ahead": crashed_enters_ahead,
          "crashed_only_changer": crashed_only_changer, "crash_while_changing": crash_while_changing,
          "decider_below": decider(FRONT_BELOW), "decider_above": decider(FRONT_ABOVE),
          "outer_deciders": outer_deciders, "slow_deciders": slow_deciders}


def with_tie(s):
    """two vehicles at exactly the same x on lanes 0 and 3, far ahead, at their target speed: tied for the whole step"""
    s = s.copy()
    hs.put(s, 14, 900.0, 0.0, 25.0, timer=0.0)
    hs.put(s, 15, 900.0, 12.0, 25.0, timer=0.0)
    return s


def all_scenes():
    out = []
    for name, make in SCENES.items():
        s, acts = make()
        out.append((name, s, acts))
        out.append((name + "+tie", with_tie(s), acts))
    return out


def first_step_record(s, action):
    subs = []
    oenvs.highway_step(s.copy(), action, on_substep=lambda **kw: subs.append({k: np.array(v) for k, v in kw.items()}))
    return subs


def trajectory(s, acts):
    """(actions, words [n + 1, 136], rewards, flags, avail) of the oracle, actions falling back to IDLE when not
    available"""
    s = s.copy()
    out_a, words, rews, flags, avail = [], [s.pack()], [], [], []
    for a in acts:
        a = a if a in oenvs.highway_available_actions(s) else I
        r, term, trunc = oenvs.highway_step(s, a)
        out_a.append(a)
        words.append(s.pack())
        rews.append(f32(r))
        flags.append((1 if term else 0) | (2 if trunc else 0))
        avail.append(hs.avail_mask(s))
    return (np.array(out_a, np.int32), np.stack(words), np.array(rews, np.float32), np.array(flags, np.int32),
            np.array(avail, np.int32))


def test_scenes_reach_the_gate_edges():
    """On the oracle: each scene reaches the case its name promises (at the first sub-step)."""
    rec = {}
    for name, make in SCENES.items():
        s, acts = make()
        rec[name] = first_step_record(s, acts[0])
    r = rec["ego_enters_ahead"][0]
    assert r["abort"][1] and set(np.nonzero(r["present"] & (r["cur"] != r["tgt"]))[0]) == {0, 1}
    r = rec["crashed_enters_ahead"][0]
    assert r["abort"][1] and r["crashed"][2] and r["cur"][2] != r["tgt"][2]
    r = rec["crashed_only_changer"][0]
    assert np.nonzero(r["present"] & (r["cur"] != r["tgt"]))[0].tolist() == [2] and r["crashed"][2]
    r = rec["crash_while_changing"]
    assert not r[0]["crashed"][1] and r[1]["crashed"][1] and r[1]["cur"][1] != r[1]["tgt"][1]

    def gain(name, i):
        s = SCENES[name]()[0]
        v, ts, x = s.v[[i]], s.tgt_speed[[i]], s.x[[i]]
        a_free = oenvs._idm(v, ts, np.array([False]), x, x, v)[0]
        self_a = oenvs._idm(v, ts, np.array([True]), x, s.x[[2]], s.v[[2]])[0]
        return f32(a_free - self_a)
    g = oenvs.MOBIL_MIN_GAIN
    assert gain("decider_below", 1) == np.nextafter(g, f32(0)) and gain("decider_above", 1) > g
    for name, moves in (("decider_below", False), ("decider_above", True)):
        r = rec[name][0]
        assert r["decide"][1] and (r["new_tgt"][1] != r["cur"][1]) == moves, name
    r = rec["outer_deciders"][0]
    assert r["decide"][1] and r["decide"][3] and r["new_tgt"][1] == 1 and r["new_tgt"][3] == 2
    r = rec["slow_deciders"][0]
    assert r["decide"][[1, 3, 7]].all() and r["new_tgt"][1] == 1 and r["new_tgt"][7] != 1
    for name, s, _ in all_scenes():
        x = s.x[s.flags & 1 != 0]
        assert (np.unique(x).size < x.size) == name.endswith("+tie"), name


@pytest.mark.gpu
def test_full_warp_step_on_gate_edges():
    import torch
    from rl_agents_b200 import _lib
    lib = _lib.load()
    scenes = all_scenes()
    runs = [trajectory(s, acts) for _, s, acts in scenes]
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
def test_half_warp_step_on_gate_edges():
    """Per-group mode: the two scenes of a warp take different numbers of decisions."""
    import torch
    from rl_agents_b200 import _lib
    lib = _lib.load()
    scenes = all_scenes()
    runs = [trajectory(s, acts) for _, s, acts in scenes]
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
        assert (trace[i, n_steps[i]:] == -1).all() and (flg[i, n_steps[i]:] == -1).all()


@pytest.mark.gpu
def test_opd_batch_kernel_on_gate_edges():
    """24 trees (the batch kernel): every scene, with and without the tie, then the tie-free ones again."""
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDEngine
    from tests.test_gpu_highway_step_paths import assert_opd_tree, np_random
    scenes = all_scenes()
    words = [s.pack() for _, s, _ in scenes]
    words = (words + [w for (name, _, _), w in zip(scenes, words) if not name.endswith("+tie")])[:24]
    assert len(words) == 24
    eng = OPDEngine(_lib.ENV_HIGHWAY, len(words), 5, 200, 0.8)
    eng.plan(torch.tensor(np.stack(words), dtype=torch.int32, device="cuda"))
    _, res = eng.finish([np_random(0) for _ in words])
    for i, w in enumerate(words):
        assert_opd_tree(eng.tree_dict(i), c_oracle.opd_plan(w, 200, 0.8), res[i])
