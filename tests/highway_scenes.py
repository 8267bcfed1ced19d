"""Deterministic HighwayLite scene families for the step-path tests, and a census of the kernel paths a trajectory
reaches.

The generator of `oracle.envs.make_highway_state` makes one kind of scene only (16 present vehicles 40-80 m apart,
headings 0, speeds 21-24 m/s, random timers).  `hw::step` has paths such scenes never take: more than 8 MOBIL
deciders in one sub-step, absent slots, exact x ties (entry and later), collisions between vehicles that are not
x-neighbours, the abort rule, the speed clamp and the heading wrap.  Each family below is built to reach some of them,
and `census` counts, on the numpy oracle, how often a trajectory does -- so that a GPU test that passes is known to
have exercised the path.

Every scene stays inside the state domain of docs/HIGHWAY_LITE_SPEC.md: slot 0 present, lanes 0..3 as targets,
finite words, speeds and distances of moderate magnitude.
"""
import functools
from collections import Counter

import numpy as np

from oracle import envs as oenvs

f32 = np.float32
V = oenvs.V_SLOTS
N_DECISIONS = 8

PATHS = ("entry_tie", "late_tie", "scan_to_ranked", "recount", "deciders_gt4", "deciders_gt8", "deciders_gt12", "absent_ranked",
         "far_collision", "ego_crash", "abort", "clamp", "wrap")


# ------------------------------------------------------------------------------------------------ scene helpers ----
def blank(t=0, si=1):
    s = oenvs.HighwayLiteState()
    for k in ("x", "y", "h", "v", "tgt_speed", "timer"):
        setattr(s, k, np.zeros(V, f32))
    s.tgt_lane = np.zeros(V, np.int32)
    s.flags = np.zeros(V, np.int32)
    s.t, s.speed_index = int(t), int(si)
    return s


def put(s, slot, x, y, v, ts=None, h=0.0, timer=0.5, tgt=None, crashed=False):
    s.x[slot], s.y[slot], s.h[slot], s.v[slot] = f32(x), f32(y), f32(h), f32(v)
    s.tgt_speed[slot] = f32(v if ts is None else ts)
    s.timer[slot] = f32(timer)
    s.tgt_lane[slot] = int(np.clip(np.rint(y / 4.0), 0, 3)) if tgt is None else int(tgt)
    s.flags[slot] = 1 | (2 if crashed else 0)


def ulp_step(x, n):
    """x moved by n units in the last place (positive finite x)"""
    return np.array([np.float32(x).view(np.int32) + n], np.int32).view(np.float32)[0]


# ------------------------------------------------------------------------------------------------------ families ----
class _Obj(object):
    pass


def _fake_highway_env(n_others, timer, seed, steps=3):
    """An object with the attribute names of upstream highway-env's HighwayEnv, as the live-env adapter reads them."""
    rng = np.random.default_rng(seed)
    env, road = _Obj(), _Obj()
    env.unwrapped = env
    ego = _Obj()
    ego_lane = int(rng.integers(0, 4))
    ego_x = float(rng.uniform(50.0, 300.0))
    ego.position = np.array([ego_x, 4.0 * ego_lane + rng.uniform(-0.4, 0.4)])
    ego.heading, ego.speed, ego.crashed = float(rng.uniform(-0.05, 0.05)), float(rng.uniform(20.0, 30.0)), False
    ego.lane_index = ("0", "1", ego_lane)
    ego.target_lane_index = ("0", "1", int(np.clip(ego_lane + rng.integers(-1, 2), 0, 3)))
    ego.target_speeds = np.array([20.0, 25.0, 30.0])
    ego.speed_index = int(rng.integers(0, 3))
    ego.target_speed = 20.0 + 5.0 * ego.speed_index
    vehicles = [ego]
    ahead = behind = ego_x
    for k in range(n_others):
        v = _Obj()
        lane = int(rng.integers(0, 4))
        if k % 2 == 0:
            ahead += rng.uniform(6.0, 30.0)
            x = ahead
        else:
            behind -= rng.uniform(6.0, 30.0)
            x = behind
        tgt = lane
        if rng.uniform() < 0.3:            # a lane change in progress
            tgt = int(np.clip(lane + (1 if rng.uniform() < 0.5 else -1), 0, 3))
        y = 4.0 * lane + (tgt - lane) * rng.uniform(0.0, 1.8)
        v.position = np.array([x, y])
        v.heading = float(rng.uniform(-0.08, 0.08)) if tgt != lane or rng.uniform() < 0.3 else 0.0
        v.speed = float(rng.uniform(15.0, 31.0))
        v.crashed = bool(rng.uniform() < 0.15)
        v.lane_index, v.target_lane_index = ("0", "1", lane), ("0", "1", tgt)
        v.target_speed, v.timer = float(rng.uniform(20.0, 30.0)), timer
        vehicles.append(v)
    road.vehicles = vehicles[1:3] + [ego] + vehicles[3:]
    env.road, env.vehicle = road, ego
    env.config = {"lanes_count": 4, "duration": 40, "policy_frequency": 1, "action": {"type": "DiscreteMetaAction"}}
    env.steps = steps
    return env


def adapter_scenes():
    """Scenes packed by the live-env adapter: 1, 4, 7 and 15 other vehicles (trailing slots absent, words zero), equal
    timers, crashed vehicles, lane changes in progress, non-zero headings."""
    from rl_agents_b200.envs.highway_adapter import scene_from_highway_env
    out = []
    for i, (n, timer) in enumerate((n, tm) for n in (1, 4, 7, 15) for tm in (0.0, 0.25, 0.999)):
        words = scene_from_highway_env(_fake_highway_env(n, timer, seed=700 + i, steps=36 if i == 5 else 3))
        out.append(oenvs.HighwayLiteState.unpack(words))
    return out


def sync_timers_scenes():
    """Generator scenes with every timer equal: 9-15 vehicles decide in the same sub-step (the MOBIL pass serves 4)."""
    out = []
    for k in range(12):
        s = oenvs.make_highway_state(2000 + k)
        s.timer[:] = f32((0.25, 0.5, 0.9, 0.0)[k % 4])
        out.append(s)
    return out


def absent_scenes():
    """1-15 present vehicles, absent slots in the middle and at the end, with stale words: x next to or equal to a
    present vehicle's (the front-most one's included), stale speeds, timers, targets and crash bits."""
    out = []
    for k, n_present in enumerate((1, 2, 3, 5, 7, 8, 9, 11, 13, 14, 15, 6)):
        rng = np.random.default_rng(3000 + k)
        s = oenvs.make_highway_state(3000 + k)
        present = np.zeros(V, bool)
        present[0] = True
        present[1 + rng.permutation(V - 1)[:n_present - 1]] = True
        if k % 3 == 0 and n_present < V - 1 and present[V - 1]:      # the last slot absent too
            present[V - 1] = False
            present[1 + np.nonzero(~present[1:V - 1])[0][0]] = True
        pres = np.nonzero(present)[0]
        front = pres[np.argmax(s.x[pres])]
        for j, a in enumerate(np.nonzero(~present)[0]):
            p = front if j == 0 else pres[rng.integers(len(pres))]
            s.x[a] = s.x[p] if j % 2 == 1 else f32(s.x[p] + rng.uniform(-4.0, 4.0))
            s.y[a] = f32(s.y[p] + rng.uniform(-1.0, 1.0))
            s.v[a] = f32(rng.uniform(-5.0, 35.0))
            s.tgt_speed[a] = f32(rng.uniform(0.0, 30.0))
            s.timer[a] = f32(rng.uniform(0.0, 3.0))
            s.h[a] = f32(rng.uniform(-0.2, 0.2))
            s.tgt_lane[a] = int(rng.integers(0, 4))
            s.flags[a] = 2 if j % 3 == 2 else 0
        out.append(s)
    return out


def _tie_follower_scene(X, lane, hi_slot, lo_slot, zero=False, seed=0):
    """Two vehicles at the same x: `hi` stopped and crashed between two lanes (on both), `lo` on the lane centre, and a
    follower on that lane whose front is the pair -- the spec gives it the larger slot, so the tie decides its IDM."""
    rng = np.random.default_rng(seed)
    s = blank()
    put(s, 0, X - 60.0, 4.0 * 3, 25.0, timer=0.0)
    put(s, hi_slot, X, 4.0 * lane + 2.0, 0.0, crashed=True)
    put(s, lo_slot, X, 4.0 * lane, 22.0, timer=0.0)
    if zero:
        s.x[hi_slot], s.x[lo_slot] = (f32(-0.0), f32(0.0)) if seed % 2 else (f32(0.0), f32(-0.0))
    follower = [k for k in range(1, V) if k not in (hi_slot, lo_slot)][0]
    # slow and 30 m back, so that its IDM term is not clipped and differs for the two fronts (stopped / 22 m/s)
    put(s, follower, float(s.x[lo_slot]) - 30.0, 4.0 * lane, 10.0, timer=0.0)
    slot = follower + 1
    for x in np.sort(rng.uniform(-80.0, 80.0, size=4)) + float(s.x[lo_slot]):
        while slot in (hi_slot, lo_slot):
            slot += 1
        put(s, slot, x, 4.0 * 3 - 4.0 * (slot % 2), float(rng.uniform(20.0, 26.0)), timer=float(rng.uniform(0, 1)))
        slot += 1
    return s


def entry_ties_scenes():
    """Exact x ties at entry: two- and three-way, on one lane and on different lanes, the ego included, a -0.0 / +0.0
    pair, and ties a follower's IDM depends on."""
    out = []
    for k in range(8):
        s = oenvs.make_highway_state(4000 + k)
        if k % 4 == 0:
            s.x[5] = s.x[3]                                 # two-way, usually different lanes
        elif k % 4 == 1:
            s.x[6], s.y[6] = s.x[2], s.y[2]                 # two-way on one lane: overlapping boxes
        elif k % 4 == 2:
            s.x[4] = s.x[7] = s.x[9]                        # three-way
        else:
            s.x[2] = s.x[11] = s.x[0]                       # three-way with the ego
            s.y[11] = s.y[0] + f32(1.0)
        out.append(s)
    out.append(_tie_follower_scene(0.0, 1, hi_slot=5, lo_slot=2, zero=True, seed=1))
    out.append(_tie_follower_scene(0.0, 0, hi_slot=7, lo_slot=3, zero=True, seed=2))
    out.append(_tie_follower_scene(123.25, 2, hi_slot=9, lo_slot=4, seed=3))
    out.append(_tie_follower_scene(-40.5, 1, hi_slot=2, lo_slot=6, seed=4))
    return out


class _Stop(Exception):
    pass


def _x_at_substep(state, slot, k):
    """x of `slot` at the start of sub-step k of the next decision (IDLE), by the oracle."""
    seen = []

    def obs(sub, x, **_):
        if sub == k:
            seen.append(x[slot])
            raise _Stop()
    try:
        oenvs.highway_step(state.copy(), oenvs.A_IDLE, on_substep=obs)
    except _Stop:
        pass
    return seen[0]


def late_ties_scenes():
    """A tie that first appears at sub-step k >= 1: a stopped, crashed vehicle at X and a vehicle on the lane centre
    (heading 0, target = lane, timer 0: it neither steers nor decides) whose x reaches exactly X after k sub-steps.
    Its start x is found among the fp32 neighbours of the estimate by running the oracle."""
    out = []
    for i, (k, X, hi, lo) in enumerate(((1, 300.0, 5, 2), (1, 410.5, 2, 5), (2, 333.0, 7, 3), (3, 360.25, 4, 1),
                                        (1, 480.0, 9, 8), (4, 299.5, 6, 2), (2, 450.0, 3, 10), (1, 377.75, 12, 4))):
        s = _tie_follower_scene(X, i % 2, hi_slot=hi, lo_slot=lo, seed=10 + i)
        target = f32(X)
        x0 = f32(X - k * float(f32(22.0) * oenvs.DT))
        for _ in range(40):
            s.x[lo] = x0
            xk = _x_at_substep(s, lo, k)
            if xk == target:
                break
            x0 = ulp_step(x0, int(target.view(np.int32)) - int(np.float32(xk).view(np.int32)))
        assert _x_at_substep(s, lo, k) == target and s.x[lo] != target, (k, X)
        out.append(s)
    return out


def jam_scenes():
    """Vehicles 6-10 m apart on all lanes, mixed speeds, lane changes in progress: abort-rule hits, collisions
    between vehicles that are not x-neighbours, ego crashes."""
    out = []
    for k in range(12):
        rng = np.random.default_rng(6000 + k)
        s = blank()
        xs, lanes = [], []
        for lane in range(4):
            x = rng.uniform(0.0, 8.0)
            for _ in range(4):
                xs.append(x)
                lanes.append(lane)
                x += rng.uniform(6.0, 10.0)
        xs = np.array(xs)
        ego = int(np.argmin(np.abs(xs - xs.mean())))
        order = [ego] + [i for i in range(V) if i != ego]
        for slot, i in enumerate(order):
            lane = lanes[i]
            tgt = lane
            if rng.uniform() < 0.35:
                tgt = int(np.clip(lane + (1 if rng.uniform() < 0.5 else -1), 0, 3))
            y = 4.0 * lane + (tgt - lane) * rng.uniform(0.3, 2.2)
            put(s, slot, xs[i], y, rng.uniform(15.0, 30.0), ts=rng.uniform(20.0, 30.0),
                h=rng.uniform(-0.05, 0.05) if tgt != lane else 0.0, timer=rng.uniform(0.0, 1.5), tgt=tgt)
        out.append(s)
    return out


def kinematic_scenes():
    """The kinematic edges the step handles with special code: |v| > 40 (clamp) and negative speeds, |v| < 1 (no
    MOBIL) and v = +-0 (not_zero), heading errors beyond +-pi (wrap), vehicles on no lane, an off-road ego, targets
    other than the current lane (two lanes away included), target speeds 0 and above the limit."""
    out = []
    for k in range(10):
        s = oenvs.make_highway_state(5000 + k)
        if k == 0:
            s.v[3], s.v[5], s.tgt_speed[3] = f32(42.0), f32(45.5), f32(30.0)
        elif k == 1:
            s.v[2], s.v[4], s.v[6] = f32(-5.0), f32(-41.0), f32(-0.5)
        elif k == 2:
            s.v[2], s.v[3], s.v[4] = f32(0.5), f32(0.0), f32(-0.0)
            s.timer[2] = s.timer[3] = s.timer[4] = f32(1.5)
        elif k == 3:
            s.h[2], s.h[3], s.h[4], s.h[5] = f32(3.5), f32(-3.5), f32(3.3), f32(-3.2)
            s.y[4] += f32(1.5)
        elif k == 4:
            s.y[2], s.y[3], s.y[4] = f32(-3.5), f32(15.5), f32(16.0)
            s.y[0] = f32(-2.5)
        elif k == 5:
            s.y[0], s.tgt_lane[0], s.h[0] = f32(14.5), 3, f32(0.3)
        elif k == 6:
            cur = np.clip(np.rint(s.y / 4.0), 0, 3).astype(np.int32)
            s.tgt_lane[:] = np.where(cur < 2, cur + 2, cur - 1)
        elif k == 7:
            s.v[0], s.tgt_speed[0], s.speed_index = f32(44.0), f32(30.0), 2
            s.v[7] = f32(40.5)
        elif k == 8:
            s.tgt_speed[2], s.tgt_speed[3], s.tgt_speed[4] = f32(0.0), f32(35.0), f32(-3.0)
        else:
            s.v[2], s.flags[2], s.h[2] = f32(0.0), 3, f32(-0.4)
            s.v[8], s.flags[8] = f32(-2.0), 3
            s.h[5] = f32(-3.3)
        out.append(s)
    return out


_FAMILIES = {"adapter": adapter_scenes, "sync_timers": sync_timers_scenes, "absent": absent_scenes,
             "entry_ties": entry_ties_scenes, "late_ties": late_ties_scenes, "jam": jam_scenes,
             "kinematic": kinematic_scenes}
FAMILY_NAMES = tuple(_FAMILIES)


@functools.lru_cache(maxsize=None)
def _family_words(name):
    return tuple(tuple(s.pack().tolist()) for s in _FAMILIES[name]())


def family(name):
    """Fresh states of a family (deterministic)."""
    return [oenvs.HighwayLiteState.unpack(np.array(w, np.int32)) for w in _family_words(name)]


# -------------------------------------------------------------------------------------------------- trajectories ----
class ActionStream(object):
    """Actions from a fixed RNG over the available ones, with runs of 3-6 LEFT or RIGHT (while available)."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.run, self.dir = 0, oenvs.A_LEFT

    def __call__(self, avail):
        if self.run > 0 and self.dir in avail:
            self.run -= 1
            return self.dir
        if self.rng.uniform() < 0.3:
            self.dir = oenvs.A_LEFT if self.rng.uniform() < 0.5 else oenvs.A_RIGHT
            self.run = int(self.rng.integers(3, 7))
            if self.dir in avail:
                self.run -= 1
                return self.dir
            self.run = 0
        return int(avail[self.rng.integers(len(avail))])


def avail_mask(state):
    return sum(1 << a for a in oenvs.highway_available_actions(state))


def _has_tie(x, present):
    xs = x[present]
    return np.unique(xs).size < xs.size          # -0.0 == +0.0, as in the spec's comparisons


def _rank_distance(x, present, i, j):
    idx = np.nonzero(present)[0]
    rank = np.empty(V, int)
    rank[idx[np.argsort(x[idx], kind="stable")]] = np.arange(idx.size)
    return abs(rank[i] - rank[j])


def _census_step(state, action, counts):
    subs = []
    ego_was = bool(state.flags[0] & 2)

    def obs(**kw):
        subs.append({k: np.array(v, copy=True) for k, v in kw.items()})
    r, term, trunc = oenvs.highway_step(state, action, on_substep=obs)
    present = subs[0]["present"]
    xs = [d["x"] for d in subs] + [state.x.copy()]        # positions the kernel's 16 passes see
    ys = [d["y"] for d in subs] + [state.y.copy()]
    tie = [_has_tie(x, present) for x in xs]
    if tie[0]:
        counts["entry_tie"] += 1
    elif any(tie):
        counts["late_tie"] += 1
    for k in range(16):
        if tie[k]:
            continue
        if not present.all():
            counts["absent_ranked"] += 1
        if k == 0:
            continue
        if tie[k - 1]:
            counts["scan_to_ranked"] += 1
        else:
            idx = np.nonzero(present)[0]
            old = idx[np.argsort(xs[k - 1][idx], kind="stable")]
            if not np.all(np.diff(xs[k][old]) > 0):
                counts["recount"] += 1
        for i in range(V):
            for j in range(i + 1, V):
                if (present[i] and present[j] and abs(xs[k][i] - xs[k][j]) < oenvs.LENGTH
                        and abs(ys[k][i] - ys[k][j]) < oenvs.WIDTH and _rank_distance(xs[k], present, i, j) >= 2):
                    counts["far_collision"] += 1
    n_dec = max(int(d["decide"].sum()) for d in subs)
    for n in (4, 8, 12):
        counts["deciders_gt%d" % n] += n_dec > n
    counts["ego_crash"] += bool(term) and not ego_was
    counts["abort"] += sum(bool(d["abort"].any()) for d in subs)
    counts["clamp"] += sum(bool((d["clamped"] & present).any()) for d in subs)
    counts["wrap"] += sum(bool((d["wrapped"] & present).any()) for d in subs)
    return r, term, trunc


def oracle_trajectory(state, n_decisions=N_DECISIONS, seed=0, counts=None):
    """Steps a copy of `state` n times with ActionStream(seed) on the numpy oracle.  Returns (actions, words
    [n + 1, 136] (the start state first), rewards f32 [n], flags [n] (bit0 terminated, bit1 truncated), avail [n]
    (available-action mask of each new state)).  With `counts` (a Counter), adds the census of the paths reached."""
    s = state.copy()
    pick = ActionStream(seed)
    acts, words, rews, flags, avail = [], [s.pack()], [], [], []
    for _ in range(n_decisions):
        a = pick(oenvs.highway_available_actions(s))
        if counts is None:
            r, term, trunc = oenvs.highway_step(s, a)
        else:
            r, term, trunc = _census_step(s, a, counts)
        acts.append(a)
        words.append(s.pack())
        rews.append(f32(r))
        flags.append((1 if term else 0) | (2 if trunc else 0))
        avail.append(avail_mask(s))
    return (np.array(acts, np.int32), np.stack(words), np.array(rews, np.float32), np.array(flags, np.int32),
            np.array(avail, np.int32))


@functools.lru_cache(maxsize=None)
def _family_runs(name, n_decisions):
    runs, counts = [], []
    for i, s in enumerate(family(name)):
        c = Counter()
        runs.append(oracle_trajectory(s, n_decisions, seed=i, counts=c))
        counts.append(c)
    return runs, counts


def family_trajectories(name, n_decisions=N_DECISIONS):
    """Oracle trajectories of every scene of a family (scene i uses ActionStream(i))."""
    return _family_runs(name, n_decisions)[0]


def census(name, n_decisions=N_DECISIONS):
    """Counter of the kernel paths the family's trajectories reach (keys: PATHS)."""
    total = sum(_family_runs(name, n_decisions)[1], Counter())
    return Counter({k: total[k] for k in PATHS})


def scene_ties(name, n_decisions=N_DECISIONS):
    """Per scene of a family: does its trajectory meet an exact x tie (at entry or later)?"""
    return [c["entry_tie"] + c["late_tie"] > 0 for c in _family_runs(name, n_decisions)[1]]
