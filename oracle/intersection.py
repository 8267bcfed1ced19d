"""IntersectionLite -- numpy statement of docs/INTERSECTION_LITE_SPEC.md (TEST INFRASTRUCTURE).

`intersection-v0` (highway-env) is third-party, unpinned and absent from /root/reference; like HighwayLite
this is the repo's own frozen model of the task BASELINE config C5 names: an unsignalised four-way
intersection, an ego with three longitudinal meta-actions following a left-turn route, IDM traffic on
twelve routes with a static-priority yield rule, deterministic in-step spawning (the spawn counter is part
of the state, so clones spawn identically -- upstream copies the env's np_random with the deep copy).
Every arithmetic operation is a single IEEE binary32 operation in the order written here; the CUDA
statement (rl_agents_b200/csrc/intersection_lite.cuh) reproduces it bit for bit.  Env dynamics parity with
upstream: unpinned (nothing in the reference pins it).
"""
import copy

import numpy as np

from oracle.envs import COMFORT_ACC_MAX, D0, EPS, SPEED_LIMIT, TAU, TWO_SQRT_AB, cos_p, f32, not_zero, sin_p, _Space

V_SLOTS = 16
N_ACTIONS = 3
A_SLOWER, A_IDLE, A_FASTER = 0, 1, 2
SUBSTEPS = 15
DURATION = 13
N_ROUTES = 12                       # entry (S, W, N, E) x turn (left, straight, right): route = 3 * entry + turn

DT = f32(1.0) / f32(15.0)
KP_A = f32(1.0) / f32(0.6)
PI = f32(np.pi)
APPROACH = f32(40.0)                # metres from the spawn point to the box edge
ARC_LEFT = f32(4.0) * PI            # radius 8, quarter circle
ARC_RIGHT = f32(2.0) * PI           # radius 4
BOX_STRAIGHT = f32(12.0)
EXIT = f32(40.0)
LEN = [APPROACH + ARC_LEFT + EXIT, APPROACH + BOX_STRAIGHT + EXIT, APPROACH + ARC_RIGHT + EXIT]
BOX = [ARC_LEFT, BOX_STRAIGHT, ARC_RIGHT]
LENGTH = f32(5.0)
HIT_D2 = f32(12.25)                 # 3.5 m between centres on crossing paths
ACC_MAX = f32(6.0)
OTHER_TS = f32(9.0)
STOP_LINE = f32(38.0)
YIELD_FROM = f32(15.0)              # yield when 15 < s < 38 ...
PRIO_FROM = f32(25.0)               # ... and a vehicle with priority has 25 < s < box exit + 4
PRIO_PAST = f32(4.0)
ENTRY_CLEAR = f32(14.0)
SPAWN_PERIOD = 23
SPAWN_SPEED = f32(8.0)
EGO_ROUTE = 0
SPEED_STEP = f32(4.5)


class IntersectionLiteState(object):
    __slots__ = ("s", "v", "route", "flags", "t", "speed_index", "spawn_clock", "spawn_seq", "arrived")

    def copy(self):
        c = IntersectionLiteState()
        for k in self.__slots__:
            val = getattr(self, k)
            setattr(c, k, val.copy() if isinstance(val, np.ndarray) else val)
        return c

    def pack(self):
        w = np.zeros(136, dtype=np.int32)
        w[0:16] = self.s.view(np.int32)
        w[16:32] = self.v.view(np.int32)
        w[32:48] = self.route
        w[48:64] = self.flags
        w[128], w[129], w[130], w[131], w[132] = self.t, self.speed_index, self.spawn_clock, self.spawn_seq, self.arrived
        return w

    @staticmethod
    def unpack(w):
        w = np.asarray(w, dtype=np.int32)
        st = IntersectionLiteState()
        st.s = w[0:16].view(np.float32).copy()
        st.v = w[16:32].view(np.float32).copy()
        st.route = w[32:48].copy()
        st.flags = w[48:64].copy()
        st.t, st.speed_index, st.spawn_clock, st.spawn_seq, st.arrived = (int(x) for x in w[128:133])
        return st


def make_intersection_state(seed, n_others=8):
    """Scene generator: the ego at s = 10 on route 0 (from the south, turning left) at 4.5 m/s; `n_others`
    vehicles on random routes at 12 m spacing per entry, speeds U(6, 9)."""
    rng = np.random.default_rng(seed)
    st = IntersectionLiteState()
    st.s = np.zeros(V_SLOTS, f32)
    st.v = np.zeros(V_SLOTS, f32)
    st.route = np.zeros(V_SLOTS, np.int32)
    st.flags = np.zeros(V_SLOTS, np.int32)
    st.s[0], st.v[0], st.route[0], st.flags[0] = f32(10.0), f32(4.5), EGO_ROUTE, 1
    next_s = [f32(24.0), f32(2.0), f32(2.0), f32(2.0)]          # the ego's entry starts behind ... ahead of the ego
    for k in range(1, 1 + int(n_others)):
        route = int(rng.integers(0, N_ROUTES))
        e = route // 3
        s0 = next_s[e] + f32(rng.uniform(0.0, 6.0))
        if s0 > f32(36.0):
            continue
        next_s[e] = s0 + f32(12.0)
        st.s[k], st.v[k], st.route[k], st.flags[k] = f32(s0), f32(rng.uniform(6.0, 9.0)), route, 1
    st.t, st.speed_index, st.spawn_clock, st.spawn_seq, st.arrived = 0, 1, 0, int(rng.integers(0, 1000)), 0
    return st


def positions(route, s):
    """World (x, y) of every slot: the entry-S geometry rotated by the entry."""
    turn = route % 3
    entry = route // 3
    x = np.full(s.shape, f32(2.0), f32)
    y = (f32(-46.0) + s).astype(f32)
    u = (s - APPROACH).astype(f32)
    # left turn: radius 8 about (-6, -6)
    th = (u * f32(0.125)).astype(f32)
    lx = (f32(-6.0) + f32(8.0) * cos_p(th)).astype(f32)
    ly = (f32(-6.0) + f32(8.0) * sin_p(th)).astype(f32)
    ul = (u - ARC_LEFT).astype(f32)
    in_l = (turn == 0) & (s >= APPROACH)
    past_l = in_l & (u >= ARC_LEFT)
    x = np.where(in_l, np.where(past_l, (f32(-6.0) - ul).astype(f32), lx), x)
    y = np.where(in_l, np.where(past_l, f32(2.0), ly), y)
    # right turn: radius 4 about (6, -6)
    th = (u * f32(0.25)).astype(f32)
    rx = (f32(6.0) - f32(4.0) * cos_p(th)).astype(f32)
    ry = (f32(-6.0) + f32(4.0) * sin_p(th)).astype(f32)
    ur = (u - ARC_RIGHT).astype(f32)
    in_r = (turn == 2) & (s >= APPROACH)
    past_r = in_r & (u >= ARC_RIGHT)
    x = np.where(in_r, np.where(past_r, (f32(6.0) + ur).astype(f32), rx), x)
    y = np.where(in_r, np.where(past_r, f32(-2.0), ry), y)
    x, y = x.astype(f32), y.astype(f32)
    # entries: S as is, W rotated clockwise, N by 180 degrees, E counter-clockwise (exact: swaps and negations)
    wx = np.where(entry == 0, x, np.where(entry == 1, y, np.where(entry == 2, -x, -y)))
    wy = np.where(entry == 0, y, np.where(entry == 1, -x, np.where(entry == 2, -y, x)))
    return wx.astype(f32), wy.astype(f32)


def _idm(v, has_front, d, v_f):
    ts = np.minimum(np.maximum(OTHER_TS, f32(0.0)), SPEED_LIMIT)
    ratio = np.maximum(v, f32(0.0)) / np.abs(not_zero(ts))
    r2 = ratio * ratio
    r4 = r2 * r2
    acc = COMFORT_ACC_MAX * (f32(1.0) - r4)
    gap = (D0 + v * TAU) + (v * (v - v_f)) / TWO_SQRT_AB
    q = gap / not_zero(d)
    return np.where(has_front, acc - COMFORT_ACC_MAX * (q * q), acc).astype(f32)


def intersection_step(st, action, on_substep=None):
    """One decision step in place; returns (reward f32, terminated, truncated).  `on_substep` (tests' path census)
    is called after every sub-step with keyword arguments: sub, present (at the sub-step's start), s_front (the
    candidate fronts' s, inf elsewhere), has_front, yields, lane, hit (pair matrices), arrived_now (the ego reached
    its route's end), left (others that left), spawn (None, or a dict of the spawn's route, clear, free slots, slot
    and the spawn_seq it used); it does not touch the step."""
    n = V_SLOTS
    if action == A_FASTER:
        st.speed_index = min(st.speed_index + 1, 2)
    elif action == A_SLOWER:
        st.speed_index = max(st.speed_index - 1, 0)
    ts0 = f32(SPEED_STEP * f32(st.speed_index))
    idx = np.arange(n)
    for sub in range(SUBSTEPS):
        present = present0 = (st.flags & 1) != 0
        crashed = (st.flags & 2) != 0
        entry = st.route // 3
        turn = st.route % 3
        box = np.array([BOX[t] for t in turn], f32)
        # ---- front vehicle: same route, or same entry while it is still on the approach ----
        same_lane = (st.route[None, :] == st.route[:, None]) | \
                    ((entry[None, :] == entry[:, None]) & (st.s[None, :] < APPROACH))
        ahead = present[None, :] & (idx[None, :] != idx[:, None]) & same_lane & (st.s[None, :] > st.s[:, None])
        s_f = np.where(ahead, st.s[None, :], f32(np.inf)).astype(f32)
        j_f = np.argmin(s_f, axis=1)                       # smallest s, ties -> smallest slot
        has_f = ahead.any(axis=1)
        d_f = (st.s[j_f] - st.s).astype(f32)
        acc = _idm(st.v, has_f, d_f, st.v[j_f])
        # ---- yield to vehicles with priority (HIGHER route id, another entry) near or inside the box:
        #      the ego (route 0) has the lowest priority, nobody yields to it ----
        prio = present[None, :] & (entry[None, :] != entry[:, None]) & (st.route[None, :] > st.route[:, None]) & \
               (st.s[None, :] > PRIO_FROM) & (st.s[None, :] < ((APPROACH + box) + PRIO_PAST).astype(f32)[None, :])
        yields = (st.s > YIELD_FROM) & (st.s < STOP_LINE) & prio.any(axis=1)
        acc_y = _idm(st.v, np.ones(n, bool), (STOP_LINE - st.s).astype(f32), np.zeros(n, f32))
        acc = np.where(yields, np.minimum(acc, acc_y), acc).astype(f32)
        acc = np.minimum(np.maximum(acc, -ACC_MAX), ACC_MAX).astype(f32)
        acc[0] = KP_A * (ts0 - st.v[0])
        acc = np.where(crashed, -st.v, acc).astype(f32)
        # ---- integrate ----
        new_s = (st.s + st.v * DT).astype(f32)
        new_v = np.maximum((st.v + acc * DT).astype(f32), f32(0.0)).astype(f32)
        st.s = np.where(present, new_s, st.s).astype(f32)
        st.v = np.where(present, new_v, st.v).astype(f32)
        # ---- collisions on the new positions ----
        x, y = positions(st.route, st.s)
        lane = (st.route[None, :] == st.route[:, None]) | \
               ((entry[None, :] == entry[:, None]) & (st.s[None, :] < APPROACH) & (st.s[:, None] < APPROACH))
        dsq = np.abs((st.s[None, :] - st.s[:, None]).astype(f32)) < LENGTH
        dx = (x[None, :] - x[:, None]).astype(f32)
        dy = (y[None, :] - y[:, None]).astype(f32)
        d2 = ((dx * dx).astype(f32) + (dy * dy).astype(f32)).astype(f32)
        hit = present[None, :] & present[:, None] & (idx[None, :] != idx[:, None]) & np.where(lane, dsq, d2 < HIT_D2)
        st.flags = np.where(hit.any(axis=1), st.flags | 2, st.flags).astype(np.int32)
        # ---- vehicles leave at the end of their route (the ego: arrived) ----
        length = np.array([LEN[t] for t in turn], f32)
        gone = present & (st.s >= length)
        arrived_now = bool(gone[0])
        if gone[0]:
            st.arrived = 1
        gone[0] = False
        st.flags = np.where(gone, 0, st.flags).astype(np.int32)
        # ---- deterministic spawning ----
        spawn = None
        st.spawn_clock += 1
        if st.spawn_clock >= SPAWN_PERIOD:
            st.spawn_clock = 0
            k = st.spawn_seq
            st.spawn_seq = (st.spawn_seq + 1) & 0x7fffffff
            h = (k * 2654435761 + 40503) & 0xffffffff
            route = int((h >> 16) % N_ROUTES)
            present = (st.flags & 1) != 0
            clear = not np.any(present & (st.route // 3 == route // 3) & (st.s < ENTRY_CLEAR))
            free = np.nonzero(~present[1:])[0]
            slot = 1 + int(free[0]) if clear and free.size else -1
            if slot > 0:
                st.s[slot], st.v[slot], st.route[slot], st.flags[slot] = f32(0.0), SPAWN_SPEED, route, 1
            spawn = {"route": route, "clear": clear, "free": 1 + free, "slot": slot, "seq": k}
        if on_substep is not None:
            on_substep(sub=sub, present=present0, s_front=s_f, has_front=has_f, yields=yields, lane=lane, hit=hit,
                       arrived_now=arrived_now, left=gone, spawn=spawn)
    st.t += 1
    crashed0 = bool(st.flags[0] & 2)
    if crashed0:
        rew = f32(0.0)
    elif st.arrived:
        rew = f32(1.0)
    else:
        sc = np.minimum(np.maximum((st.v[0] - f32(7.0)) * f32(0.5), f32(0.0)), f32(1.0))
        rew = f32((f32(5.0) + sc) / f32(6.0))
    return f32(rew), crashed0 or bool(st.arrived), st.t >= DURATION


class IntersectionLite(object):
    """gym-style wrapper driven by the reference planners / the oracle planners (deep copy + step)."""

    def __init__(self, state=None, seed=0):
        self.state = state if state is not None else make_intersection_state(seed)
        self.action_space = _Space(N_ACTIONS)

    @property
    def unwrapped(self):
        return self

    def seed(self, seed=None):
        return [seed]

    def simplify(self):
        return copy.deepcopy(self)

    def get_available_actions(self):
        si = self.state.speed_index
        return [A_IDLE] + ([A_FASTER] if si < 2 else []) + ([A_SLOWER] if si > 0 else [])

    def __deepcopy__(self, memo):
        return IntersectionLite(self.state.copy())

    def step(self, action):
        r, term, trunc = intersection_step(self.state, int(action))
        return self.state.pack(), float(r), bool(term), bool(trunc), {}
