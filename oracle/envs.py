"""CPU env models for the oracle -- TEST INFRASTRUCTURE, not product code.

The reference planners never look inside an env: they deep-copy it and call
`step(a)` (rl_agents/agents/common/factory.py:119-134,
rl_agents/agents/tree_search/deterministic.py:36-43).  The env packages the
reference is run on upstream (finite-mdp, highway-env) are third-party,
unpinned and absent from /root/reference (SURVEY.md section 8c), so the repo
freezes its own two models and implements each twice: here in numpy (driven
by the UNMODIFIED reference planners to make the golden vectors) and in CUDA
(rl_agents_b200/csrc).  "parity unpinned" applies to the env dynamics only:
no reference test pins any env arithmetic.

  FiniteMDPLite  table semantics read by value_iteration.py:51-63 plus
                 `step`: r = R[s,a]; s' = T[s,a] (deterministic) or
                 s' ~ P[s,a,:]; done = terminal[s] (the state the action is taken
                 in, as the `finite_mdp` package's MDP.step and value_iteration.py:62 do).
  HighwayLite    docs/HIGHWAY_LITE_SPEC.md -- straight 4-lane highway, one
                 meta-action ego + IDM/MOBIL traffic, 15 physics sub-steps per
                 decision, every operation a single IEEE fp32 op (no FMA) so
                 the CUDA kernel reproduces it bit for bit.
"""
import copy

import numpy as np

f32 = np.float32


# --------------------------------------------------------------------------
# Finite MDP
# --------------------------------------------------------------------------
class _Space(object):
    def __init__(self, n):
        self.n = int(n)


class _MDP(object):
    """Field names follow what value_iteration.py reads: mode / transition /
    reward / terminal / next / state (value_iteration.py:52-63,91-92)."""

    def __init__(self, mode, transition, reward, terminal, nxt=None, state=0):
        self.mode = mode
        self.transition = transition
        self.reward = reward
        self.terminal = terminal
        self.next = nxt
        self.state = int(state)

    def next_state(self, state, action):
        return int(self.transition[state, action])


class FiniteMDPLite(object):
    """gym-like env over explicit tables (5-tuple step API)."""

    def __init__(self, transition, reward, terminal=None, mode="deterministic",
                 nxt=None, state=0, seed=None):
        transition = np.asarray(transition)
        reward = np.asarray(reward, dtype=np.float64)
        if terminal is None:
            terminal = np.zeros(reward.shape[0], dtype=bool)
        terminal = np.asarray(terminal).astype(bool)
        if mode == "deterministic":
            transition = transition.astype(np.int64)
        else:
            transition = transition.astype(np.float64)
        if nxt is not None:
            nxt = np.asarray(nxt).astype(np.int64)
        self.mdp = _MDP(mode, transition, reward, terminal, nxt, state)
        self.action_space = _Space(reward.shape[1])
        self.np_random = np.random.default_rng(seed)

    @property
    def unwrapped(self):
        return self

    def seed(self, seed=None):
        self.np_random = np.random.default_rng(seed)
        return [seed]

    def to_finite_mdp(self):
        # value_iteration.py:14-19: without the finite_mdp package installed
        # the agent takes this conversion path
        return self.mdp

    def step(self, action):
        m = self.mdp
        s = m.state
        r = float(m.reward[s, action])
        if m.mode == "deterministic":
            s2 = int(m.transition[s, action])
        elif m.mode == "stochastic":
            p = m.transition[s, action]
            s2 = int(self.np_random.choice(p.size, p=p))
        elif m.mode == "sparse":
            p = m.transition[s, action]
            s2 = int(m.next[s, action, int(self.np_random.choice(p.size, p=p))])
        else:
            raise ValueError("Unknown mode")
        m.state = s2
        return s2, r, bool(m.terminal[s]), False, {}


class LegacyStepEnv(object):
    """4-tuple `step` + `seed` adapter for olop.py:73,87 (legacy gym API)."""

    def __init__(self, env):
        self.env = env
        self.action_space = env.action_space

    @property
    def unwrapped(self):
        return self.env.unwrapped

    def seed(self, seed=None):
        return self.env.seed(seed)

    def get_available_actions(self):
        return self.env.get_available_actions()

    def __getattr__(self, name):
        if name in ("env", "action_space") or name.startswith("__"):
            raise AttributeError(name)
        return getattr(self.env, name)

    def __deepcopy__(self, memo):
        return LegacyStepEnv(copy.deepcopy(self.env, memo))

    def step(self, action):
        obs, r, done, trunc, info = self.env.step(action)
        return obs, r, done, info


class NoAvailableActions(object):
    """Hide get_available_actions (AttributeError fallback at
    deterministic.py:32-35)."""


def garnet(num_states, num_actions, num_transitions, seed, reward_sparsity=0.5,
           deterministic=False):
    """Seeded garnet-style sparse MDP (SURVEY.md 8(d) C4 input recipe)."""
    rng = np.random.default_rng(seed)
    S, A, B = num_states, num_actions, num_transitions
    nxt = rng.integers(0, S, size=(S, A, B), dtype=np.int64)
    p = rng.uniform(0.0, 1.0, size=(S, A, B))
    p /= p.sum(axis=-1, keepdims=True)
    r = rng.uniform(0.0, 1.0, size=(S, A))
    r *= rng.uniform(0.0, 1.0, size=(S, A)) >= reward_sparsity
    if deterministic:
        return nxt[:, :, 0].copy(), r
    return p, nxt, r


# --------------------------------------------------------------------------
# HighwayLite  (docs/HIGHWAY_LITE_SPEC.md)
# --------------------------------------------------------------------------
V_SLOTS = 16
N_LANES = 4
N_ACTIONS = 5
A_LEFT, A_IDLE, A_RIGHT, A_FASTER, A_SLOWER = 0, 1, 2, 3, 4
SUBSTEPS = 15
DURATION = 40

# every constant is an fp32 value obtained by the fp32 expression shown
LANE_W = f32(4.0)
LENGTH = f32(5.0)
WIDTH = f32(2.0)
HALF_LENGTH = f32(2.5)
DT = f32(1.0) / f32(15.0)
KP_A = f32(1.0) / f32(0.6)
KP_HEADING = f32(1.0) / f32(0.2)
KP_LATERAL = f32(1.0) / f32(0.6)
PI = f32(np.pi)
TWO_PI = f32(2.0) * PI
QUARTER_PI_SIN = f32(0.70710678)      # sin(pi/4): clip of the asin argument
S_BETA_MAX = f32(0.65465367)          # sin(atan(tan(pi/3)/2)): steering clip
HALF_PI = f32(np.pi / 2)
MAX_SPEED = f32(40.0)
SPEED_LIMIT = f32(30.0)
ACC_MAX = f32(6.0)
COMFORT_ACC_MAX = f32(3.0)
D0 = f32(10.0)                        # DISTANCE_WANTED = 5 + LENGTH
TAU = f32(1.5)
TWO_SQRT_AB = f32(2.0) * np.sqrt(f32(15.0))
LANE_CHANGE_DELAY = f32(1.0)
MOBIL_MAX_BRAKING = f32(-2.0)
MOBIL_MIN_GAIN = f32(0.2)
ON_LANE_MARGIN = f32(3.0)             # width/2 + margin 1
EPS = f32(0.01)
SPEED_LO = f32(20.0)
SPEED_RANGE = f32(10.0)
LAT_DEADBAND = f32(1e-9)              # |lateral error| below this is treated as 0 (m)
HEADING_DEADBAND = f32(1e-12)         # |heading error| below this is treated as 0 (rad)

# odd/even polynomials (coefficients are frozen fp32 literals, see spec)
ASIN_C = [f32(x) for x in (0.16666667, 0.075, 0.044642857, 0.030381944,
                           0.022372159, 0.017352764, 0.01396484,
                           0.011551816, 0.0097616, 0.0083903)]
SIN_C = [f32(x) for x in (-1.0 / 6, 1.0 / 120, -1.0 / 5040, 1.0 / 362880,
                          -1.0 / 39916800)]
COS_C = [f32(x) for x in (-0.5, 1.0 / 24, -1.0 / 720, 1.0 / 40320,
                          -1.0 / 3628800, 1.0 / 479001600)]


def _poly(z, coeffs):
    """Horner in fp32, one rounding per op: c0 + z*(c1 + z*(c2 + ...))."""
    acc = np.full_like(z, coeffs[-1])
    for c in coeffs[-2::-1]:
        acc = c + z * acc
    return acc


def asin_p(u):
    """asin on |u| <= sin(pi/4): u * (1 + u^2 * P(u^2))."""
    z = u * u
    return u * (f32(1.0) + z * _poly(z, ASIN_C))


def sin_p(x):
    x = np.minimum(np.maximum(x, -HALF_PI), HALF_PI)
    z = x * x
    return x * (f32(1.0) + z * _poly(z, SIN_C))


def cos_p(x):
    x = np.minimum(np.maximum(x, -HALF_PI), HALF_PI)
    z = x * x
    return f32(1.0) + z * _poly(z, COS_C)


def not_zero(x):
    return np.where(np.abs(x) > EPS, x, np.where(x >= 0, EPS, -EPS)).astype(f32)


class HighwayLiteState(object):
    """Struct-of-arrays state of one env: the same 136 32-bit words the CUDA
    kernel reads (rl_agents_b200/csrc/highway_lite.cuh)."""
    __slots__ = ("x", "y", "h", "v", "tgt_speed", "timer", "tgt_lane",
                 "flags", "t", "speed_index")

    def copy(self):
        s = HighwayLiteState()
        for k in self.__slots__:
            val = getattr(self, k)
            setattr(s, k, val.copy() if isinstance(val, np.ndarray) else val)
        return s

    def pack(self):
        w = np.zeros(136, dtype=np.int32)
        for k, name in enumerate(("x", "y", "h", "v", "tgt_speed", "timer")):
            w[16 * k:16 * k + 16] = getattr(self, name).view(np.int32)
        w[96:112] = self.tgt_lane
        w[112:128] = self.flags
        w[128] = self.t
        w[129] = self.speed_index
        return w

    @staticmethod
    def unpack(w):
        w = np.asarray(w, dtype=np.int32)
        s = HighwayLiteState()
        for k, name in enumerate(("x", "y", "h", "v", "tgt_speed", "timer")):
            setattr(s, name, w[16 * k:16 * k + 16].view(np.float32).copy())
        s.tgt_lane = w[96:112].copy()
        s.flags = w[112:128].copy()
        s.t = int(w[128])
        s.speed_index = int(w[129])
        return s


def make_highway_state(seed, n_vehicles=V_SLOTS):
    """Synthetic highway-v0-like scene: per-lane cumulative gaps U(40,80) m
    (about the IDM desired gap, as upstream's density-1 spacing gives), speeds
    U(21,24) (=0.7..0.8 x speed limit), ego = the vehicle nearest x=0."""
    rng = np.random.default_rng(seed)
    n = int(n_vehicles)
    lanes = rng.integers(0, N_LANES, size=n)
    next_x = -160.0 + rng.uniform(0.0, 40.0, size=N_LANES)
    xs = np.zeros(n)
    for k in range(n):
        xs[k] = next_x[lanes[k]] + rng.uniform(40.0, 80.0)
        next_x[lanes[k]] = xs[k]
    speeds = rng.uniform(21.0, 24.0, size=n)
    timers = rng.uniform(0.0, 1.0, size=n)
    ego = int(np.argmin(np.abs(xs)))
    order = [ego] + [k for k in range(n) if k != ego]
    s = HighwayLiteState()
    s.x = np.zeros(V_SLOTS, f32)
    s.y = np.zeros(V_SLOTS, f32)
    s.h = np.zeros(V_SLOTS, f32)
    s.v = np.zeros(V_SLOTS, f32)
    s.tgt_speed = np.zeros(V_SLOTS, f32)
    s.timer = np.zeros(V_SLOTS, f32)
    s.tgt_lane = np.zeros(V_SLOTS, np.int32)
    s.flags = np.zeros(V_SLOTS, np.int32)
    for slot, k in enumerate(order):
        s.x[slot] = f32(xs[k])
        s.y[slot] = f32(4.0 * lanes[k])
        s.v[slot] = f32(speeds[k])
        s.tgt_speed[slot] = f32(speeds[k])
        s.timer[slot] = f32(timers[k])
        s.tgt_lane[slot] = lanes[k]
        s.flags[slot] = 1
    s.v[0] = f32(25.0)
    s.tgt_speed[0] = f32(25.0)
    s.t = 0
    s.speed_index = 1
    return s


def _idm(v_i, ts_i, has_front, x_i, x_f, v_f):
    """IDM acceleration (unclipped) of vehicles i w.r.t. optional fronts."""
    ts = np.minimum(np.maximum(ts_i, f32(0.0)), SPEED_LIMIT)
    ratio = np.maximum(v_i, f32(0.0)) / np.abs(not_zero(ts))
    r2 = ratio * ratio
    r4 = r2 * r2
    acc = COMFORT_ACC_MAX * (f32(1.0) - r4)
    d = x_f - x_i
    gap = (D0 + v_i * TAU) + (v_i * (v_i - v_f)) / TWO_SQRT_AB
    q = gap / not_zero(d)
    acc_f = acc - COMFORT_ACC_MAX * (q * q)
    return np.where(has_front, acc_f, acc).astype(f32)


def _neighbours(x, present, lane_y_of_i, y):
    """front/rear of every vehicle i among vehicles on the lane centred at
    lane_y_of_i[i].  Index-order tie rules of a sequential scan with
    `s <= s_v and s_v <= s_front` (later index wins ties) for the front and
    `s_v < s and s_v > s_rear` (first index wins) for the rear."""
    n = x.size
    idx = np.arange(n)
    on_lane = np.abs(y[None, :] - lane_y_of_i[:, None]) <= ON_LANE_MARGIN
    cand = on_lane & present[None, :] & (idx[None, :] != idx[:, None])
    is_front = cand & (x[None, :] >= x[:, None])
    is_rear = cand & (x[None, :] < x[:, None])
    xf = np.where(is_front, x[None, :], np.inf)
    fmin = xf.min(axis=1)
    has_front = is_front.any(axis=1)
    # later index wins ties -> last arg-min
    front = n - 1 - np.argmax((xf == fmin[:, None])[:, ::-1], axis=1)
    xr = np.where(is_rear, x[None, :], -np.inf)
    rmax = xr.max(axis=1)
    has_rear = is_rear.any(axis=1)
    rear = np.argmax(xr == rmax[:, None], axis=1)
    return has_front, front, has_rear, rear


def highway_available_actions(state):
    cur = int(np.clip(np.rint(state.y[0] / LANE_W), 0, N_LANES - 1))
    actions = [A_IDLE]
    if cur > 0:
        actions.append(A_LEFT)
    if cur < N_LANES - 1:
        actions.append(A_RIGHT)
    if state.speed_index < 2:
        actions.append(A_FASTER)
    if state.speed_index > 0:
        actions.append(A_SLOWER)
    return actions


def highway_step(state, action, on_substep=None):
    """One decision step (15 sub-steps) in place; returns (reward f32,
    terminated, truncated).

    `on_substep`, when given, is called once per sub-step, after the lane
    decisions and before the integration, with keyword arguments (arrays over
    the 16 slots, read-only): sub, x, y, v, present, crashed (as of the
    sub-step start), cur, tgt (target lanes at the sub-step start), new_tgt,
    decide (MOBIL deciders), abort (abort rule fired), wrapped (heading error
    wrapped by 2*pi) and clamped (|v| > MAX_SPEED).  It observes only: the
    step computes the same values with or without it."""
    s = state
    n = V_SLOTS
    idx = np.arange(n)
    present = (s.flags & 1) != 0
    crashed = (s.flags & 2) != 0
    is_idm = idx > 0

    # ---- ego meta-action (frame 0) ----
    if action in (A_FASTER, A_SLOWER):
        si = int(np.clip(np.rint(((s.v[0] - SPEED_LO) / SPEED_RANGE) * f32(2.0)), 0, 2))
        si = si + 1 if action == A_FASTER else si - 1
        si = min(max(si, 0), 2)
        s.speed_index = si
        s.tgt_speed[0] = f32(20.0 + 5.0 * si)
    elif action == A_LEFT:
        s.tgt_lane[0] = max(int(s.tgt_lane[0]) - 1, 0)
    elif action == A_RIGHT:
        s.tgt_lane[0] = min(int(s.tgt_lane[0]) + 1, N_LANES - 1)

    for sub in range(SUBSTEPS):
        x, y, h, v = s.x, s.y, s.h, s.v
        cur = np.clip(np.rint(y / LANE_W), 0, N_LANES - 1).astype(np.int32)
        cur_y = cur.astype(f32) * LANE_W
        tgt = s.tgt_lane.copy()
        active = present & ~crashed & is_idm

        # ---- lane-change policy (IDM vehicles) ----
        changing = active & (cur != tgt)
        # abort rule
        d_ij = x[None, :] - x[:, None]
        gap_ij = (D0 + v[:, None] * TAU) + (v[:, None] * (v[:, None] - v[None, :])) / TWO_SQRT_AB
        conflict = (present[None, :] & (idx[None, :] != idx[:, None])
                    & (cur[None, :] != tgt[:, None]) & (tgt[None, :] == tgt[:, None])
                    & (d_ij > 0) & (d_ij < gap_ij))
        abort = changing & conflict.any(axis=1)
        new_tgt = np.where(abort, cur, tgt)
        # MOBIL, once LANE_CHANGE_DELAY has elapsed
        decide = active & ~changing & (s.timer > LANE_CHANGE_DELAY)
        timer = np.where(decide, f32(0.0), s.timer).astype(f32)
        hf_c, f_c, _, _ = _neighbours(x, present, cur_y, y)
        self_a = _idm(v, s.tgt_speed, hf_c, x, x[f_c], v[f_c])
        for side in (-1, 1):
            lane = cur + side
            ok = decide & (lane >= 0) & (lane < N_LANES) & (np.abs(v) >= f32(1.0))
            lane_y = lane.astype(f32) * LANE_W
            hf_n, f_n, hr_n, r_n = _neighbours(x, present, lane_y, y)
            # new follower (rear on the side lane) braking behind i
            foll_pred = _idm(v[r_n], s.tgt_speed[r_n], np.ones(n, bool), x[r_n], x, v)
            foll_pred = np.where(hr_n, foll_pred, f32(0.0))
            self_pred = _idm(v, s.tgt_speed, hf_n, x, x[f_n], v[f_n])
            jerk = self_pred - self_a
            go = ok & ~(foll_pred < MOBIL_MAX_BRAKING) & ~(jerk < MOBIL_MIN_GAIN)
            new_tgt = np.where(go, lane, new_tgt)
        tgt = new_tgt.astype(np.int32)

        # ---- steering (all controlled vehicles, ego included) ----
        lat = y - tgt.astype(f32) * LANE_W
        lat = np.where(np.abs(lat) < LAT_DEADBAND, f32(0.0), lat).astype(f32)
        lat_speed_cmd = -(KP_LATERAL * lat)
        nzv = not_zero(v)
        u = lat_speed_cmd / nzv
        u = np.minimum(np.maximum(u, -QUARTER_PI_SIN), QUARTER_PI_SIN)
        heading_ref = asin_p(u)
        dh = heading_ref - h
        if on_substep is not None:
            wrapped = (dh > PI) | (np.where(dh > PI, dh - TWO_PI, dh) < -PI)
            on_substep(sub=sub, x=x, y=y, v=v, present=present, crashed=crashed, cur=cur, tgt=s.tgt_lane,
                       new_tgt=tgt, decide=decide, abort=abort, wrapped=wrapped, clamped=np.abs(v) > MAX_SPEED)
        dh = np.where(dh > PI, dh - TWO_PI, dh)
        dh = np.where(dh < -PI, dh + TWO_PI, dh)
        dh = np.where(np.abs(dh) < HEADING_DEADBAND, f32(0.0), dh).astype(f32)
        rate = KP_HEADING * dh
        sb = (HALF_LENGTH / nzv) * rate
        sb = np.minimum(np.maximum(sb, -S_BETA_MAX), S_BETA_MAX)

        # ---- longitudinal ----
        acc = _idm(v, s.tgt_speed, hf_c, x, x[f_c], v[f_c])
        tgt_y = tgt.astype(f32) * LANE_W
        hf_t, f_t, _, _ = _neighbours(x, present, tgt_y, y)
        acc_t = _idm(v, s.tgt_speed, hf_t, x, x[f_t], v[f_t])
        acc = np.where(cur != tgt, np.minimum(acc, acc_t), acc)
        acc = np.minimum(np.maximum(acc, -ACC_MAX), ACC_MAX)
        acc[0] = KP_A * (s.tgt_speed[0] - v[0])

        # ---- kinematics ----
        sb = np.where(crashed, f32(0.0), sb).astype(f32)
        acc = np.where(crashed, -v, acc).astype(f32)
        acc = np.where(v > MAX_SPEED, np.minimum(acc, MAX_SPEED - v), acc)
        acc = np.where(v < -MAX_SPEED, np.maximum(acc, -MAX_SPEED - v), acc).astype(f32)
        cb = np.sqrt(f32(1.0) - sb * sb)
        sh = sin_p(h)
        ch = cos_p(h)
        c_hb = ch * cb - sh * sb
        s_hb = sh * cb + ch * sb
        nx = x + (v * c_hb) * DT
        ny = y + (v * s_hb) * DT
        nh = h + ((v * sb) / HALF_LENGTH) * DT
        nv = v + acc * DT
        ntimer = np.where(is_idm, timer + DT, timer)
        s.x = np.where(present, nx, x).astype(f32)
        s.y = np.where(present, ny, y).astype(f32)
        s.h = np.where(present, nh, h).astype(f32)
        s.v = np.where(present, nv, v).astype(f32)
        s.timer = np.where(present, ntimer, s.timer).astype(f32)
        s.tgt_lane = np.where(present, tgt, s.tgt_lane).astype(np.int32)

        # ---- collisions (axis-aligned boxes, all pairs) ----
        hit = (present[:, None] & present[None, :] & (idx[:, None] != idx[None, :])
               & (np.abs(s.x[:, None] - s.x[None, :]) < LENGTH)
               & (np.abs(s.y[:, None] - s.y[None, :]) < WIDTH))
        crashed = crashed | hit.any(axis=1)
        s.flags = (present.astype(np.int32) | (crashed.astype(np.int32) << 1)).astype(np.int32)

    # ---- reward ----
    ego_crashed = bool(crashed[0])
    lane_r = f32(s.tgt_lane[0]) / f32(N_LANES - 1)
    fs = s.v[0] * cos_p(s.h[0:1])[0]
    sc = (fs - SPEED_LO) / SPEED_RANGE
    sc = min(max(sc, f32(0.0)), f32(1.0))
    r = (f32(-1.0) if ego_crashed else f32(0.0)) + f32(0.1) * lane_r
    r = r + f32(0.4) * sc
    r = (r + f32(1.0)) / f32(1.5)
    on_road = (s.y[0] >= f32(-2.0)) and (s.y[0] <= f32(14.0))
    if not on_road:
        r = f32(0.0)
    s.t += 1
    return f32(r), ego_crashed, s.t >= DURATION


# ---------------------------------------------------------------------------
# TTC-grid MDP of a HighwayLite scene (docs/HIGHWAY_LITE_SPEC.md section 9): what
# `env.unwrapped.to_finite_mdp()` hands to ValueIterationAgent
# (rl_agents/agents/dynamic_programming/value_iteration.py:17,32).  It follows the
# published algorithm of highway-env's `envs/common/finite_mdp.py` (not under
# /root/reference, not installed: restated from its documented behaviour --
# `compute_ttc_grid(env, time_quantization=1., horizon=10.)` is how the reference
# itself calls it, agents/dynamic_programming/graphics.py:46).  Literal loops.
# ---------------------------------------------------------------------------
TTC_SPEEDS = (20.0, 25.0, 30.0)
TTC_HORIZON = 10.0
TTC_TIME_QUANTIZATION = 1.0
TTC_COLLISION_REWARD, TTC_RIGHT_LANE_REWARD, TTC_HIGH_SPEED_REWARD, TTC_LANE_CHANGE_REWARD = -1.0, 0.1, 0.4, 0.0


def highway_ttc_grid(state):
    """grid[h, lane, t] in {0, 0.5, 1}: cost of being on `lane` in t seconds when driving at TTC_SPEEDS[h]."""
    n_t = int(TTC_HORIZON / TTC_TIME_QUANTIZATION)
    grid = np.zeros((len(TTC_SPEEDS), N_LANES, n_t))
    margin = float(LENGTH) / 2 + float(LENGTH) / 2
    for h, ego_speed in enumerate(TTC_SPEEDS):
        for k in range(1, V_SLOTS):
            if not (state.flags[k] & 1):
                continue
            if ego_speed == float(state.v[k]):
                continue
            c = cos_p(np.array([f32(state.h[k] - state.h[0])], dtype=f32))[0]      # fp32, the step's own polynomial
            projected = float(state.v[k]) * float(c)
            diff = ego_speed - projected
            nz = diff if abs(diff) > 0.01 else (0.01 if diff >= 0 else -0.01)
            lane = int(np.clip(np.rint(state.y[k] / f32(4.0)), 0, N_LANES - 1))
            for m, cost in ((0.0, 1.0), (-margin, 0.5), (margin, 0.5)):
                distance = (float(state.x[k]) - float(state.x[0])) + m
                ttc = distance / nz
                if ttc < 0:
                    continue
                for t in (int(ttc / TTC_TIME_QUANTIZATION), int(np.ceil(ttc / TTC_TIME_QUANTIZATION))):
                    if 0 <= t < n_t:
                        grid[h, lane, t] = max(grid[h, lane, t], cost)
    return grid


def highway_finite_mdp(state):
    """Deterministic MDP over (speed index, lane, time) cells: transition [S, A] int, reward [S, A], terminal [S]."""
    grid = highway_ttc_grid(state)
    n_h, n_l, n_t = grid.shape
    n_s = grid.size

    def cell(h, i, j):
        return (min(max(h, 0), n_h - 1) * n_l + min(max(i, 0), n_l - 1)) * n_t + min(max(j, 0), n_t - 1)

    transition = np.zeros((n_s, N_ACTIONS), dtype=np.int64)
    reward = np.zeros((n_s, N_ACTIONS))
    terminal = np.zeros(n_s, dtype=bool)
    action_reward = (TTC_LANE_CHANGE_REWARD, 0.0, TTC_LANE_CHANGE_REWARD, 0.0, 0.0)
    for h in range(n_h):
        for i in range(n_l):
            for j in range(n_t):
                s = (h * n_l + i) * n_t + j
                state_reward = (TTC_COLLISION_REWARD * grid[h, i, j] + TTC_RIGHT_LANE_REWARD * (i / max(n_l - 1, 1))
                                + TTC_HIGH_SPEED_REWARD * (h / max(n_h - 1, 1)))
                terminal[s] = grid[h, i, j] == 1 or j == n_t - 1
                for a in range(N_ACTIONS):
                    nh, ni = h, i
                    if a == A_LEFT:
                        ni = i - 1
                    elif a == A_RIGHT:
                        ni = i + 1
                    elif a == A_FASTER and j == 0:
                        nh = h + 1
                    elif a == A_SLOWER and j == 0:
                        nh = h - 1
                    transition[s, a] = cell(nh, ni, j + 1)
                    reward[s, a] = state_reward + action_reward[a]
    ego_lane = int(np.clip(np.rint(state.y[0] / f32(4.0)), 0, N_LANES - 1))
    mdp = _MDP("deterministic", transition, reward, terminal, state=cell(int(state.speed_index), ego_lane, 0))
    mdp.original_shape = grid.shape
    return mdp


class HighwayLite(object):
    """gym-like wrapper the reference planners can deepcopy and step."""

    def __init__(self, state=None, seed=0):
        self.state = state if state is not None else make_highway_state(seed)
        self.action_space = _Space(N_ACTIONS)

    @property
    def unwrapped(self):
        return self

    def seed(self, seed=None):
        return [seed]

    def simplify(self):
        return copy.deepcopy(self)

    def get_available_actions(self):
        return highway_available_actions(self.state)

    def to_finite_mdp(self):
        return highway_finite_mdp(self.state)

    def __deepcopy__(self, memo):
        return HighwayLite(self.state.copy())

    def step(self, action):
        r, term, trunc = highway_step(self.state, int(action))
        return self.state.t, float(r), term, trunc, {}
