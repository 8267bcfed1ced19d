"""IntersectionLite env (docs/INTERSECTION_LITE_SPEC.md): host-side container of one scene (136 32-bit words) with a
gymnasium-style API -- the repo's model of BASELINE config C5's `intersection-v0`.  `step` runs the CUDA transition
(b2_intersection_step), the same device code the wavefront OPD kernel expands nodes with.  `set_route_at_intersection`
makes the route-hypothesis copies DROP plans over (spec "Route hypotheses"), in numpy on the host."""
import copy

import numpy as np

from rl_agents_b200 import _lib

V_SLOTS, N_ACTIONS, N_ROUTES = 16, 3, 12
N_TURNS = 3
APPROACH = np.float32(40.0)          # the box edge: vehicles with s < APPROACH are still on their entry's approach
ACTIONS = {0: "SLOWER", 1: "IDLE", 2: "FASTER"}


class _Space(object):
    def __init__(self, n):
        self.n = int(n)


def make_scene(seed, n_others=8):
    """The ego at s = 10 on route 0 (from the south, turning left) at 4.5 m/s; `n_others` vehicles on random routes
    at 12 m spacing per entry, speeds U(6, 9); the spawn sequence starts at a seeded counter."""
    f32 = np.float32
    rng = np.random.default_rng(seed)
    w = np.zeros(_lib.HW_STATE_WORDS, dtype=np.int32)
    f = w[:32].view(np.float32)
    f[0], f[16], w[32], w[48] = f32(10.0), f32(4.5), 0, 1
    next_s = [f32(24.0), f32(2.0), f32(2.0), f32(2.0)]
    for k in range(1, 1 + int(n_others)):
        route = int(rng.integers(0, N_ROUTES))
        e = route // 3
        s0 = next_s[e] + f32(rng.uniform(0.0, 6.0))
        if s0 > f32(36.0):
            continue
        next_s[e] = s0 + f32(12.0)
        f[k], f[16 + k], w[32 + k], w[48 + k] = f32(s0), f32(rng.uniform(6.0, 9.0)), route, 1
    w[128], w[129], w[130], w[131], w[132] = 0, 1, 0, int(rng.integers(0, 1000)), 0
    return w


def route_hypothesis(words, _to):
    """The scene `words` (left untouched) with every present other vehicle still on its approach (slot >= 1,
    s < 40) turned towards `_to`: an integer turn (0 left, 1 straight, 2 right, taken mod 3) or "random" (a turn
    hashed from t, the slot and spawn_seq).  Raises ValueError on any other argument."""
    if isinstance(_to, str) and _to == "random":
        turn = None
    elif isinstance(_to, (int, np.integer)) and not isinstance(_to, (bool, np.bool_)):
        turn = int(_to) % N_TURNS
    else:
        raise ValueError("set_route_at_intersection takes an integer turn or \"random\", got %r" % (_to,))
    w = np.array(words, dtype=np.int32)
    s = w[0:V_SLOTS].view(np.float32)
    t, seq = int(w[128]), int(w[131])
    for k in range(1, V_SLOTS):
        if not (w[48 + k] & 1) or not s[k] < APPROACH:
            continue
        k_turn = turn
        if turn is None:
            h = ((t * 16 + k) * 2654435761 + seq * 40503) & 0xffffffff
            k_turn = (h >> 16) % N_TURNS
        w[32 + k] = N_TURNS * (int(w[32 + k]) // N_TURNS) + k_turn
    return w


def available_actions(words):
    si = int(words[129])
    return [1] + ([2] if si < 2 else []) + ([0] if si > 0 else [])


class IntersectionLiteEnv(object):
    b2_env_kind = "intersection"

    def __init__(self, words=None, seed=0, config=None):
        self.config = dict(config or {})
        self.words = np.array(words, dtype=np.int32) if words is not None else make_scene(seed)
        assert self.words.shape == (_lib.HW_STATE_WORDS,)
        self.action_space = _Space(N_ACTIONS)
        self._seed = seed

    @property
    def unwrapped(self):
        return self

    def seed(self, seed=None):
        self._seed = seed
        return [seed]

    def reset(self, seed=None, options=None):
        if seed is not None:
            self._seed = seed
        self.words = make_scene(self._seed if self._seed is not None else 0)
        return self.observation(), {}

    def simplify(self):
        return copy.deepcopy(self)

    def get_available_actions(self):
        return available_actions(self.words)

    def set_route_at_intersection(self, _to):
        """A copy of the env in which the other vehicles still on their approach take the exit `_to` (0 left,
        1 straight, 2 right, mod 3) or "random"; the env itself is unchanged (route_hypothesis)."""
        env = copy.deepcopy(self)
        env.words = route_hypothesis(self.words, _to)
        return env

    def observation(self):
        f = self.words[:32].view(np.float32).reshape(2, V_SLOTS)
        present = (self.words[48:64] & 1).astype(np.float32)
        return np.stack([present, f[0], f[1], self.words[32:48].astype(np.float32)], axis=1)

    def step(self, action):
        import torch
        lib = _lib.load()
        dev = torch.device("cuda")
        st = torch.from_numpy(self.words.reshape(1, -1)).to(dev)
        act = torch.tensor([int(action)], dtype=torch.int32, device=dev)
        rew = torch.empty(1, dtype=torch.float32, device=dev)
        flg = torch.empty(1, dtype=torch.int32, device=dev)
        _lib.check(lib.b2_intersection_step(_lib.ptr(st), _lib.ptr(act), _lib.ptr(rew), _lib.ptr(flg), None, 1,
                                            _lib.current_stream()))
        self.words = st.cpu().numpy().reshape(-1)
        flags = int(flg.item())
        return self.observation(), float(rew.item()), bool(flags & 1), bool(flags & 2), {}
