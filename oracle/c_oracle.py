"""ctypes wrapper of the C oracle (oracle/c) -- TEST INFRASTRUCTURE.  Third statement of the
HighwayLite spec and a literal C OPD; pinned bit-exactly against oracle/envs.py and
oracle/planners.py (tests/test_c_oracle.py), hence against the reference's golden vectors.  Also the
third statement of the IntersectionLite spec (`il_*`), pinned against oracle/intersection.py and the
same planners (tests/test_intersection_scene_families.py)."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "c")
LIB = os.path.join(HERE, "liboracle_c.so")
_lib = None


def build(force=False):
    srcs = [os.path.join(HERE, f) for f in ("highway_lite.c", "intersection_lite.c", "opd.c", "mcts.c", "highway_lite.h",
                                               "intersection_lite.h", "Makefile")]
    if force or not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in srcs):
        subprocess.run(["make", "-C", HERE, "-s", "-B"], check=True)
    return LIB


def load():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(LIB)
        _lib.opd_highway_plan.restype = ctypes.c_int
        _lib.opd_highway_plan_wave.restype = ctypes.c_int
        _lib.il_opd_plan.restype = ctypes.c_int
        _lib.il_opd_plan_wave.restype = ctypes.c_int
        _lib.mcts_highway_plan.restype = ctypes.c_int
        _lib.mcts_highway_plan_wave.restype = ctypes.c_int
        _lib.hl_ttc_value_iteration.restype = ctypes.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _step_batch(fn, words, actions):
    w = np.ascontiguousarray(words, dtype=np.int32).copy()
    a = np.ascontiguousarray(actions, dtype=np.int32)
    r = np.zeros(len(a), dtype=np.float32)
    f = np.zeros(len(a), dtype=np.int32)
    fn(_p(w), _p(a), _p(r), _p(f), ctypes.c_int(len(a)))
    return w, r, f


def step_batch(words, actions):
    """words [n,136] int32 (updated copy returned), actions [n] -> (words, rewards f32, flags)."""
    return _step_batch(load().hl_step_batch, words, actions)


def il_step_batch(words, actions):
    """IntersectionLite: words [n,136] int32 (updated copy returned), actions [n] -> (words, rewards f32, flags
    (bit0 terminated, bit1 truncated))."""
    return _step_batch(load().il_step_batch, words, actions)


def _tree_arrays(cap):
    i32 = {k: np.zeros(cap, dtype=np.int32) for k in ("parent", "action", "depth", "count", "first_child",
                                                      "n_children", "done")}
    f64 = {k: np.zeros(cap, dtype=np.float64) for k in ("reward", "lower", "upper")}
    ptrs = [_p(i32[k]) for k in ("parent", "action", "depth", "count", "first_child", "n_children", "done")]
    return i32, f64, ptrs + [_p(f64["reward"]), _p(f64["lower"]), _p(f64["upper"])]


def _strict(fn, n_actions, root_words, budget, gamma, terminal_reward):
    i32, f64, ptrs = _tree_arrays(1 + (int(budget) // n_actions) * n_actions)
    n_leaves = ctypes.c_int32(0)
    root = np.ascontiguousarray(root_words, dtype=np.int32)
    n = fn(_p(root), ctypes.c_int(int(budget)), ctypes.c_double(gamma), ctypes.c_double(terminal_reward), *ptrs,
           ctypes.byref(n_leaves))
    if n < 0:
        raise ValueError("This planner assumes that all rewards are normalized in [0, 1]")
    out = {k: v[:n] for k, v in {**i32, **f64}.items()}
    out["n_leaves"] = n_leaves.value
    return out


def _wave(fn, n_actions, root_words, budget, gamma, width, terminal_reward, lag, wave_end=None):
    i32, f64, ptrs = _tree_arrays(1 + (int(budget) // n_actions) * n_actions)
    n_leaves, n_waves = ctypes.c_int32(0), ctypes.c_int32(0)
    root = np.ascontiguousarray(root_words, dtype=np.int32)
    extra = [] if wave_end is None else [_p(wave_end)]
    n = fn(_p(root), ctypes.c_int(int(budget)), ctypes.c_double(gamma), ctypes.c_double(terminal_reward),
           ctypes.c_int(int(width)), ctypes.c_int(int(lag)), *ptrs, ctypes.byref(n_leaves), ctypes.byref(n_waves), *extra)
    if n < 0:
        raise ValueError("This planner assumes that all rewards are normalized in [0, 1]")
    out = {k: v[:n] for k, v in {**i32, **f64}.items()}
    out["n_leaves"], out["n_waves"] = n_leaves.value, n_waves.value
    if wave_end is not None:
        out["wave_end"] = wave_end[:n_waves.value].copy()
    return out


def opd_plan(root_words, budget, gamma, terminal_reward=0.0):
    """Returns a dict of node arrays in creation order (same fields as oracle.planners.Tree)."""
    return _strict(load().opd_highway_plan, 5, root_words, budget, gamma, terminal_reward)


def opd_plan_wave(root_words, budget, gamma, width, terminal_reward=0.0, lag=0):
    """The wavefront specification (oracle.planners.opd_plan_wavefront) in C; same dict as opd_plan + n_waves."""
    return _wave(load().opd_highway_plan_wave, 5, root_words, budget, gamma, width, terminal_reward, lag)


def il_opd_plan(root_words, budget, gamma, terminal_reward=0.0):
    """OPD on an IntersectionLite scene (3 actions); the same dict as opd_plan."""
    return _strict(load().il_opd_plan, 3, root_words, budget, gamma, terminal_reward)


def il_opd_plan_wave(root_words, budget, gamma, width, terminal_reward=0.0, lag=0):
    """The wavefront specification on an IntersectionLite scene; the same dict as opd_plan_wave, plus `wave_end`:
    per wave, the number of nodes after it (wave w created the ids wave_end[w - 1] .. wave_end[w] - 1)."""
    wave_end = np.zeros(1 + int(budget) // 3, dtype=np.int32)
    return _wave(load().il_opd_plan_wave, 3, root_words, budget, gamma, width, terminal_reward, lag, wave_end)


def mcts_plan(root_words, episodes, horizon, gamma, temperature, rng_words):
    """rng_words: uint64[6] numpy PCG64 state (advanced copy returned).  Returns (tree dict, rng_words)."""
    lib = load()
    cap = 1 + int(episodes) * 5
    i32 = {k: np.zeros(cap, dtype=np.int32) for k in ("parent", "action", "count", "first_child", "n_children")}
    f64 = {k: np.zeros(cap, dtype=np.float64) for k in ("value", "prior")}
    cdf = np.ones((6, 5), dtype=np.float64)
    for n in range(1, 6):
        c = (np.ones(n) / n).cumsum()
        c /= c[-1]
        cdf[n, :n] = c
    words = np.ascontiguousarray(rng_words, dtype=np.uint64).copy()
    root = np.ascontiguousarray(root_words, dtype=np.int32)
    n = lib.mcts_highway_plan(_p(root), ctypes.c_int(int(episodes)), ctypes.c_int(int(horizon)), ctypes.c_double(gamma),
                              ctypes.c_double(temperature), _p(words), _p(cdf), _p(i32["parent"]), _p(i32["action"]),
                              _p(i32["count"]), _p(i32["first_child"]), _p(i32["n_children"]), _p(f64["value"]),
                              _p(f64["prior"]))
    return {k: v[:n] for k, v in {**i32, **f64}.items()}, words


def mcts_plan_wave(root_words, episodes, horizon, gamma, temperature, width, seed):
    """The wavefront MCTS specification (oracle.planners.mcts_plan_wavefront) in C -> tree dict + env_steps."""
    lib = load()
    cap = 1 + int(episodes) * 5
    i32 = {k: np.zeros(cap, dtype=np.int32) for k in ("parent", "action", "count", "first_child", "n_children")}
    vsum = np.zeros(cap, dtype=np.int64)
    value = np.zeros(cap, dtype=np.float64)
    gp = np.array([float(gamma) ** h for h in range(int(horizon) + 1)], dtype=np.float64)
    root = np.ascontiguousarray(root_words, dtype=np.int32)
    steps = lib.mcts_highway_plan_wave(_p(root), ctypes.c_int(int(episodes)), ctypes.c_int(int(horizon)), _p(gp),
                                       ctypes.c_double(temperature), ctypes.c_int(int(width)),
                                       ctypes.c_uint64(int(seed) & ((1 << 64) - 1)), _p(i32["parent"]), _p(i32["action"]),
                                       _p(i32["count"]), _p(i32["first_child"]), _p(i32["n_children"]), _p(vsum), _p(value))
    out = dict(i32)
    out["vsum"], out["value"], out["env_steps"] = vsum, value, steps
    return out


def ttc_grid(words):
    """TTC cost grid [3, 4, 10] of a scene (docs/HIGHWAY_LITE_SPEC.md section 9)."""
    lib = load()
    w = np.ascontiguousarray(words, dtype=np.int32)
    g = np.zeros((3, 4, 10), dtype=np.float64)
    lib.hl_ttc_grid(_p(w), _p(g))
    return g


def ttc_value_iteration(words, gamma, iterations, rtol=1e-5, atol=1e-8):
    """ValueIterationAgent on the scene's TTC-grid MDP: (Q [120, 5], mdp.state, action, sweeps)."""
    lib = load()
    w = np.ascontiguousarray(words, dtype=np.int32)
    q = np.zeros((120, 5), dtype=np.float64)
    st, act = ctypes.c_int32(0), ctypes.c_int32(0)
    sweeps = lib.hl_ttc_value_iteration(_p(w), ctypes.c_double(gamma), ctypes.c_int(int(iterations)), ctypes.c_double(rtol),
                                        ctypes.c_double(atol), _p(q), ctypes.byref(st), ctypes.byref(act))
    return q, int(st.value), int(act.value), int(sweeps)


def ttc_value_iteration_batch(words, gamma, iterations):
    """Actions for n scenes, one after the other on one core (the CPU data point beside b2_highway_ttc_vi)."""
    lib = load()
    w = np.ascontiguousarray(words, dtype=np.int32).reshape(-1, 136)
    a = np.zeros(len(w), dtype=np.int32)
    lib.hl_ttc_value_iteration_batch(_p(w), ctypes.c_int(len(w)), ctypes.c_double(gamma), ctypes.c_int(int(iterations)), _p(a))
    return a
