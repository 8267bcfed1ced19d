"""ctypes wrapper of the C statement of MCTS on IntersectionLite (oracle/c/mcts_intersection.c) -- TEST
INFRASTRUCTURE.  Pinned bit-exactly against oracle/planners.py::mcts_plan on oracle.intersection.IntersectionLite
(tests/test_intersection_planners_oracle.py), so full-size trees can be checked on the GPU without the Python
oracle's cost.  Built on its own with the flags of oracle/c/Makefile, beside liboracle_c.so."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "c")
LIB = os.path.join(HERE, "libmcts_intersection.so")
SOURCES = ("highway_lite.c", "intersection_lite.c", "mcts_intersection.c")   # IntersectionLite shares sin_p / cos_p
CFLAGS = ["-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-std=c11", "-Wall"]
_lib = None


def build(force=False):
    deps = [os.path.join(HERE, f) for f in SOURCES + ("highway_lite.h", "intersection_lite.h")]
    if force or not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in deps):
        subprocess.run([os.environ.get("CC", "gcc")] + CFLAGS + ["-o", LIB] + [os.path.join(HERE, f) for f in SOURCES]
                       + ["-lm"], check=True)
    return LIB


def load():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(LIB)
        _lib.mcts_intersection_plan.restype = ctypes.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def mcts_intersection_plan(root_words, episodes, horizon, gamma, temperature, rng_words):
    """MCTS with the random_available policies from one IntersectionLite scene.  rng_words: uint64[6] numpy PCG64
    state (an advanced copy is returned).  -> (tree dict: parent, action, count, first_child, n_children, value, prior
    in creation order, plus env_steps; rng_words)."""
    lib = load()
    cap = 1 + int(episodes) * 3
    i32 = {k: np.zeros(cap, dtype=np.int32) for k in ("parent", "action", "count", "first_child", "n_children")}
    f64 = {k: np.zeros(cap, dtype=np.float64) for k in ("value", "prior")}
    cdf = np.ones((4, 3), dtype=np.float64)
    for n in range(1, 4):
        c = (np.ones(n) / n).cumsum()
        c /= c[-1]
        cdf[n, :n] = c
    words = np.ascontiguousarray(rng_words, dtype=np.uint64).copy()
    root = np.ascontiguousarray(root_words, dtype=np.int32)
    assert root.shape == (136,)
    steps = ctypes.c_int64(0)
    n = lib.mcts_intersection_plan(_p(root), ctypes.c_int(int(episodes)), ctypes.c_int(int(horizon)),
                                   ctypes.c_double(gamma), ctypes.c_double(temperature), _p(words), _p(cdf),
                                   _p(i32["parent"]), _p(i32["action"]), _p(i32["count"]), _p(i32["first_child"]),
                                   _p(i32["n_children"]), _p(f64["value"]), _p(f64["prior"]), ctypes.byref(steps))
    out = {k: v[:n] for k, v in {**i32, **f64}.items()}
    out["env_steps"] = steps.value
    return out, words
