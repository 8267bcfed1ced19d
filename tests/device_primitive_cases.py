"""The inputs on which the device's KL primitives are compared with the reference (tests/golden/
make_golden_device_primitives.py), the float64 statement (tests/test_device_primitives_oracle.py) and the device
(tests/test_gpu_device_primitives.py).  Generated from fixed seeds, so the golden only has to record the answers."""
import math

import numpy as np

TINY = 5e-324
ONE_MINUS = 1.0 - 2.0 ** -53


def kl_inputs():
    """[(tag, p, q)]: the edge grid of p in [0, 1] against every q, random pairs and pairs one ulp apart."""
    out = []
    edge = [0.0, TINY, 1e-300, 1e-17, 0.25, 0.5, ONE_MINUS, 1.0, -0.0, -0.5, 1.5, math.inf, -math.inf]
    for p in edge:
        for q in edge:
            if 0.0 <= p <= 1.0:
                out.append(["edge", p, q])
    rng = np.random.default_rng(31)
    for p, q in zip(rng.uniform(0, 1, 500), rng.uniform(0, 1, 500)):
        out.append(["random", float(p), float(q)])
    for p, q in zip(rng.uniform(0, 1, 200), rng.uniform(0, 1, 200)):
        out.append(["near", float(p), float(np.nextafter(p, rng.choice([-1.0, 2.0])))])
    return out


def kl_bound_inputs():
    """[(tag, sum, count, threshold, lower)]: the named edges on both sides, then 10^4 random pairs."""
    olop = float(4 * np.log(1e6))                             # OLOP's threshold at 10^6 episodes
    gape = float(3 * np.log(1 + np.log(1e6)) + 10 * np.log(4) + np.log(1 / (1 - 0.9)))
    trans = float(0.1 * np.log(1e6))
    cases = []
    for lower in (False, True):
        cases += [("count0", 0.0, 0, 1.0, lower), ("count0", 3.0, 0, olop, lower),
                  ("sum0", 0.0, 5, 2.0, lower), ("sum_eq_count", 5.0, 5, 2.0, lower),
                  ("mu_1_minus_ulp", ONE_MINUS, 1, 1.0, lower), ("mu_1_minus_ulp", ONE_MINUS * 3, 3, olop, lower),
                  ("mu_tiny", TINY, 1, 1.0, lower), ("mu_tiny", 1e-300, 1, 1.0, lower),
                  ("mu_tiny", TINY, 7, olop, lower), ("mu_tiny", 1e-300, 2 ** 31 - 1, olop, lower),
                  ("threshold0", 3.0, 7, 0.0, lower), ("threshold0", 0.5, 1, 0.0, lower),
                  ("threshold_inf", 3.0, 7, math.inf, lower),
                  ("olop", 0.5, 1, olop, lower), ("olop", 17.5, 40, olop, lower), ("gape", 3.25, 7, gape, lower),
                  ("gape_transition", 1.0, 3, trans, lower),
                  ("count_max", 2.0 ** 30 + 0.5, 2 ** 31 - 1, olop, lower), ("count_max", 0.5, 2 ** 31 - 1, olop, lower),
                  ("count_max", 2.0 ** 31 - 1.25, 2 ** 31 - 1, gape, lower)]
    cases += [("stop_tie", s, 1, math.inf, lower) for s, lower in stop_ties()]
    rng = np.random.default_rng(37)
    thresholds = [0.0, 1.0, olop, gape, trans, 1e-3, 50.0]
    for _ in range(10000):
        count = int(np.exp(rng.uniform(0, np.log(2 ** 31 - 1))))
        count = max(1, min(count, 2 ** 31 - 1))
        r = rng.uniform()
        s = float(rng.uniform(0, count)) if r < 0.8 else float(rng.integers(0, count + 1)) * (0.5 if r < 0.9 else 1)
        cases.append(("random", s, count, thresholds[int(rng.integers(0, len(thresholds)))], bool(rng.integers(0, 2))))
    return cases


def stop_ties():
    """Sums (count 1, lower bound) whose first step, at an infinite threshold (f = -inf, so the Newton step leaves
    [0, mu] and is pulled back to 0.1 x: no log is involved), moves by exactly eps = 1e-2, where the stop test
    |x - x_next| > eps says stop.  (On the upper side x >= 0.5, whose ulp does not divide 1e-2.)"""
    k = np.arange(-4000, 4000)
    x0 = np.nextafter(0.01 / 0.9, 1.0) + k * np.spacing(0.01 / 0.9)
    x1 = 0.9 * 0.0 + (1.0 - 0.9) * x0
    hits = np.flatnonzero(np.abs(x0 - x1) == 1e-2)
    return [(float(2.0 * x0[i]), True) for i in hits[:3]]


def isclose_edge(rng):
    """f0 and d with d = 1e-8 + 1e-5 * |f0| exactly equal to |(f0 + d) - f0| in float64."""
    f0 = rng.uniform(-3.0, 3.0, size=200000)
    tol = 1e-8 + 1e-5 * np.abs(f0)
    f1 = f0 + tol
    ok = np.abs(f1 - f0) == tol
    i = int(np.flatnonzero(ok)[0])
    return float(f0[i]), float(f1[i])


def expectation_inputs():
    """[(tag, f, counts, c)] in the reference's dict order (placeholders, count 0, first) for K = 2..15, n = 1..K."""
    rng = np.random.default_rng(41)
    f0e, f1e = isclose_edge(rng)
    out = []
    for K in range(2, 16):
        for n in range(1, K + 1):
            m = K - n                                      # unobserved placeholders, first in dict order
            def mk(f, counts, c, tag):
                out.append((tag, [float(v) for v in f], [int(v) for v in counts], float(c)))
            counts = rng.integers(1, 6, size=n)
            f_obs = rng.uniform(-2.0, 3.0, size=n)
            # Newton: the unobserved stay below the observed maximum
            mk(np.concatenate([f_obs.min() - rng.uniform(0, 2, m), f_obs]), np.r_[np.zeros(m), counts],
               rng.uniform(0.05, 1.5), "newton")
            mk(np.concatenate([f_obs.min() - rng.uniform(0, 2, m), f_obs]), np.r_[np.zeros(m), counts],
               rng.uniform(1e-4, 1e-2), "newton_small_c")
            mk(np.full(K, f_obs[0]), np.r_[np.zeros(m), counts], 0.3, "all_equal")
            if n >= 2:
                g = f_obs.copy()
                g[:] = f0e
                g[-1] = f1e
                for tag, last in (("isclose_at", f1e), ("isclose_below", float(np.nextafter(f1e, -np.inf))),
                                  ("isclose_above", float(np.nextafter(f1e, np.inf)))):
                    g[-1] = last
                    mk(np.concatenate([np.full(m, f0e - 1.0), g]), np.r_[np.zeros(m), counts], 0.4, tag)
                mk(np.concatenate([np.full(m, 1e308), -1e308 * (1 + 0.5 * np.arange(n) / n)]),
                   np.r_[np.zeros(m), counts], 0.5, "huge" if m else "huge_observed")
                g = f_obs.copy()
                g[0] = np.inf
                mk(np.concatenate([np.full(m, -np.inf), g]), np.r_[np.zeros(m), counts], 0.5, "inf_observed")
            if m >= 1:
                for n_max in range(1, m + 1):
                    top = f_obs.max() + rng.uniform(0.5, 2.0)
                    fu = np.full(m, f_obs.min() - 1.0)
                    fu[rng.permutation(m)[:n_max]] = top
                    mk(np.concatenate([fu, f_obs]), np.r_[np.zeros(m), counts], rng.uniform(1.0, 3.0),
                       "moved_ties%d" % n_max)
                fu = np.full(m, f_obs.max() + 1.0)
                mk(np.concatenate([fu, f_obs]), np.r_[np.zeros(m), counts], 800.0, "beta_zero")
                mk(np.concatenate([fu, f_obs]), np.r_[np.zeros(m), counts], np.inf, "beta_zero_c_inf")
                mk(np.concatenate([fu, f_obs]), np.r_[np.zeros(m), counts], 1e-3, "not_moved_small_c")
                fu[0] = np.inf
                mk(np.concatenate([fu, f_obs]), np.r_[np.zeros(m), counts], 0.5, "inf_unobserved")
    return out


def digest(answers):
    """sha256 of a list of answers (floats, or lists of floats), each written as float.hex: how the golden records the
    reference's answers on the generated inputs."""
    import hashlib
    lines = [",".join(float.hex(float(v)) for v in a) if isinstance(a, (list, tuple)) else float.hex(float(a))
             for a in answers]
    return hashlib.sha256("\n".join(lines).encode()).hexdigest()


def q_of(counts):
    """p_hat as the reference and the device form it: counts / their sum, in float64."""
    return (np.asarray(counts, dtype=np.float64) / float(sum(counts))).tolist()
