"""The Newton solves of the device's KL primitives, stated once over two arithmetics -- TEST INFRASTRUCTURE.

  kl_bound(sum, count, threshold, lower)    kl_bound.cuh::kl_bound (rl_agents/utils.py:123-203)
  max_expectation(f, q, c)                  mdp_gape.cu::gape_expectation_kl (utils.py:279-342)

F64 runs them in float64 as the device does, with the host's functions the reference calls (numpy's log in the
Bernoulli KL and exp in the expectation, libm's log inside the numba-compiled theta), dot products as fma chains and
the finite difference wherever the device takes it; MP runs the same steps at 60 significant digits.  Both record every decision the
iteration takes -- (name, outcome, margin) -- so that a test can see which branches a case reaches and how close it
came to taking the other one.

Only log and exp can differ between the device and the host (CUDA's and glibc's are both within 1 ulp, not equal), so
MP starts from the same float64 inputs and rounds what comes before the first log as float64 does: mu, the threshold
over count, the interval, the first Newton point, and the isclose test of the observed values.  A decision whose
operands come from a log gets the margin |u - v| / max(|u|, |v|, scale), scale the size of the terms that make u up;
any other decision is exact (margin inf).  A margin below NEAR_TIE is a near tie: a one-ulp log may take either
branch there, and `flip` re-runs a case with one decision reversed to get the other path's answer.
"""
import math

import mpmath
import numpy as np

from oracle.mdp_gape_stochastic import fma

NEAR_TIE = 1e-12
EPS = 1e-2
WEIGHT = 0.9
MP_DPS = 60


class F64(object):
    @staticmethod
    def num(x):
        return float(x)

    @staticmethod
    def log(x):
        if math.isnan(x) or x < 0:
            return math.nan
        if x == 0:
            return -math.inf
        return math.log(x) if x != math.inf else math.inf

    @staticmethod
    def np_log(x):
        with np.errstate(all="ignore"):
            return float(np.log(np.float64(x)))

    @staticmethod
    def exp(x):
        with np.errstate(all="ignore"):
            return float(np.exp(np.float64(x)))

    @staticmethod
    def div(a, b):
        with np.errstate(all="ignore"):
            return float(np.float64(a) / np.float64(b))

    @staticmethod
    def fma(a, b, c):
        return fma(a, b, c)

    @staticmethod
    def sub(a, b):
        return a - b

    @staticmethod
    def f64(x):
        return float(x)


class MP(object):
    ctx = mpmath.MPContext()
    ctx.dps = MP_DPS

    @classmethod
    def num(cls, x):
        return cls.ctx.mpf(x)

    @classmethod
    def log(cls, x):
        if cls.ctx.isnan(x) or x < 0:
            return cls.ctx.nan
        if x == 0:
            return cls.ctx.ninf
        return cls.ctx.log(x)

    @classmethod
    def np_log(cls, x):
        return cls.log(x)

    @classmethod
    def exp(cls, x):
        if cls.ctx.isnan(x):
            return cls.ctx.nan
        return cls.ctx.exp(x)

    @classmethod
    def div(cls, a, b):
        if b == 0:
            if cls.ctx.isnan(a) or a == 0:
                return cls.ctx.nan
            return cls.ctx.inf if a > 0 else cls.ctx.ninf
        return a / b

    @classmethod
    def fma(cls, a, b, c):
        return a * b + c

    @classmethod
    def sub(cls, a, b):
        """a - b, overflowing to inf past float64's range as float64 does."""
        d = a - b
        if cls.ctx.isfinite(d) and abs(d) > 1.7976931348623157e308:
            return cls.ctx.inf if d > 0 else cls.ctx.ninf
        return d

    @staticmethod
    def f64(x):
        return float(x)


def _margin(ops, u, v, scale=0.0):
    u, v = ops.f64(u), ops.f64(v)
    if not (math.isfinite(u) and math.isfinite(v)):
        return math.inf
    den = max(abs(u), abs(v), abs(float(scale)))
    return abs(u - v) / den if den > 0 else math.inf


class _Trace(object):
    def __init__(self, ops, flip):
        self.ops, self.flip, self.decisions = ops, flip, []

    def take(self, name, outcome, margin=math.inf):
        """Record a decision; the `flip`-th one (counted from 0) goes the other way."""
        if len(self.decisions) == self.flip:
            outcome = not outcome
        self.decisions.append((name, bool(outcome), margin))
        return outcome


def bernoulli_kl(ops, p, q):
    """kl_bound.cuh::bernoulli_kl (utils.py:89-106) in ops' arithmetic."""
    kl1, kl2 = ops.num(0.0), ops.num(math.inf)
    if p > 0 and q > 0:
        kl1 = p * ops.np_log(ops.div(p, q))
    if q < 1:
        kl2 = (1 - p) * ops.np_log(ops.div(1 - p, 1 - q)) if p < 1 else ops.num(0.0)
    return kl1 + kl2


def kl_bound(ops, _sum, count, threshold, lower, flip=None):
    """-> (bound as float, decisions).  kl_bound.cuh::kl_bound step by step; mu, the interval and the first Newton
    point are float64 in both arithmetics."""
    t = _Trace(ops, flip)
    if count == 0:
        t.take("count0", True)
        return (0.0 if lower else 1.0), t.decisions
    mu64 = float(_sum) / float(count)
    max_div = ops.num(float(threshold) / float(count))
    a64, b64 = (0.0, mu64) if lower else (mu64, 1.0)
    if t.take("a_eq_b", a64 == b64):
        return a64, t.decisions
    mu, a, b = ops.num(mu64), ops.num(a64), ops.num(b64)
    x, x_next = ops.num(math.inf), ops.num((a64 + b64) / 2.0)
    exact, x_scale = True, 0.0          # x_next is a float64 value no log has touched (the midpoint, its pull-backs)
    it = 0
    while True:
        if exact:                       # x too: float64 values, compared as float64 compares them
            dx = ops.num(abs(ops.f64(x) - ops.f64(x_next)))
        else:
            dx = abs(x - x_next)
        go = dx > EPS
        if it == 0 or exact:
            go = t.take("stop", go)
        else:
            go = t.take("stop", go, _margin(ops, dx, EPS, max(abs(ops.f64(x)), abs(ops.f64(x_next)))))
        if not go:
            break
        if t.take("cap", it >= 100):
            break
        it += 1
        x = x_next
        f_x = bernoulli_kl(ops, mu, x) - max_div
        at_edge = x == 0 or x == 1
        m = math.inf if exact else min(_margin(ops, x, 0.0, x_scale), _margin(ops, x, 1.0))
        if t.take("fd", at_edge, m):
            df_x = ops.div(f_x - (bernoulli_kl(ops, mu, x - EPS) - max_div), EPS)
        else:
            df_x = ops.div(1 - mu, 1 - x) - ops.div(mu, x)
        x_exact, x_scale = exact, abs(ops.f64(x))
        if df_x != 0:
            x_next = x - ops.div(f_x, df_x)
        exact = False
        scale = abs(ops.f64(x))
        # a pull-back reads x and the interval only: from a float64 x it is float64 arithmetic on both sides
        if t.take("pull_lo", x_next < a, _margin(ops, x_next, a, scale)):
            x_next = ops.num(WEIGHT * a64 + (1 - WEIGHT) * ops.f64(x)) if x_exact else WEIGHT * a + (1 - WEIGHT) * x
            exact = x_exact
        elif t.take("pull_hi", x_next > b, _margin(ops, x_next, b, scale)):
            x_next = ops.num(WEIGHT * b64 + (1 - WEIGHT) * ops.f64(x)) if x_exact else WEIGHT * b + (1 - WEIGHT) * x
            exact = x_exact
    scale = abs(ops.f64(x))
    if t.take("clamp_lo", x_next < a, math.inf if exact else _margin(ops, x_next, a, scale)):
        x_next = a
    if t.take("clamp_hi", x_next > b, math.inf if exact else _margin(ops, x_next, b, scale)):
        x_next = b
    return ops.f64(x_next), t.decisions


def isclose_all(f_p):
    """np.isclose(f_p, f_p[0]).all() in float64, as the device writes it."""
    f0 = f_p[0]
    return all((abs(fi - f0) <= 1e-8 + 1e-5 * abs(f0) and math.isfinite(f0)) or fi == f0 for fi in f_p[1:])


def max_expectation(ops, f, q, c, flip=None):
    """-> (p as float64 list, decisions).  gape_expectation_kl's p for values f (float64) and p_hat q (float64, from
    integer counts, at least one positive), in the order given."""
    t = _Trace(ops, flip)
    f64 = [float(v) for v in f]
    plus = [i for i in range(len(q)) if q[i] > 0]
    zero = [i for i in range(len(q)) if q[i] == 0]
    f_p64 = [f64[i] for i in plus]
    fp_max = max(f_p64)
    f_star64 = max(f64)
    qp = [ops.num(q[i]) for i in plus]
    fp = [ops.num(v) for v in f_p64]
    c = ops.num(c)

    def theta(l):
        s1, s2, scale = ops.num(0.0), ops.num(0.0), 0.0
        for qi, fi in zip(qp, fp):
            lg = ops.log(ops.sub(l, fi))
            s1 = ops.fma(qi, lg, s1)
            s2 = ops.fma(qi, ops.div(1, ops.sub(l, fi)), s2)
            scale += abs(ops.f64(qi * lg)) if ops.f64(lg) == ops.f64(lg) else 0.0
        lg2 = ops.log(s2)
        val = s1 + lg2 - c
        return val, scale + abs(ops.f64(lg2)) + abs(ops.f64(c))

    f_star = ops.num(f_star64)
    lam, z, moved, solved, n_max, share = None, ops.num(0.0), False, False, 0, ops.num(0.0)
    if t.take("unobserved_max", f_star64 > fp_max):
        th, sc = theta(f_star)
        if t.take("theta_star_neg", th < 0, _margin(ops, th, 0.0, sc)):
            moved = solved = True
            lam = f_star
            z = 1 - ops.exp(th)
            n_max = sum(f64[i] == f_star64 for i in zero)
            t.take("n_max_gt1", n_max > 1)
            share = ops.div(z, n_max)
    close = False
    if not solved:
        close = t.take("isclose", isclose_all(f_p64))
    if not solved and not close:
        x, x_next = ops.num(math.inf), f_star + 1
        it = 0
        while True:
            dx = abs(x - x_next)
            go = dx > EPS
            if it == 0:
                go = t.take("stop", go, math.inf)
            else:
                go = t.take("stop", go, _margin(ops, dx, EPS, max(abs(ops.f64(x)), abs(ops.f64(x_next)))))
            if not go or t.take("cap", it >= 100):
                break
            it += 1
            x = x_next
            f_x, _ = theta(x)
            s1, s2 = ops.num(0.0), ops.num(0.0)
            for qi, fi in zip(qp, fp):
                inv = ops.div(1, ops.sub(x, fi))
                s1 = ops.fma(qi, inv, s1)
                s2 = ops.fma(qi, inv * inv, s2)
            if t.take("s1_zero", s1 == 0, _margin(ops, s1, 0.0) if ops.f64(s1) == 0 and s1 != 0 else math.inf):
                df_x = ops.div(f_x - theta(x - EPS)[0], EPS)
            else:
                df_x = s1 - ops.div(s2, s1)
            if df_x != 0:
                x_next = x - ops.div(f_x, df_x)
            if t.take("pull", x_next < f_star, _margin(ops, x_next, f_star, abs(ops.f64(x)))):
                x_next = WEIGHT * f_star + (1 - WEIGHT) * x
        lam = f_star if x_next < f_star else x_next
    p = [ops.num(0.0)] * len(f64)
    for i in zero:
        if moved and f64[i] == f_star64:
            p[i] = share
    if close:
        for i in plus:
            p[i] = ops.num(q[i])
    else:
        sb = ops.num(0.0)
        for qi, fi in zip(qp, fp):
            sb = ops.fma(qi, ops.div(1, ops.sub(lam, fi)), sb)
        beta = ops.div(1 - z, sb)
        # moved: beta is 0 when 1 - z = exp(theta(f*)) rounds to 0, a near tie unless theta(f*) is -inf
        m = _margin(ops, 1 - z, 0.0, 1.0) if moved and th != -math.inf else math.inf
        if t.take("beta_zero", beta == 0, m):
            n_uni = sum(f64[i] == f_star64 for i in plus)
            for i in plus:
                p[i] = ops.div(1 - z, n_uni) if f64[i] == f_star64 else ops.num(0.0)
        else:
            for k, i in enumerate(plus):
                p[i] = ops.div(beta * qp[k], ops.sub(lam, fp[k]))
    return [ops.f64(v) for v in p], t.decisions


def near_ties(decisions):
    """Indices of the decisions taken within NEAR_TIE of the other branch."""
    return [k for k, (_, _, m) in enumerate(decisions) if m < NEAR_TIE]


def branches(decisions):
    """The set of (name, outcome) a run reached."""
    return {(n, o) for n, o, _ in decisions}
