"""The device primitives the planners share, each run on its own through the b2_selftest_* entry points and compared
with numpy and with the unmodified reference's answers (the float64 statement of tests/test_device_primitives_oracle.py,
checked against tests/golden/golden_device_primitives.json here too):

  PCG64 (pcg64.cuh) and searchsorted_right / sampled_next (lane_env.cuh): bit for bit, every output and final words;
  bernoulli_kl: bit for bit where no log is evaluated, else within 4 ulp of |kl1| + |kl2|;
  kl_bound: bit for bit where no log is evaluated, NaN where the reference gives NaN, the Python-float answer on the
            cases where the sum's float type matters, else within 2^-44 (or equal to a near tie's other path);
  gape_expectation_kl: bit for bit on the isclose branch, else within 2^-44 * max|f| of p_ref @ values.

Each test prints the largest distance it finds in ulps."""
import math

import numpy as np
import pytest
import torch

from oracle.pcg64 import PCG64
from oracle.mdp_gape_stochastic import dot_fma
from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import sampled_mdp_tables
from tests.test_pcg64_skip import skip32
from oracle.device_primitives import isclose_all
from tests import device_primitive_cases as cases
from tests.test_device_primitives_oracle import (G, expectation_table, float_type_cases, kl_bound_table, kl_table,
                                                 same)
from tests.util import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
NEXT64, NEXT32, RANDOM, INTEGERS, SKIP32, SEED_FROM = range(6)
TOL = 2.0 ** -44


def t(a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def ulps(a, b):
    a, b = float(a), float(b)
    if same(a, b):
        return 0.0
    return abs(a - b) / math.ulp(max(abs(a), abs(b)))


def words_of(gen):
    return PCG64.from_numpy(gen).words()


def run_pcg64(words, ops, args):
    lib = _lib.load()
    n, k = ops.shape
    w = t(words.view(np.int64), torch.int64)
    o = t(ops, torch.int32)
    a = t(np.asarray(args, dtype=np.uint64).view(np.int64), torch.int64)
    out = torch.zeros((n, k), dtype=torch.int64, device=DEV)
    wo = torch.zeros((n, 6), dtype=torch.int64, device=DEV)
    _lib.check(lib.b2_selftest_pcg64(_lib.ptr(w), _lib.ptr(o), _lib.ptr(a), _lib.ptr(out), _lib.ptr(wo), n, k,
                                     _lib.current_stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint64), wo.cpu().numpy().view(np.uint64)


INTEGER_NS = [1, 2, 3, 5, 2 ** 30, 2 ** 31 + 1, 3 * 2 ** 30 + 1, 2 ** 32 - 1]
SKIPS = [0, 1, 2, 3, 2 ** 32 - 1, 2 ** 32 + 1, 2 ** 63, 2 ** 64 - 1]
SEEDS = [0, 1, 2 ** 30 - 1, 2 ** 31, 2 ** 32 - 1]


def test_pcg64_streams_match_numpy_bit_for_bit():
    """8192 streams, 24 ops each: next64 / random / integers(n) against numpy's Generator itself, integers with the
    buffer empty and full, next32 and skip32 against the oracle's PCG64 (numpy cannot set a half-buffered skip)."""
    rng = np.random.default_rng(2024)
    n_streams, n_ops = 8192, 24
    ops = np.zeros((n_streams, n_ops), np.int32)
    args = np.zeros((n_streams, n_ops), np.uint64)
    words = np.zeros((n_streams, 6), np.uint64)
    for s in range(n_streams):
        kind = s % 4
        words[s] = words_of(np.random.Generator(np.random.PCG64(int(rng.integers(2 ** 62)))))
        if s % 8 >= 4:                      # start with a buffered half
            g = PCG64.from_words(words[s])
            g.next32()
            words[s] = g.words()
        for i in range(n_ops):
            if kind == 0:
                ops[s, i] = (NEXT64, RANDOM, NEXT32)[i % 3]
            elif kind == 1:
                ops[s, i] = INTEGERS
                args[s, i] = INTEGER_NS[(s // 4 + i) % len(INTEGER_NS)] if i < 16 else int(rng.integers(1, 2 ** 32))
            elif kind == 2:
                ops[s, i] = (SKIP32, NEXT32)[i % 2]
                args[s, i] = SKIPS[(s // 4 + i) % len(SKIPS)] if i < 16 else int(rng.integers(0, 2 ** 64,
                                                                                               dtype=np.uint64))
            else:
                ops[s, i] = (SEED_FROM, NEXT64, INTEGERS)[i % 3]
                args[s, i] = (SEEDS[(s // 4 + i) % len(SEEDS)] if i < 15 else int(rng.integers(0, 2 ** 32))) \
                    if i % 3 == 0 else (0 if i % 3 == 1 else int(rng.integers(1, 2 ** 32)))
    out, wo = run_pcg64(words, ops, args)
    for s in range(n_streams):
        g = PCG64.from_words(words[s])
        for i in range(n_ops):
            op, a = int(ops[s, i]), int(args[s, i])
            if op == NEXT64:
                r = g.next64()
            elif op == NEXT32:
                r = g.next32()
            elif op == RANDOM:
                r = int(np.float64(g.random()).view(np.uint64))
            elif op == INTEGERS:
                r = g.integers(a)
            elif op == SKIP32:
                skip32(g, a)
                r = g.state & (2 ** 64 - 1)
            else:
                g = _seeded(a)
                r = g.state & (2 ** 64 - 1)
            assert int(out[s, i]) == r, (s, i, op, a)
        assert [int(v) for v in wo[s]] == [int(v) for v in g.words()], s


def _seeded(seed):
    return PCG64.from_numpy(np.random.default_rng(seed))


def test_integers_rejection_and_buffer_against_numpy():
    """integers(0, n) for the rejection-heavy n, buffer empty and full, against numpy's Generator; the 32-bit halves
    numpy consumed show that rejections happened."""
    ns = INTEGER_NS
    n_streams = 4096
    n_ops = 32
    rng = np.random.default_rng(7)
    seeds = rng.integers(0, 2 ** 62, size=n_streams)
    words = np.zeros((n_streams, 6), np.uint64)
    gens = []
    for s in range(n_streams):
        gen = np.random.Generator(np.random.PCG64(int(seeds[s])))
        if s % 2:
            gen.integers(0, 3)              # leaves a buffered half
        words[s] = words_of(gen)
        gens.append(gen)
    ops = np.full((n_streams, n_ops), INTEGERS, np.int32)
    args = np.array([[ns[(s + i) % len(ns)] for i in range(n_ops)] for s in range(n_streams)], np.uint64)
    out, wo = run_pcg64(words, ops, args)
    halves, calls = 0, 0
    for s in range(n_streams):
        gen = gens[s]
        for i in range(n_ops):
            n = int(args[s, i])
            b0 = _numpy_halves(gen)
            assert int(out[s, i]) == int(gen.integers(0, n)), (s, i, n)
            if n > 1:
                halves += _numpy_halves(gen) - b0
                calls += 1
            else:
                assert _numpy_halves(gen) == b0
        assert [int(v) for v in wo[s]] == [int(v) for v in words_of(gen)]
    print("integers: %d calls, %d 32-bit halves" % (calls, halves))
    assert halves > calls


def _numpy_halves(gen):
    st = gen.bit_generator.state
    _numpy_halves.ref = getattr(_numpy_halves, "ref", {})
    key = st["state"]["inc"]
    base = _numpy_halves.ref.setdefault(key, (st["state"]["state"], 0))
    # advance a copy until it reaches the current state
    from oracle.pcg64 import MASK128, PCG_MULT
    s0, k = base
    while s0 != st["state"]["state"]:
        s0 = (s0 * PCG_MULT + st["state"]["inc"]) & MASK128
        k += 1
    _numpy_halves.ref[key] = (s0, k)
    return 2 * k - st["has_uint32"]


def test_seed_from_matches_default_rng():
    seeds = SEEDS + [int(v) for v in np.random.default_rng(3).integers(0, 2 ** 32, size=4091)]
    n = len(seeds)
    words = np.zeros((n, 6), np.uint64)
    words[:, 4] = 1
    words[:, 5] = 12345
    ops = np.full((n, 2), SEED_FROM, np.int32)
    ops[:, 1] = RANDOM
    args = np.zeros((n, 2), np.uint64)
    args[:, 0] = seeds
    out, wo = run_pcg64(words, ops, args)
    for s, seed in enumerate(seeds):
        gen = np.random.default_rng(seed)
        assert int(out[s, 1]) == int(np.float64(gen.random()).view(np.uint64)), seed
        assert [int(v) for v in wo[s]] == [int(v) for v in words_of(gen)], seed


def test_skip32_matches_numpy_advance():
    """skip32(n) with the buffer empty and full equals n next32() calls: numpy's PCG64.advance for the whole steps."""
    rng = np.random.default_rng(5)
    ns = SKIPS + [int(v) for v in rng.integers(0, 2 ** 64, size=24, dtype=np.uint64)]
    runs = [(n, buffered, int(rng.integers(2 ** 62))) for n in ns for buffered in (0, 1) for _ in range(64)]
    words = np.zeros((len(runs), 6), np.uint64)
    for s, (n, buffered, seed) in enumerate(runs):
        g = PCG64.from_numpy(np.random.Generator(np.random.PCG64(seed)))
        if buffered:
            g.next32()
        words[s] = g.words()
    ops = np.tile(np.array([[SKIP32, NEXT32, NEXT64]], np.int32), (len(runs), 1))
    args = np.zeros((len(runs), 3), np.uint64)
    args[:, 0] = [r[0] for r in runs]
    out, wo = run_pcg64(words, ops, args)
    for s, (n, buffered, seed) in enumerate(runs):
        g = PCG64.from_words(words[s])
        m = n
        if buffered and m:
            g.has_uint32, m = 0, m - 1
        if m:
            bg = np.random.PCG64()
            st = bg.state
            st["state"]["state"], st["state"]["inc"], st["has_uint32"], st["uinteger"] = g.state, g.inc, 0, 0
            bg.state = st
            bg.advance((m - 1) // 2)
            g = PCG64.from_words(words_of(np.random.Generator(bg)))
            g.next32()
            if m % 2 == 0:
                g.next32()
        assert int(out[s, 0]) == g.state & (2 ** 64 - 1), (n, buffered)
        assert int(out[s, 1]) == g.next32() and int(out[s, 2]) == g.next64(), (n, buffered)
        assert [int(v) for v in wo[s]] == [int(v) for v in g.words()], (n, buffered)


def run_searchsorted(cdf, u, rows):
    lib = _lib.load()
    c = t(cdf, torch.float64)
    uu = t(u, torch.float64)
    r = t(rows, torch.int32)
    k = torch.zeros(len(u), dtype=torch.int32, device=DEV)
    _lib.check(lib.b2_selftest_sampled_next(_lib.ptr(c), cdf.shape[1], _lib.ptr(uu), _lib.ptr(r), len(u), _lib.ptr(k),
                                            None, None, None, None, 0, None, None, _lib.current_stream()))
    torch.cuda.synchronize()
    return k.cpu().numpy()


def test_searchsorted_right_on_edges():
    rng = np.random.default_rng(11)
    for B in (1, 2, 7, 4096, 2 ** 16 + 1):
        rows = []
        p = rng.uniform(size=(4, B))
        if B > 1:
            p[1, ::3] = 0.0                             # zero-probability next states: repeated cdf entries
            p[2, : B // 2] = 0.0
        p[3] = 1.0
        cdf = p.cumsum(axis=1)
        cdf /= cdf[:, -1:]
        us, rs = [], []
        for r in range(4):
            picks = cdf[r, rng.integers(0, B, size=min(B, 200))]
            for u in list(picks) + [0.0, 1.0 - 2.0 ** -53, 1.0] + list(rng.uniform(size=50)):
                for v in (u, np.nextafter(u, -1.0), np.nextafter(u, 2.0)):
                    if 0.0 <= v < 1.0:
                        us.append(float(v))
                        rs.append(r)
        k = run_searchsorted(cdf, np.array(us), np.array(rs))
        want = [int(np.searchsorted(cdf[r], u, side="right")) for u, r in zip(us, rs)]
        assert k.tolist() == want, B


def test_sampled_next_on_built_tables():
    from types import SimpleNamespace
    lib = _lib.load()
    rng = np.random.default_rng(13)
    S, A, B = 40, 3, 5
    p = rng.uniform(size=(S, A, B))
    p[p < 0.3] = 0.0
    p[:, :, 0] += 0.01
    p /= p.sum(axis=-1, keepdims=True)
    mdp = SimpleNamespace(mode="sparse", transition=p, next=rng.integers(0, S, size=(S, A, B)),
                          reward=rng.uniform(size=(S, A)))
    tab = sampled_mdp_tables(mdp)
    dev = {k: t(v, {np.float64: torch.float64, np.int32: torch.int32, np.uint8: torch.uint8}[v.dtype.type])
           for k, v in tab.items()}
    m = _lib.FiniteMDPSampled(S, A, B, 0, dev["cdf"].data_ptr(), dev["next"].data_ptr(), dev["reward"].data_ptr(),
                              dev["row_ok"].data_ptr())
    n = 4096
    rows = rng.integers(0, S * A, size=n)
    draw = (np.arange(n) % 3 != 0).astype(np.int32)
    words = np.stack([words_of(np.random.default_rng(int(s))) for s in rng.integers(0, 2 ** 30, size=n)])
    w = t(words.view(np.int64), torch.int64)
    rows_d, draw_d = t(rows, torch.int64), t(draw, torch.int32)          # kept alive until the launch has run
    nxt = torch.zeros(n, dtype=torch.int32, device=DEV)
    wo = torch.zeros((n, 6), dtype=torch.int64, device=DEV)
    assert rows.min() >= 0 and rows.max() < S * A
    _lib.check(lib.b2_selftest_sampled_next(None, 0, None, None, 0, None, m, _lib.ptr(rows_d), _lib.ptr(draw_d),
                                            _lib.ptr(w), n, _lib.ptr(nxt), _lib.ptr(wo), _lib.current_stream()))
    torch.cuda.synchronize()
    nxt, wo = nxt.cpu().numpy(), wo.cpu().numpy().view(np.uint64)
    for i in range(n):
        g = PCG64.from_words(words[i])
        flat_p = p.reshape(-1, B)[rows[i]]
        if draw[i]:
            gen = np.random.Generator(np.random.PCG64())
            g.to_numpy(gen)
            k = int(gen.choice(B, p=flat_p))          # Generator.choice itself
            g = PCG64.from_numpy(gen)
        else:
            k = 0
        assert nxt[i] == tab["next"].reshape(-1, B)[rows[i], k], i
        assert [int(v) for v in wo[i]] == [int(v) for v in g.words()], i


def run_kl(p, q, s, n, thr, lower):
    lib = _lib.load()
    args = [t(p, torch.float64), t(q, torch.float64), t(s, torch.float64), t(n, torch.int32), t(thr, torch.float64),
            t(lower, torch.int32)]
    kl = torch.zeros(len(p), dtype=torch.float64, device=DEV)
    bound = torch.zeros(len(s), dtype=torch.float64, device=DEV)
    _lib.check(lib.b2_selftest_kl(_lib.ptr(args[0]), _lib.ptr(args[1]), len(p), _lib.ptr(kl), _lib.ptr(args[2]),
                                  _lib.ptr(args[3]), _lib.ptr(args[4]), _lib.ptr(args[5]), len(s), _lib.ptr(bound),
                                  _lib.current_stream()))
    torch.cuda.synchronize()
    return kl.cpu().numpy(), bound.cpu().numpy()


def _kl_terms(p, q):
    with np.errstate(all="ignore"):
        kl1 = p * float(np.log(p / q)) if p > 0 and q > 0 else 0.0
        kl2 = (1 - p) * float(np.log((1 - p) / (1 - q))) if q < 1 and p < 1 else 0.0
    logs = (p > 0 and q > 0, q < 1 and p < 1)
    return abs(kl1) + abs(kl2), logs


def test_bernoulli_kl_against_the_reference():
    table = kl_table()
    assert cases.digest([r for _, _, r in table]) == G["kl"]["sha256"]       # the expected values are the reference's
    ps, qs = [p for p, _, _ in table], [q for _, q, _ in table]
    kl, _ = run_kl(ps, qs, [0.0], [1], [1.0], [0])
    worst = 0.0
    for (p, q, r), d in zip(table, kl):
        mag, logs = _kl_terms(p, q)
        exact_args = [p / q if logs[0] else 1.0, (1 - p) / (1 - q) if logs[1] else 1.0]
        if not math.isfinite(r) or all(a in (0.0, 1.0) or not math.isfinite(a)
                                       for a, log in zip(exact_args, logs) if log):
            assert same(float(d), r), (p, q, d, r)                      # no log, or log of 0, 1 or inf
        else:
            err = abs(float(d) - r)
            assert err <= 4 * math.ulp(mag), (p, q, d, r)
            worst = max(worst, err / math.ulp(mag))
    print("bernoulli_kl: largest distance %.2f ulp of |kl1| + |kl2|" % worst)


def test_kl_bound_against_the_reference():
    table = kl_bound_table()
    assert cases.digest([row[5] for row in table]) == G["kl_bound"]["sha256"]
    float_type = float_type_cases()
    _, got = run_kl([0.5], [0.5], [r[1] for r in table], [r[2] for r in table], [r[3] for r in table],
                    [int(r[4]) for r in table])
    worst = 0.0
    for i, ((tag, s, n, thr, lower, py, _, alt), d) in enumerate(zip(table, got)):
        d = float(d)
        if n == 0 or (0.0 if lower else s / n) == (s / n if lower else 1.0) or i in float_type:
            assert same(d, py), (tag, s, n, thr, lower, d, py)           # no log, or the float-type edge
        elif math.isnan(py):
            assert math.isnan(d), (tag, s, n, thr, lower, d)
        elif alt:
            assert any(abs(d - a) <= TOL for a in [py] + alt), (tag, s, n, thr, lower, d, py, alt)
        else:
            assert abs(d - py) <= TOL, (tag, s, n, thr, lower, d, py)
            worst = max(worst, ulps(d, py))
    print("kl_bound: largest distance %.0f ulp off the near ties" % worst)


def run_expectation(cases):
    """cases: [(f, counts, c, qp or None)] in the reference's order; -> out [n, 2] (upper, lower).  The kernel layout
    puts the observed children (count > 0) first, in order, then the placeholders; its dict order is the reverse
    grouping, which dict_order() gives."""
    lib = _lib.load()
    max_k = max(len(c[0]) for c in cases)
    n_cases = len(cases)
    F = np.zeros((n_cases, max_k))
    C = np.zeros((n_cases, max_k), np.int32)
    K, N, CNT, QP, CC = [], [], [], [], []
    for i, (f, counts, c, qp) in enumerate(cases):
        obs = [j for j in range(len(f)) if counts[j] > 0]
        free = [j for j in range(len(f)) if counts[j] == 0]
        order = obs + free
        F[i, :len(f)] = [f[j] for j in order]
        C[i, :len(f)] = [counts[j] for j in order]
        K.append(len(f))
        N.append(0 if qp is not None else len(obs))
        CNT.append(int(sum(counts)))
        QP.append(qp if qp is not None else 0.0)
        CC.append(c)
    f = t(F, torch.float64)
    neg = t(-F, torch.float64)
    cnt = t(C, torch.int32)
    zeros = torch.zeros_like(f)
    out = torch.zeros((n_cases, 2), dtype=torch.float64, device=DEV)
    ins = [t(K, torch.int32), t(N, torch.int32), t(CNT, torch.int32), t(QP, torch.float64), t(CC, torch.float64)]
    _lib.check(lib.b2_selftest_gape_expectation(_lib.ptr(f), _lib.ptr(neg), _lib.ptr(cnt), _lib.ptr(zeros), max_k,
                                                *[_lib.ptr(x) for x in ins], n_cases, _lib.ptr(out),
                                                _lib.current_stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def dict_order(v, counts):
    return [v[j] for j in range(len(v)) if counts[j] == 0] + [v[j] for j in range(len(v)) if counts[j] > 0]


def test_gape_expectation_kl_against_the_reference():
    table = expectation_table()
    assert cases.digest([row[4] for row in table if not row[0].startswith("stochastic_golden_")]) == \
        G["expectation"]["sha256"]
    out = run_expectation([(f, counts, c, None) for _, f, counts, c, _, _, _ in table])
    worst = 0.0
    for (tag, f, counts, c, p, _, alt), (up, lo) in zip(table, out):
        vals = dict_order(f, counts)
        scale = max([abs(v) for v in f if math.isfinite(v)] + [1e-300])
        f_p = [f[j] for j in range(len(f)) if counts[j] > 0]
        f_star_moved = max(f) > max(f_p)
        for side, got in ((1.0, up), (-1.0, lo)):
            sv = [side * v for v in vals]
            want = dot_fma(dict_order(p, counts), sv)
            candidates = [want] + [dot_fma(dict_order(a, counts), sv) for a in alt]
            if (isclose_all(f_p) and not f_star_moved) or not math.isfinite(want):
                assert same(float(got), want), (tag, side, got, want)
            else:
                assert any(abs(float(got) - w) <= TOL * scale for w in candidates), (tag, f, counts, c, side, got,
                                                                                      want)
                if not alt:
                    worst = max(worst, abs(float(got) - want) / (TOL * scale))
    print("gape_expectation_kl: largest distance %.3g of the 2^-44 * max|f| tolerance" % worst)


def test_gape_expectation_one_positive():
    vecs = load_golden("golden_mdp_gape.json")["max_expectation_one_positive"]
    cases = []
    for f, q, c, p in vecs:
        counts = [1 if v > 0 else 0 for v in q]
        cases.append((f, counts, c, float(max(q))))
    out = run_expectation(cases)
    for (f, q, c, p), (up, lo) in zip(vecs, out):
        counts = [1 if v > 0 else 0 for v in q]
        scale = max([abs(v) for v in f if math.isfinite(v)] + [1e-300])
        for side, got in ((1.0, up), (-1.0, lo)):
            want = dot_fma(dict_order(p, counts), [side * v for v in dict_order(f, counts)])
            assert same(float(got), want) or abs(float(got) - want) <= TOL * scale, (f, q, c, side, got, want)
