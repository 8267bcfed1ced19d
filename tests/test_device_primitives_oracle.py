"""Pin the statements of the device's KL primitives (oracle/device_primitives.py) to the unmodified reference's answers
on the generated inputs of tests/device_primitive_cases.py, recorded in tests/golden/golden_device_primitives.json
(and to the max-expectation vectors of the MDP-GapE goldens), and check them against the 60-digit run of the same
Newton iterations: the branches each case takes, how far from a tie, and that the inputs reach every branch they are
there for.  The tables below are also the expected values of tests/test_gpu_device_primitives.py."""
import filecmp
import functools
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import device_primitives as dp
from oracle import ref_loader
from oracle.mdp_gape_stochastic import dot_fma
from tests import device_primitive_cases as cases
from tests.util import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
G = load_golden("golden_device_primitives.json")
X = float.fromhex


def same(a, b):
    return (math.isnan(a) and math.isnan(b)) or a == b and math.copysign(1, a) == math.copysign(1, b)


def same_vec(a, b):
    return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))


def _alternatives(run, args, decisions):
    """float64 answers of the other branch at each near tie of a 60-digit run."""
    return [run(dp.F64, *args, flip=k)[0] for k in dp.near_ties(decisions)]


@functools.lru_cache(None)
def kl_table():
    """[(p, q, answer)]: the float64 statement's bernoulli_kl, equal to the reference's (test below)."""
    return [(p, q, float(dp.bernoulli_kl(dp.F64, p, q))) for _, p, q in cases.kl_inputs()]


@functools.lru_cache(None)
def kl_bound_table():
    """[(tag, sum, count, threshold, lower, answer, 60-digit decisions, near-tie alternatives)]; answer is the float64
    statement's, equal to the reference's with a Python-float sum (test below)."""
    out = []
    for tag, s, n, thr, lower in cases.kl_bound_inputs():
        args = (s, n, thr, lower)
        _, dec = dp.kl_bound(dp.MP, *args)
        out.append((tag, s, n, thr, lower, dp.kl_bound(dp.F64, *args)[0], dec,
                    _alternatives(dp.kl_bound, args, dec)))
    return out


@functools.lru_cache(None)
def expectation_table():
    """[(tag, f, counts, c, p, 60-digit decisions, near-tie alternatives)] in the reference's order: the generated
    inputs with the float64 statement's p, then the vectors of golden_mdp_gape_stochastic.json whose p_hat comes from
    integer counts, with the reference's p."""
    rows = [(tag, f, counts, c, None) for tag, f, counts, c in cases.expectation_inputs()]
    for tag, f, q, c, p in load_golden("golden_mdp_gape_stochastic.json")["max_expectation_under_constraint"]:
        counts = counts_of(q)
        if counts is not None:
            rows.append(("stochastic_golden_" + tag, f, counts, c, p))
    out = []
    for tag, f, counts, c, p in rows:
        args = (f, cases.q_of(counts), c)
        _, dec = dp.max_expectation(dp.MP, *args)
        out.append((tag, f, counts, c, p if p is not None else dp.max_expectation(dp.F64, *args)[0], dec,
                    _alternatives(dp.max_expectation, args, dec)))
    return out


def counts_of(q):
    """Integer counts k with k / sum(k) == q bit for bit, or None."""
    q = np.asarray(q, dtype=np.float64)
    for total in range(1, 200):
        k = np.round(q * total)
        if k.sum() == total and np.array_equal(k / float(total), q):
            return [int(v) for v in k]
    return None


def float_type_cases():
    """{index into kl_bound_table(): (Python-float answer, np.float64 answer)} where the sum's float type matters."""
    return {i: (X(py), X(npf)) for i, py, npf in G["kl_bound"]["float_type"]}


@pytest.mark.skipif(not ref_loader.reference_available(), reason="needs the reference tree")
def test_golden_generator_reproduces_its_json(tmp_path):
    out = tmp_path / "golden.json"
    subprocess.run([sys.executable, os.path.join(GOLDEN, "make_golden_device_primitives.py"), "--out", str(out)],
                   check=True, cwd=ROOT, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    assert filecmp.cmp(str(out), os.path.join(GOLDEN, "golden_device_primitives.json"), shallow=False)


def test_kl_statement_equals_the_reference():
    answers = [a for _, _, a in kl_table()]
    assert (len(answers), cases.digest(answers)) == (G["kl"]["n"], G["kl"]["sha256"])


def test_kl_bound_statement_equals_the_python_float_reference_bit_for_bit():
    table = kl_bound_table()
    answers = [row[5] for row in table]
    assert (len(answers), cases.digest(answers)) == (G["kl_bound"]["n"], G["kl_bound"]["sha256"])
    rows = [row for row in table if row[0] != "random"]
    assert len(rows) == len(G["kl_bound"]["named"])
    for (tag, s, n, thr, lower, a), row in zip(G["kl_bound"]["named"], rows):
        assert (tag, n, lower) == (row[0], row[2], row[4]) and same(X(s), row[1]) and same(X(thr), row[3])
        assert same(X(a), row[5]), row[:5]
    for s, n, thr, ref in load_golden("golden_mdp_gape.json")["kl_lower_bound"]:
        assert same(dp.kl_bound(dp.F64, s, n, thr, True)[0], ref)


def test_kl_bound_float_type_cases():
    """Sum 5e-324, count 1, lower: 5e-324 through the finite difference with a Python float, 0.0 through -inf with an
    np.float64; the device follows the Python float, as the planners' sums are."""
    table = kl_bound_table()
    ft = float_type_cases()
    assert all(same(table[i][5], py) and not same(py, npf) for i, (py, npf) in ft.items())
    assert any(table[i][1:5] == (5e-324, 1, 1.0, True) and py == 5e-324 and npf == 0.0 for i, (py, npf) in ft.items())


def test_kl_bound_high_precision_run_agrees_off_the_near_ties():
    """Off the near ties the float64 statement takes the 60-digit run's branches and lands within 2^-46 of it."""
    for tag, s, n, thr, lower, py, dec, _ in kl_bound_table():
        if dp.near_ties(dec):
            continue
        hp = dp.kl_bound(dp.MP, s, n, thr, lower)[0]
        _, dec64 = dp.kl_bound(dp.F64, s, n, thr, lower)
        assert [d[:2] for d in dec64] == [d[:2] for d in dec], (tag, s, n, thr, lower)
        assert same(hp, py) or abs(hp - py) <= 2.0 ** -46, (tag, s, n, thr, lower, hp, py)


def test_expectation_statement_equals_the_reference_bit_for_bit():
    table = expectation_table()
    generated = [row[4] for row in table if not row[0].startswith("stochastic_golden_")]
    assert (len(generated), cases.digest(generated)) == (G["expectation"]["n"], G["expectation"]["sha256"])
    for tag, f, counts, c, p, _, _ in table:
        if tag.startswith("stochastic_golden_"):
            assert same_vec(dp.max_expectation(dp.F64, f, cases.q_of(counts), c)[0], p), (tag, f, counts, c)


def test_expectation_high_precision_run_agrees_off_the_near_ties():
    for tag, f, counts, c, p, dec, _ in expectation_table():
        if dp.near_ties(dec):
            continue
        hp, _ = dp.max_expectation(dp.MP, f, cases.q_of(counts), c)
        _, dec64 = dp.max_expectation(dp.F64, f, cases.q_of(counts), c)
        assert [d[:2] for d in dec64] == [d[:2] for d in dec], (tag, f, counts, c)
        scale = max([abs(v) for v in f if math.isfinite(v)] + [1.0])
        e_hp, e_64 = dot_fma(hp, f), dot_fma(p, f)
        # small c makes the solve ill-conditioned: float64 rounding alone moves the answer by ~1e-14 there
        assert same(e_hp, e_64) or abs(e_hp - e_64) <= 2.0 ** -40 * scale, (tag, e_hp, e_64)


def test_every_named_branch_is_reached():
    """Judged by the 60-digit run, so that the case lists cannot go stale."""
    kl = set()
    for row in kl_bound_table():
        kl |= dp.branches(row[6])
    for b in [("count0", True), ("a_eq_b", True), ("a_eq_b", False), ("fd", True), ("fd", False),
              ("pull_lo", True), ("pull_hi", True), ("clamp_lo", False), ("stop", False)]:
        assert b in kl, b
    # a first step of exactly eps (log-free: an infinite threshold pulls the step back): the stop test stops there
    ties = [row for row in kl_bound_table() if row[0] == "stop_tie"]
    assert ties and all(abs(row[1] / 2 - row[5]) == 1e-2 for row in ties)
    # No input of the lists reaches the 100-iteration cap: the damped step at least divides the distance to the
    # bound by ten, so |dx| falls below 1e-2 long before.
    assert ("cap", True) not in kl
    ex = {}
    for row in expectation_table():
        for b in dp.branches(row[5]):
            ex.setdefault(b, set()).add(row[0].split("_golden_")[-1])
    for b in [("unobserved_max", True), ("theta_star_neg", True), ("theta_star_neg", False), ("n_max_gt1", True),
              ("isclose", True), ("isclose", False), ("beta_zero", True), ("beta_zero", False), ("s1_zero", True),
              ("pull", True), ("stop", False)]:
        assert b in ex, b
    assert "isclose_at" in ex[("isclose", True)] and "isclose_below" in ex[("isclose", True)]
    assert "isclose_above" in ex[("isclose", False)] and "isclose_at" not in ex[("isclose", False)]
    assert "beta_zero_c_inf" in ex[("beta_zero", True)]
    # the lengths and observed counts the kernel layout has to handle: K = 2..15, n = 1..K, ties among the unobserved
    ks = {(len(row[2]), sum(k > 0 for k in row[2])) for row in expectation_table()}
    assert all((K, n) in ks for K in range(2, 16) for n in range(1, K + 1))
    assert {"moved_ties%d" % k for k in range(1, 15)} <= {row[0] for row in expectation_table()}
