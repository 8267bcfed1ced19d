"""skip32, the CPU twin of Pcg64::skip32 in csrc/pcg64.cuh, which the level-synchronous sparse-sampling kernel uses to
place the planner's stream after all the samples of a search, pinned here: the jump against numpy's own PCG64.advance,
and the buffered-half bookkeeping against n calls of next32() of the oracle's PCG64 (oracle/pcg64.py)."""
import numpy as np

from oracle.pcg64 import MASK128, PCG_MULT, PCG64


def advance_lcg128(state, delta, mult, plus):
    """pcg_advance_lcg_128: state after `delta` steps of state * mult + plus (mod 2^128), by square-and-multiply."""
    acc_mult, acc_plus = 1, 0
    while delta > 0:
        if delta & 1:
            acc_mult = (acc_mult * mult) & MASK128
            acc_plus = (acc_plus * mult + plus) & MASK128
        plus = ((mult + 1) * plus) & MASK128
        mult = (mult * mult) & MASK128
        delta >>= 1
    return (acc_mult * state + acc_plus) & MASK128


def skip32(g, n):
    """Leave the PCG64 `g` as n next32() calls would: the buffered half first; then, for the m >= 1 halves left,
    floor((m - 1) / 2) LCG steps (pcg_advance_lcg_128) and the last next64() as next32() runs it -- once when m is odd
    (its high half stays buffered), twice when m is even (`uinteger` keeps that step's high half)."""
    n = int(n)
    if n and g.has_uint32:
        g.has_uint32 = 0
        n -= 1
    if n == 0:
        return
    g.state = advance_lcg128(g.state, (n - 1) >> 1, PCG_MULT, g.inc)
    g.next32()
    if not n & 1:
        g.next32()


def numpy_state(k, seed=12345):
    bg = np.random.PCG64(seed)
    bg.advance(k)
    return bg.state["state"]["state"]


def start(seed=12345):
    return PCG64.from_numpy(np.random.Generator(np.random.PCG64(seed)))


def test_skip32_jump_equals_numpy_advance():
    rs = np.random.default_rng(7)
    ks = [0, 1, 2, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, 2 ** 63, 2 ** 64 - 1]
    ks += [int(x) for x in rs.integers(0, 2 ** 63, size=300)] + [int(x) for x in rs.integers(0, 1000, size=100)]
    for k in ks:
        g = start()
        skip32(g, 2 * k)                 # an empty buffer: 2k halves are k LCG steps and leave the buffer empty
        assert g.state == numpy_state(k) & MASK128, k
        assert g.has_uint32 == 0


def test_skip32_equals_repeated_next32_with_the_buffer_empty_and_full():
    for buffered in (False, True):
        base = start(99)
        if buffered:
            base.next32()
            assert base.has_uint32 == 1
        for n in range(301):
            a = PCG64(base.state, base.inc, base.has_uint32, base.uinteger)
            b = PCG64(base.state, base.inc, base.has_uint32, base.uinteger)
            skip32(a, n)
            for _ in range(n):
                b.next32()
            assert (a.state, a.inc, a.has_uint32, a.uinteger) == (b.state, b.inc, b.has_uint32, b.uinteger), (buffered, n)
            assert a.next32() == b.next32() and a.next64() == b.next64()


def test_skip32_equals_numpy_integers_draws():
    """C draws of integers(2**30) are C halves: integers(2^30) never rejects."""
    for n in (0, 1, 5, 98 * 3, 1001):
        g = np.random.Generator(np.random.PCG64(3))
        g.integers(2)                   # leaves a half buffered
        p = PCG64.from_numpy(g)
        for _ in range(n):
            g.integers(2 ** 30)
        skip32(p, n)
        assert (p.state, p.has_uint32, p.uinteger) == (PCG64.from_numpy(g).state, PCG64.from_numpy(g).has_uint32,
                                                       PCG64.from_numpy(g).uinteger), n
