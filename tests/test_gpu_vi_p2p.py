"""GPU: b2_vi_sweep_p2p (rl_agents_b200/csrc/vi_p2p.cu), the sweep kernel of DistributedVI(exchange="p2p") with the
exchange step fused in, against the numpy comparator, on one GPU.

Sweep k of a rank waits only for every rank's sweep k - 1 (their arrival flags).  Launched on one stream sweep after
sweep and, within a sweep, rank after rank, every flag a kernel acquires is already set, so no kernel ever waits: one
process on cuda:0 plays G ranks, each with its own VIEngine slab and its own peer buffer, laid out by
distributed.p2p_layout and wired by distributed.p2p_exchange as DistributedVI wires them.  That runs the whole protocol:
V' stored into every rank's copy of V, the table of per-slab violation counts in every rank's buffer, the arrival flags,
the launches after convergence that only pass the flag on, and the return of the old iterate.

Every case compares, bit for bit (a NaN matches any NaN), with a loop that mirrors oracle.planners.value_iteration
at the case's tolerances and records, at every sweep and for every slab, the count of ~np.isclose(Q, Q') (numpy's
rule: equal values are close whatever the tolerances, so rtol = 0, atol = -1 counts only changed values):
  * the concatenated Q slabs and the sweep count (and planners.value_iteration itself at the default tolerances);
  * every rank's copy of the table: parts[r'][k, r] = slab r's count at sweep k, 0 for a sweep launched after
    convergence;
  * both Q buffers of every rank and both V copies of every rank hold the last two iterates a computing sweep made
    (V' = max_a Q'): the exchange reached every copy, and the launches after convergence changed nothing;
  * flags[r'][r] = sweeps launched and status = 0 on every rank.  A non-zero status means a flag wait timed out:
    the launch order or the flag protocol is broken.

The same element test (np_isclose, common.cuh) runs in b2_vi_sweep's single-GPU kernels, which one section checks at
rtol = 0, atol = -1.  The last section drives DistributedVI(exchange="p2p") itself in a single-process gloo group
(world 1)."""
import numpy as np
import pytest

from oracle import planners
from rl_agents_b200 import _lib
from rl_agents_b200.distributed import p2p_exchange, p2p_layout, p2p_result, shard_range
from tests import vi_cases

pytestmark = pytest.mark.gpu

DEFAULT_TOL = (1e-5, 1e-8)          # np.allclose's, DistributedVI's
EXIT_OFF = (0.0, -1.0)              # bench.py's C4 setting: only an exact fixed point stops


def same(got, want):
    return np.array_equal(got.cpu().numpy() if hasattr(got, "cpu") else got, want, equal_nan=True)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def garnet(mode, S, A, B, seed, terminal_every=97):
    T, R, _, N = vi_cases.garnet_mdp(mode, S, A, B, seed=seed)
    term = np.zeros(S, bool)
    term[::terminal_every] = True
    return T, R, term, N


def oracle_sweeps(mode, T, R, term, N, gamma, iterations, tol, bounds):
    """planners.value_iteration's loop with np.isclose at tol = (rtol, atol).  Returns (iterates, counts, converged):
    iterates = [Q_0 = 0, Q_1, ...] (Q_{k+1} is what sweep k computes), counts[k][r] = the (s, a) pairs of slab r that
    np.isclose(Q_k, Q_{k+1}) finds apart, for every sweep that computed."""
    qs, counts = [np.zeros(R.shape)], []
    with np.errstate(invalid="ignore", over="ignore"):
        for _ in range(iterations):
            nq = planners.bellman_expectation(mode, T, R, term, qs[-1].max(axis=-1), gamma, nxt=N)
            apart = ~np.isclose(qs[-1], nq, rtol=tol[0], atol=tol[1])
            counts.append([int(apart[b:e].sum()) for b, e in bounds])
            qs.append(nq)
            if not apart.any():
                return qs, np.array(counts), True
    return qs, np.array(counts, dtype=np.int64).reshape(-1, len(bounds)), False


def latest_by_parity(qs):
    """The iterates the two ping-pong buffers hold at the end: the last one of each parity (zeros if none)."""
    out = [np.zeros_like(qs[0]), np.zeros_like(qs[0])]
    for m, q in enumerate(qs):
        out[m & 1] = q
    return out


class Ranks(object):
    """G ranks of DistributedVI(exchange="p2p") in one process on cuda:0: one VIEngine per slab shard_range(S, r, G),
    one zeroed peer buffer per rank in p2p_layout, one b2_vi_p2p per rank naming all G buffers."""

    def __init__(self, mode, T, R, term, N, gamma, world, max_iterations, tol=DEFAULT_TOL):
        import torch
        from rl_agents_b200.engine.vi import VIEngine
        self.torch, self.lib = torch, _lib.load()
        S = R.shape[0]
        self.S, self.world, self.max_iterations = S, world, max_iterations
        self.bounds = [shard_range(S, r, world) for r in range(world)]
        self.engines = [VIEngine(mode, T[b:e], R[b:e], term[b:e], nxt=None if N is None else N[b:e], gamma=gamma,
                                 device="cuda:0", row_begin=b, row_end=e, n_states=S, rtol=tol[0], atol=tol[1])
                        for b, e in self.bounds]
        self.layout = p2p_layout(S, world, max_iterations)
        self.bufs = [torch.zeros(self.layout["nbytes"], dtype=torch.uint8, device="cuda:0") for _ in range(world)]
        self.x = [p2p_exchange(self.layout, [b.data_ptr() for b in self.bufs], r) for r in range(world)]

    def region(self, r, offset, dtype, n):
        return self.bufs[r][offset:offset + n * dtype.itemsize].view(dtype)

    def v(self, r, i):
        return self.region(r, self.layout["v"][i], self.torch.float64, self.S)

    def flags(self, r):
        return self.region(r, self.layout["flags"], self.torch.int32, self.world).cpu().numpy()

    def parts(self, r):
        t = self.region(r, self.layout["parts"], self.torch.int32, self.max_iterations * self.world)
        return t.cpu().numpy().reshape(self.max_iterations, self.world)

    def status(self, r):
        return int(self.region(r, self.layout["status"], self.torch.int32, 1).item())

    def sweep(self, r, k, problem=None, x=None, q_new=None):
        """b2_vi_sweep_p2p of rank r at sweep k (raises B2Error on a refusal)."""
        eng = self.engines[r]
        _lib.check(self.lib.b2_vi_sweep_p2p(
            eng.problem if problem is None else problem, self.x[r] if x is None else x, _lib.ptr(eng.q[k & 1]),
            _lib.ptr(eng.q[(k + 1) & 1] if q_new is None else q_new), k, _lib.current_stream()))

    def solve(self, iterations):
        """What DistributedVI._solve_p2p does on every rank: zero Q and the buffers, launch the sweeps (sweep-major,
        rank-minor), pick the result from the violation table.  Returns (the concatenated Q, sweeps)."""
        assert iterations <= self.max_iterations
        for eng in self.engines:
            for q in eng.q:
                q.zero_()
        for b in self.bufs:
            b.zero_()
        for k in range(iterations):
            for r in range(self.world):
                self.sweep(r, k)
        self.torch.cuda.synchronize()
        k, sweeps = p2p_result(self.parts(0)[:iterations])
        return np.concatenate([eng.q[k & 1].cpu().numpy() for eng in self.engines]), sweeps

    def check_state(self, qs, counts, iterations):
        """Every rank's status, flags, violation table, Q buffers and V copies after `iterations` launched sweeps."""
        for r in range(self.world):
            assert self.status(r) == 0, \
                "rank %d: a flag wait timed out: the launch order or the flag protocol is broken" % r
        table = np.zeros((self.max_iterations, self.world), dtype=np.int64)
        table[:len(counts)] = counts
        last = latest_by_parity(qs)
        v_last = [q.max(axis=-1) for q in last]
        for r in range(self.world):
            assert (self.flags(r) == iterations).all(), (r, self.flags(r))
            assert np.array_equal(self.parts(r), table), r
            for i in (0, 1):
                assert same(self.v(r, i), v_last[i]), (r, i)
        for (b, e), eng in zip(self.bounds, self.engines):
            for i in (0, 1):
                assert same(eng.q[i], last[i][b:e]), (b, i)


def reference(mode, T, R, term, N, gamma, iterations):
    with np.errstate(invalid="ignore", over="ignore"):
        return planners.value_iteration(mode, T, R, term, gamma, iterations, nxt=N)


def solve_and_check(ranks, mode, T, R, term, N, gamma, iterations, tol=DEFAULT_TOL):
    """One solve of the G ranks against the oracle loop (and planners.value_iteration at the default tolerances).
    Returns (Q, sweeps, converged)."""
    qs, counts, converged = oracle_sweeps(mode, T, R, term, N, gamma, iterations, tol, ranks.bounds)
    want = qs[-2] if converged else qs[-1]
    if tol == DEFAULT_TOL:
        q_ref, sweeps_ref = reference(mode, T, R, term, N, gamma, iterations)
        assert sweeps_ref == len(counts) and same(want, q_ref)
    q, sweeps = ranks.solve(iterations)
    assert sweeps == len(counts)
    assert same(q, want)
    ranks.check_state(qs, counts, iterations)
    return q, sweeps, converged


# ------------------------------------------------------------ shapes at world 3 ----
@pytest.mark.parametrize("A", [1, 2, 4, 8, 16, 32])
@pytest.mark.parametrize("mode,B", [("deterministic", 1), ("sparse", 1), ("sparse", 2), ("sparse", 4), ("sparse", 8)])
def test_shapes_world_3(mode, A, B):
    """Every shape the kernel takes: A a power of two <= 32 (A = 16 and 32: the max over actions spans half a warp and
    the whole warp), deterministic and sparse B in {1, 2, 4, 8} (B = 8: numpy's pairwise tree).  S = 1001 over 3 ranks:
    slabs of 334, 334 and 333 states, whose (s, a) counts are not multiples of a CTA, and a rank 2 whose first state
    is not a multiple of 32.  12 sweeps at gamma = 0.9 do not converge: the last iterate is returned."""
    S = 1001
    T, R, term, N = garnet(mode, S, A, B, seed=100 + 10 * A + B)
    ranks = Ranks(mode, T, R, term, N, 0.9, 3, 16)
    assert all(((e - b) * A) % 256 for b, e in ranks.bounds)
    _, sweeps, converged = solve_and_check(ranks, mode, T, R, term, N, 0.9, 12)
    assert not converged and sweeps == 12


# --------------------------------------------------------------------- worlds ----
@pytest.mark.parametrize("world", [1, 2, 5, 8])
@pytest.mark.parametrize("mode,A,B", [("sparse", 8, 4), ("deterministic", 4, 1)])
def test_worlds(mode, A, B, world):
    """World 1 (every store goes to the own copy), 2, 5 and 8 (B2_MAX_PEERS) ranks on S = 4099, ragged for every world
    but 1; gamma = 0.7 converges well inside the 60 sweeps launched."""
    S = 4099
    T, R, term, N = garnet(mode, S, A, B, seed=world + A)
    ranks = Ranks(mode, T, R, term, N, 0.7, world, 64)
    _, sweeps, converged = solve_and_check(ranks, mode, T, R, term, N, 0.7, 60)
    assert converged and sweeps < 50


# ---------------------------------------------------------------- grid stride ----
@pytest.mark.parametrize("world", [2, 8])
def test_grid_stride(world):
    """The grid is capped at sm_count * 8 CTAs of 256 threads; every rank's slab holds more (s, a) pairs, so every
    thread strides (world 8: just past one round, the second a ragged tail).  bench.py's C4 p2p setting: sparse A = 8,
    B = 4, gamma = 0.95, rtol = 0, atol = -1; 4 sweeps."""
    A, B = 8, 4
    cap = sm_count() * 8 * 256
    S = 8 * (cap // A + 37) + 5
    T, R, term, N = garnet("sparse", S, A, B, seed=world)
    ranks = Ranks("sparse", T, R, term, N, 0.95, world, 4, tol=EXIT_OFF)
    assert min((e - b) * A for b, e in ranks.bounds) > cap
    _, sweeps, converged = solve_and_check(ranks, "sparse", T, R, term, N, 0.95, 4, tol=EXIT_OFF)
    assert not converged and sweeps == 4


# ---------------------------------------------------------- convergence edges ----
SHAPES = [("sparse", 8, 4), ("deterministic", 4, 1)]


@pytest.mark.parametrize("tol", [DEFAULT_TOL, EXIT_OFF])
@pytest.mark.parametrize("mode,A,B", SHAPES)
def test_zero_rewards_converge_at_sweep_0(mode, A, B, tol):
    """R = 0: Q' = Q = 0 at sweep 0, which meets np.isclose even at atol = -1 (equal values); the returned Q is the
    zeros of Q_0 after one sweep, and the 9 sweeps launched after it leave every buffer at zero."""
    S = 1001
    T, R, term, N = garnet(mode, S, A, B, seed=1)
    R = np.zeros_like(R)
    ranks = Ranks(mode, T, R, term, N, 0.9, 3, 16, tol=tol)
    q, sweeps, converged = solve_and_check(ranks, mode, T, R, term, N, 0.9, 10, tol=tol)
    assert converged and sweeps == 1 and not q.any()


@pytest.mark.parametrize("tol", [DEFAULT_TOL, EXIT_OFF])
@pytest.mark.parametrize("mode,A,B", SHAPES)
def test_gamma_0_converges_at_sweep_1(mode, A, B, tol):
    """gamma = 0: Q' = R at every sweep, so sweep 1 meets np.isclose (at atol = -1 too) and Q_1 = R is returned after
    two sweeps."""
    S = 1001
    T, R, term, N = garnet(mode, S, A, B, seed=2)
    ranks = Ranks(mode, T, R, term, N, 0.0, 3, 16, tol=tol)
    q, sweeps, converged = solve_and_check(ranks, mode, T, R, term, N, 0.0, 10, tol=tol)
    assert converged and sweeps == 2 and np.array_equal(q, R)


@pytest.mark.parametrize("mode,A,B", SHAPES)
def test_early_exit_then_idle_sweeps_and_resolve(mode, A, B):
    """gamma = 0.6 converges within about 30 of the 80 sweeps launched; the launches after it only pass the flags
    on.  Then, in the same buffers, a 3-sweep solve (not converged) and the 80-sweep solve again: the same bits."""
    S = 1001
    T, R, term, N = garnet(mode, S, A, B, seed=3)
    ranks = Ranks(mode, T, R, term, N, 0.6, 3, 80)
    q1, sweeps1, converged = solve_and_check(ranks, mode, T, R, term, N, 0.6, 80)
    assert converged and sweeps1 < 40
    _, sweeps, converged = solve_and_check(ranks, mode, T, R, term, N, 0.6, 3)
    assert not converged and sweeps == 3
    q2, sweeps2, _ = solve_and_check(ranks, mode, T, R, term, N, 0.6, 80)
    assert sweeps2 == sweeps1 and np.array_equal(q1, q2)


@pytest.mark.parametrize("mode,A,B", SHAPES)
def test_no_convergence_returns_last_iterate(mode, A, B):
    """gamma = 0.99, 5 sweeps: no sweep meets np.allclose; the iterate of the fifth sweep is returned."""
    S = 1001
    T, R, term, N = garnet(mode, S, A, B, seed=4)
    ranks = Ranks(mode, T, R, term, N, 0.99, 3, 8)
    _, sweeps, converged = solve_and_check(ranks, mode, T, R, term, N, 0.99, 5)
    assert not converged and sweeps == 5


@pytest.mark.parametrize("mode,A,B", SHAPES)
def test_zero_iterations(mode, A, B):
    """iterations = 0: nothing launched, Q = 0 after 0 sweeps, every flag and count 0."""
    S = 1001
    T, R, term, N = garnet(mode, S, A, B, seed=5)
    ranks = Ranks(mode, T, R, term, N, 0.9, 3, 4)
    q, sweeps, _ = solve_and_check(ranks, mode, T, R, term, N, 0.9, 0)
    assert sweeps == 0 and not q.any()


# ------------------------------------------------------------ non-finite MDPs ----
@pytest.mark.parametrize("tol", [DEFAULT_TOL, EXIT_OFF])
@pytest.mark.parametrize("gamma", [0.9, 0.0])
@pytest.mark.parametrize("mode,A,B", [("sparse", 4, 8), ("sparse", 8, 2), ("deterministic", 8, 1)])
def test_nonfinite_mdp(mode, A, B, gamma, tol):
    """tests/vi_cases.nonfinite_mdp: +-inf rewards and zero probabilities turn into NaN (-inf + gamma * inf, 0 * inf),
    which numpy's max over actions keeps after a number; the NaN V crosses the slabs through the exchange.  NaN is
    close to nothing, equal infinities are close at any tolerance."""
    S = 1001
    T, R, term, N = vi_cases.nonfinite_mdp(mode, S, A, B, seed=S + A + B)
    ranks = Ranks(mode, T, R, term, N, gamma, 3, 8, tol=tol)
    q, _, _ = solve_and_check(ranks, mode, T, R, term, N, gamma, 6, tol=tol)
    assert np.isnan(q).any() and np.isinf(q).any()


# ------------------------------------------- the single-GPU sweeps' element test ----
@pytest.mark.parametrize("mode,S,A,B,path", [("deterministic", 400, 4, 1, "row"),
                                             ("deterministic", 400, 3, 1, "gather"), ("sparse", 400, 4, 2, "row"),
                                             ("sparse", 400, 3, 3, "gather"), ("stochastic", 150, 3, None, "dense")])
def test_single_gpu_sweeps_stop_at_an_exact_fixed_point_at_negative_atol(mode, S, A, B, path):
    """The element test np_isclose (common.cuh) is shared with b2_vi_sweep's kernels (vi.cu).  At rtol = 0, atol = -1
    numpy's isclose still holds for equal values, so at gamma = 0, where Q' = R at every sweep, np.allclose holds at
    sweep 1 and R is returned after two sweeps; at gamma = 0.9 no sweep repeats Q exactly and the whole budget runs.
    Register, gather and dense kernels."""
    from rl_agents_b200.engine.vi import VIEngine
    from tests.test_gpu_vi_paths import engine_selects_row_kernel
    if mode == "stochastic":
        rng = np.random.default_rng(S)
        T = rng.uniform(size=(S, A, S))
        T /= T.sum(axis=-1, keepdims=True)
        R, term, N = rng.uniform(size=(S, A)), rng.uniform(size=S) < 0.05, None
    else:
        T, R, term, N = vi_cases.garnet_mdp(mode, S, A, B, seed=S + A)
    assert np.isclose(R, R, rtol=0.0, atol=-1.0).all() and not (np.abs(R - R) <= -1.0).any()
    for gamma, sweeps_want in ((0.0, 2), (0.9, 30)):
        eng = VIEngine(mode, T, R, term, nxt=N, gamma=gamma, rtol=0.0, atol=-1.0)
        if path != "dense":
            assert engine_selects_row_kernel(eng) == (path == "row")
        q_ref, sweeps_ref = reference(mode, T, R, term, N, gamma, 30)
        assert sweeps_ref == sweeps_want
        q, sweeps = eng.solve(30)
        assert sweeps == sweeps_want and same(q, q_ref)
        if gamma == 0.0:
            assert np.array_equal(q_ref, R)


# ----------------------------------------------------------------- refusals ----
def _set(obj, name, value):
    return lambda p, x: setattr(p if obj == "p" else x, name, value(p, x) if callable(value) else value)


def _null(field, i, j=None):
    def f(p, x):
        arr = getattr(x, field) if j is None else getattr(x, field)[j]
        arr[i] = None
    return f


REFUSALS = {
    "stochastic": _set("p", "mode", _lib.VI_STOCHASTIC),
    "A=3": _set("p", "n_actions", 3),
    "A=64": _set("p", "n_actions", 64),
    "B=3": _set("p", "n_next", 3),
    "B=16": _set("p", "n_next", 16),
    "next+1": _set("p", "next", lambda p, x: p.next + 4),                   # one int32 off
    "transition+1": _set("p", "transition", lambda p, x: p.transition + 8),  # one double off
    "empty slab": _set("p", "row_end", lambda p, x: p.row_begin),
    "world=0": _set("x", "world", 0),
    "world=9": _set("x", "world", 9),
    "rank=world": _set("x", "rank", lambda p, x: x.world),
    "v[0][1]=null": _null("v", 1, 0),
    "v[1][1]=null": _null("v", 1, 1),
    "flags[1]=null": _null("flags", 1),
    "parts[1]=null": _null("parts", 1),
    "viol_local=null": _set("x", "viol_local", None),
    "done=null": _set("x", "done", None),
    "status=null": _set("x", "status", None),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_refusals(case):
    """b2_vi_sweep_p2p refuses, with an error that _lib.check raises as B2Error, and launches nothing: Q', the flags,
    the violation tables and every V copy are as they were.  Rank 1 of a world of 2 at sweep 1, after both ranks' sweep
    0; each case breaks one thing of an accepted call (mode or shape, alignment, world / rank, a missing pointer)."""
    import torch
    S, A, B = 64, 8, 4
    T, R, term, N = garnet("sparse", S, A, B, seed=6)
    ranks = Ranks("sparse", T, R, term, N, 0.9, 2, 4)
    for r in range(2):
        ranks.sweep(r, 0)
    p = _lib.VIProblem.from_buffer_copy(ranks.engines[1].problem)
    x = _lib.VIP2P.from_buffer_copy(ranks.x[1])
    REFUSALS[case](p, x)
    torch.cuda.synchronize()
    q_new = torch.full_like(ranks.engines[1].q[0], 7.0)
    flags, parts = [ranks.flags(r) for r in range(2)], [ranks.parts(r) for r in range(2)]
    v = [[ranks.v(r, i).clone() for i in (0, 1)] for r in range(2)]
    with pytest.raises(_lib.B2Error):
        ranks.sweep(1, 1, problem=p, x=x, q_new=q_new)
    torch.cuda.synchronize()
    assert (q_new == 7.0).all()
    for r in range(2):
        assert np.array_equal(ranks.flags(r), flags[r]) and (ranks.flags(r) == 1).all()
        assert np.array_equal(ranks.parts(r), parts[r])
        assert all(torch.equal(ranks.v(r, i), v[r][i]) for i in (0, 1))
        assert ranks.status(r) == 0
    for r in range(2):                     # the call as it was is accepted
        ranks.sweep(r, 1)
    torch.cuda.synchronize()
    assert all((ranks.flags(r) == 2).all() for r in range(2))


# ------------------------------------------------- DistributedVI at world 1 ----
@pytest.fixture(scope="module")
def gloo_world_1(tmp_path_factory):
    """A single-process gloo group on a file store: DistributedVI's collectives and PeerBuffer's handle exchange
    without any network address."""
    import torch.distributed as dist
    store = dist.FileStore(str(tmp_path_factory.mktemp("gloo") / "store"), 1)
    dist.init_process_group("gloo", store=store, rank=0, world_size=1)
    yield
    dist.destroy_process_group()


@pytest.mark.parametrize("mode,A,B", SHAPES)
def test_distributed_vi_p2p_world_1(gloo_world_1, mode, A, B):
    """DistributedVI(exchange="p2p") at world 1 equals planners.value_iteration bit for bit, twice in the same
    buffers; v_slab(sweeps) holds max_a Q of the iterate returned after an unconverged solve, v_slab(sweeps - 1)
    after a converged one.  exchange="nccl" (host-staged under gloo) gives the same bits."""
    from rl_agents_b200.distributed import DistributedVI
    S = 2003
    T, R, term, N = garnet(mode, S, A, B, seed=7)
    dvi = DistributedVI(mode, T, R, term, nxt=N, gamma=0.7, device="cuda:0", exchange="p2p", max_iterations=64)
    try:
        q_ref, sweeps_ref = reference(mode, T, R, term, N, 0.7, 60)
        assert sweeps_ref < 60
        for _ in range(2):
            q, sweeps = dvi.solve(60)
            assert sweeps == sweeps_ref and same(q, q_ref)
            assert same(dvi.v_slab(sweeps - 1), q_ref.max(axis=-1))
        q_ref5, _ = reference(mode, T, R, term, N, 0.7, 5)
        q, sweeps = dvi.solve(5)
        assert sweeps == 5 and same(q, q_ref5) and same(dvi.v_slab(5), q_ref5.max(axis=-1))
        with pytest.raises(ValueError, match="max_iterations"):
            dvi.solve(65)
    finally:
        dvi.close()
    q, sweeps = DistributedVI(mode, T, R, term, nxt=N, gamma=0.7, device="cuda:0", exchange="nccl").solve(60)
    assert sweeps == sweeps_ref and same(q, q_ref)


@pytest.mark.parametrize("mode,A,B,match", [("stochastic", 4, None, "mode"), ("sparse", 3, 4, "power of two"),
                                            ("sparse", 64, 1, "power of two"), ("deterministic", 6, 1, "power of two"),
                                            ("sparse", 8, 3, "successors"), ("sparse", 4, 16, "successors")])
def test_distributed_vi_p2p_refuses_before_allocating(gloo_world_1, mode, A, B, match):
    """A problem b2_vi_sweep_p2p refuses on every rank is refused by DistributedVI's constructor with ValueError,
    before the VIEngine uploads a table or PeerBuffer allocates."""
    import torch
    from rl_agents_b200.distributed import DistributedVI
    S = 64
    if mode == "stochastic":
        T = np.full((S, A, S), 1.0 / S)
        R, term, N = np.zeros((S, A)), np.zeros(S, bool), None
    else:
        T, R, term, N = garnet(mode, S, A, B or 1, seed=8)
    torch.cuda.synchronize()
    allocated = torch.cuda.memory_allocated(0)
    with pytest.raises(ValueError, match=match):
        DistributedVI(mode, T, R, term, nxt=N, gamma=0.9, device="cuda:0", exchange="p2p", max_iterations=8)
    assert torch.cuda.memory_allocated(0) == allocated


def offset_view(a, dtype):
    """a copied to the device one element into a larger buffer: contiguous, but not 16-byte aligned."""
    import torch
    flat = torch.as_tensor(np.ascontiguousarray(a).ravel()).to(dtype)
    buf = torch.zeros(flat.numel() + 1, dtype=dtype, device="cuda:0")
    buf[1:].copy_(flat)
    return buf[1:].view(a.shape)


@pytest.mark.parametrize("mode,A,B", SHAPES)
def test_distributed_vi_p2p_copies_misaligned_device_slabs(gloo_world_1, mode, A, B):
    """Device slabs (tables_are_local) at an odd element offset, which b2_vi_sweep_p2p refuses and which only their
    own rank can see: DistributedVI copies them into aligned allocations, and the solve equals numpy's."""
    import torch
    from rl_agents_b200.distributed import DistributedVI
    S = 1001
    T, R, term, N = garnet(mode, S, A, B, seed=9)
    if mode == "sparse":
        T_dev, N_dev = offset_view(T, torch.float64), offset_view(N, torch.int32)
        assert T_dev.data_ptr() % 16 and N_dev.data_ptr() % 16
    else:
        T_dev, N_dev = offset_view(T, torch.int32), None
        assert T_dev.data_ptr() % 16
    dvi = DistributedVI(mode, T_dev, R, term, nxt=N_dev, gamma=0.7, device="cuda:0", exchange="p2p",
                        tables_are_local=True, n_states=S, max_iterations=64)
    try:
        assert dvi.engine.transition.data_ptr() % 16 == 0
        assert dvi.engine.problem.transition == dvi.engine.transition.data_ptr()
        if mode == "sparse":
            assert dvi.engine.next.data_ptr() % 16 == 0 and dvi.engine.problem.next == dvi.engine.next.data_ptr()
        q, sweeps = dvi.solve(60)
        q_ref, sweeps_ref = reference(mode, T, R, term, N, 0.7, 60)
        assert sweeps == sweeps_ref and same(q, q_ref)
    finally:
        dvi.close()
