"""GPU: every launch path of the value-iteration sweep kernels (rl_agents_b200/csrc/vi.cu) against the numpy comparator
(oracle.planners.value_iteration / robust_value_iteration): the same sweep count and the same Q, bit for bit, also on
MDPs with infinite rewards, where numpy's max over actions and min over models propagate NaN.  NaN payloads and signs
may differ between the host and the device, so a NaN matches any NaN; every other value matches bit for bit.

b2_vi_sweep selects the kernel from the shape and the alignment of the tables (vi.cu, b2_vi_sweep):
  * vi_sweep_row_kernel<B, HAS_P>: A a power of two <= 32, B in {1, 2, 4, 8}, N (and P) 16-byte aligned;
  * vi_sweep_gather_kernel: every other sparse or deterministic shape with A * B <= 8192 (larger is refused);
  * vi_sweep_dense_group_kernel + vi_rowmax_kernel: stochastic (dense) mode;
and b2_vi_robust_sweep runs vi_robust_kernel + vi_rowmax_kernel."""
import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import planners
from tests import vi_cases

pytestmark = pytest.mark.gpu


def sm_count():
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def row_kernel_selected(A, B, n_ptr, p_ptr=None):
    """vi.cu's rule for vi_sweep_row_kernel, written as b2_vi_sweep writes it."""
    return ((A & (A - 1)) == 0 and A <= 32 and B in (1, 2, 4, 8) and n_ptr % 16 == 0
            and (p_ptr is None or p_ptr % 16 == 0))


def engine_selects_row_kernel(eng):
    if eng.mode == "sparse":
        return row_kernel_selected(eng.n_actions, eng.n_next, eng.next.data_ptr(), eng.transition.data_ptr())
    assert eng.mode == "deterministic"
    return row_kernel_selected(eng.n_actions, 1, eng.transition.data_ptr())


def gather_tile(A, B):
    """States per CTA of vi_sweep_gather_kernel, as b2_vi_sweep sizes it."""
    tile = max(4096 // (A * B), 1)
    if tile * A > 2048:
        tile = max(2048 // A, 1)
    return tile


def reference(mode, T, R, term, gamma, iterations, nxt=None):
    with np.errstate(invalid="ignore", over="ignore"):
        return planners.value_iteration(mode, T, R, term, gamma, iterations, nxt=nxt)


def robust_reference(mode, T, R, gamma, iterations):
    with np.errstate(invalid="ignore", over="ignore"):
        return planners.robust_value_iteration(mode, T, R, gamma, iterations)


def same(got, want):
    return np.array_equal(got.cpu().numpy() if hasattr(got, "cpu") else got, want, equal_nan=True)


def make_engine(mode, T, R, term, nxt, gamma):
    from rl_agents_b200.engine.vi import VIEngine
    return VIEngine(mode, T, R, term, nxt=nxt, gamma=gamma)


def solve_and_compare(eng, mode, T, R, term, gamma, iterations, nxt=None):
    q_ref, sweeps_ref = reference(mode, T, R, term, gamma, iterations, nxt=nxt)
    q, sweeps = eng.solve(iterations)
    assert sweeps == sweeps_ref
    assert same(q, q_ref)
    return q_ref, sweeps_ref


def sweep_by_sweep(eng, mode, T, R, term, gamma, n, nxt=None):
    """n sweeps launched one at a time; after each, Q' and V' = max_a Q' against numpy's.  Returns numpy's iterates.
    The cases never converge within n sweeps (a converged sweep leaves the buffers as they were)."""
    eng.reset(n)
    v = np.zeros(eng.n_states)
    iterates = []
    for k in range(n):
        eng.sweep(k)
        with np.errstate(invalid="ignore", over="ignore"):
            q_ref = planners.bellman_expectation(mode, T, R, term, v, gamma, nxt=nxt)
        v = q_ref.max(axis=-1)
        assert same(eng.q[(k + 1) & 1], q_ref), k
        assert same(eng.v[(k + 1) & 1], v), k
        iterates.append(q_ref)
    assert (eng.viol.cpu().numpy() > 0).all()
    return iterates


# ------------------------------------------------------------ register kernel ----
@pytest.mark.parametrize("mode,A,B", [("sparse", A, B) for A in (1, 2, 16, 32) for B in (1, 2, 4, 8)]
                         + [("deterministic", A, 1) for A in (1, 2, 16, 32)])
def test_row_kernel_shapes(mode, A, B):
    """vi_sweep_row_kernel: A a power of two <= 32 and B in {1, 2, 4, 8}, tables 16-byte aligned.  A = 16 and 32 make
    the segmented shuffle of the max over actions span half a warp and the whole warp; A = 1 has no shuffle."""
    S = 40000 // A + 3
    T, R, term, N = vi_cases.garnet_mdp(mode, S, A, B, seed=A * 10 + B)
    eng = make_engine(mode, T, R, term, N, 0.9)
    assert engine_selects_row_kernel(eng)
    solve_and_compare(eng, mode, T, R, term, 0.9, 30, nxt=N)


def test_row_kernel_grid_stride():
    """vi_sweep_row_kernel at S * A above its grid cap of sm_count() * 64 CTAs of 256 threads: every thread takes
    several (s, a) rows, and the warps of a later stride still hold whole states (A = 32: the whole warp)."""
    S, A, B = 100_000, 32, 2
    assert S * A > sm_count() * 64 * 256
    T, R, term, N = vi_cases.garnet_mdp("sparse", S, A, B, seed=3)
    eng = make_engine("sparse", T, R, term, N, 0.95)
    assert engine_selects_row_kernel(eng)
    sweep_by_sweep(eng, "sparse", T, R, term, 0.95, 4, nxt=N)


# ------------------------------------------------------------ gather kernel ----
@pytest.mark.parametrize("mode,S,A,B", [("sparse", 3001, 64, 1), ("deterministic", 3001, 64, 1),
                                        ("sparse", 300, 3, 264), ("sparse", 150, 8, 1000), ("sparse", 40, 2, 4096),
                                        ("deterministic", 50, 8192, 1)])
def test_gather_kernel_shapes(mode, S, A, B):
    """vi_sweep_gather_kernel: every sparse or deterministic shape outside the register kernel's rule (A not a power of
    two <= 32, or B not in {1, 2, 4, 8}) with A * B <= 8192.  A = 64 is a power of two but too wide for a warp;
    B = 264 and 1000 make numpy's pairwise sum recurse more than one level; A * B = 8000 and 8192 leave one state per
    tile; A * B = 8192 needs more than 64 KB of dynamic shared memory, 128 KB at A = 8192 with B = 1 (the products and
    the Q of 8192 actions)."""
    T, R, term, N = vi_cases.garnet_mdp(mode, S, A, B, seed=S + A + B)
    eng = make_engine(mode, T, R, term, N, 0.9)
    assert not engine_selects_row_kernel(eng) and A * B <= 8192
    if A * B > 4096:
        assert gather_tile(A, B) == 1
    if A * B == 8192:
        assert (A * B + A) * 8 > 64 * 1024
    solve_and_compare(eng, mode, T, R, term, 0.9, 20, nxt=N)


def test_gather_kernel_grid_stride():
    """vi_sweep_gather_kernel with more than two rounds of its capped grid (sm_count() * 8 CTAs): each CTA loops over
    several tiles, through the tile loop's barriers, and sums its allclose violations across them."""
    S, A, B = 400_000, 5, 7
    n_tiles = -(-S // gather_tile(A, B))
    assert n_tiles > 2 * sm_count() * 8
    T, R, term, N = vi_cases.garnet_mdp("sparse", S, A, B, seed=5)
    eng = make_engine("sparse", T, R, term, N, 0.9)
    assert not engine_selects_row_kernel(eng)
    sweep_by_sweep(eng, "sparse", T, R, term, 0.9, 4, nxt=N)


@pytest.mark.parametrize("mode,A,B", [("sparse", 3, 2731), ("deterministic", 8193, 1)])
def test_gather_kernel_refuses_rows_over_8192(mode, A, B):
    """A * B = 8193 does not fit vi_sweep_gather_kernel's shared memory: b2_vi_sweep refuses it, it runs nothing."""
    from rl_agents_b200 import _lib
    assert A * B == 8193
    T, R, term, N = vi_cases.garnet_mdp(mode, 4, A, B, seed=0)
    eng = make_engine(mode, T, R, term, N, 0.9)
    with pytest.raises(_lib.B2Error, match="8192"):
        eng.solve(2)


# ------------------------------------------------------- alignment fallback ----
def offset_view(a, dtype):
    """a copied to the device one element into a larger buffer: contiguous, but not 16-byte aligned."""
    import torch
    flat = torch.as_tensor(np.ascontiguousarray(a).ravel()).to(dtype)
    buf = torch.zeros(flat.numel() + 1, dtype=dtype, device="cuda")
    buf[1:].copy_(flat)
    return buf[1:].view(a.shape)


@pytest.mark.parametrize("mode,A,B,shifted", [("sparse", 4, 4, "P"), ("sparse", 8, 2, "N"), ("sparse", 2, 8, "both"),
                                              ("deterministic", 8, 1, "N")])
def test_misaligned_tables_fall_back_to_gather_kernel(mode, A, B, shifted):
    """A register-kernel shape whose N or P is not 16-byte aligned (a view at an odd element offset, used by VIEngine as
    it is) takes vi_sweep_gather_kernel instead: the same bits as numpy and as the aligned tables."""
    import torch
    S = 5003
    T, R, term, N = vi_cases.garnet_mdp(mode, S, A, B, seed=A + B)
    aligned = make_engine(mode, T, R, term, N, 0.9)
    assert engine_selects_row_kernel(aligned)
    if mode == "sparse":
        P_dev = offset_view(T, torch.float64) if shifted in ("P", "both") else T
        N_dev = offset_view(N, torch.int32) if shifted in ("N", "both") else N
        eng = make_engine(mode, P_dev, R, term, N_dev, 0.9)
    else:
        eng = make_engine(mode, offset_view(T, torch.int32), R, term, None, 0.9)
    assert not engine_selects_row_kernel(eng)
    q_ref, sweeps_ref = solve_and_compare(eng, mode, T, R, term, 0.9, 25, nxt=N)
    q_aligned, sweeps_aligned = aligned.solve(25)
    assert sweeps_aligned == sweeps_ref and same(q_aligned, q_ref)


# ------------------------------------------------------------------- slabs ----
@pytest.mark.parametrize("mode,S,A,B", [("stochastic", 500, 3, None), ("sparse", 1001, 8, 4), ("deterministic", 999, 16, 1)])
def test_two_slabs_compose(mode, S, A, B):
    """Two row slabs sharing V reproduce numpy's sweeps, cut at a row that is not a multiple of 32: dense mode writes
    V' at row_begin + s through vi_rowmax_kernel; the register kernel (A * B a register shape) through its shuffle."""
    import torch
    from rl_agents_b200.engine.vi import VIEngine
    rng = np.random.default_rng(S)
    if mode == "stochastic":
        T = rng.uniform(size=(S, A, S))
        T /= T.sum(axis=-1, keepdims=True)
        R = rng.uniform(size=(S, A))
        term, N = rng.uniform(size=S) < 0.05, None
    else:
        T, R, term, N = vi_cases.garnet_mdp(mode, S, A, B, seed=S)
    cut, n = 403, 7
    assert 0 < cut < S and cut % 32

    def part(x, lo, hi):
        return None if x is None else x[lo:hi]
    slabs = [VIEngine(mode, part(T, lo, hi), R[lo:hi], term[lo:hi], nxt=part(N, lo, hi), gamma=0.9, row_begin=lo,
                      n_states=S) for lo, hi in ((0, cut), (cut, S))]
    if mode != "stochastic":
        assert all(engine_selects_row_kernel(e) for e in slabs)
    for e in slabs:
        e.reset(n)
    v = np.zeros(S)
    for k in range(n):
        for e in slabs:
            e.sweep(k)
        torch.cuda.synchronize()
        out = slabs[0].v[(k + 1) & 1]
        out[cut:] = slabs[1].v[(k + 1) & 1][cut:]          # the all-gather step
        slabs[1].v[(k + 1) & 1].copy_(out)
        viol = slabs[0].viol + slabs[1].viol                # the all-reduce step
        for e in slabs:
            e.viol.copy_(viol)
        q_ref = planners.bellman_expectation(mode, T, R, term, v, 0.9, nxt=N)
        v = q_ref.max(axis=-1)
        q = torch.cat([slabs[0].q[(k + 1) & 1], slabs[1].q[(k + 1) & 1]]).cpu().numpy()
        assert np.array_equal(q, q_ref) and np.array_equal(out.cpu().numpy(), v), k


# -------------------------------------------------------------- dense mode ----
@pytest.mark.parametrize("S,A", [(8, 3), (136, 3), (264, 2), (1200, 5), (1000, 7)])
def test_dense_kernels(S, A):
    """vi_sweep_dense_group_kernel + vi_rowmax_kernel: S = 8, 136 and 264 put numpy's pairwise sum at a single block of
    eight, at one split and at a split of a split; A = 5 and 7 at large S leave the actions of many states straddling
    two CTAs of 32 rows."""
    rng = np.random.default_rng(S * A)
    P = rng.uniform(size=(S, A, S))
    P /= P.sum(axis=-1, keepdims=True)
    R = rng.uniform(size=(S, A))
    term = rng.uniform(size=S) < 0.05
    if A in (5, 7):
        assert sum((s * A) // 32 != (s * A + A - 1) // 32 for s in range(S)) > 100
    eng = make_engine("stochastic", P, R, term, None, 0.9)
    solve_and_compare(eng, "stochastic", P, R, term, 0.9, 12)


# ------------------------------------------------------------------ robust ----
def robust_models(mode, M, S, A, seed):
    rng = np.random.default_rng(seed)
    if mode == "deterministic":
        ms = [oenvs.garnet(S, A, 1, seed=seed + m, deterministic=True) for m in range(M)]
        return np.array([m[0] for m in ms]), np.array([m[1] for m in ms])
    P = rng.uniform(size=(M, S, A, S))
    P /= P.sum(axis=-1, keepdims=True)
    return P, rng.uniform(size=(M, S, A))


def robust_solve_and_compare(mode, T, R, gamma, iterations):
    from rl_agents_b200.engine.vi import RobustVIEngine
    q_ref, sweeps_ref = robust_reference(mode, T, R, gamma, iterations)
    q, sweeps = RobustVIEngine(mode, T, R, gamma=gamma).solve(iterations)
    assert sweeps == sweeps_ref
    assert same(q, q_ref)
    return q_ref, sweeps_ref


@pytest.mark.parametrize("S,M", [(129, 1), (129, 3), (300, 1), (300, 3)])
def test_robust_dense(S, M):
    """vi_robust_kernel, dense models with S > 128: each thread runs numpy's recursive pairwise sum over a whole row of
    every model."""
    T, R = robust_models("stochastic", M, S, 3, seed=S + M)
    robust_solve_and_compare("stochastic", T, R, 0.9, 15)


@pytest.mark.parametrize("M,A", [(1, 1), (1, 3), (1, 8), (5, 1), (5, 3), (5, 8)])
def test_robust_deterministic(M, A):
    """vi_robust_kernel, deterministic models at S * A > 10^5: many 128-thread blocks, each thread looping over the
    models; A = 1 leaves vi_rowmax_kernel a single action."""
    S = -(-120_000 // A)
    T, R = robust_models("deterministic", M, S, A, seed=40 + M + A)
    robust_solve_and_compare("deterministic", T, R, 0.9, 15)


@pytest.mark.parametrize("mode", ["deterministic", "stochastic"])
def test_robust_single_model_is_plain_value_iteration(mode):
    """vi_robust_kernel with M = 1 is value iteration without terminal states: the same bits as VIEngine."""
    from rl_agents_b200.engine.vi import RobustVIEngine
    S, A = (5000, 4) if mode == "deterministic" else (200, 3)
    T, R = robust_models(mode, 1, S, A, seed=7)
    q, sweeps = RobustVIEngine(mode, T, R, gamma=0.9).solve(40)
    q_plain, sweeps_plain = make_engine(mode, T[0], R[0], np.zeros(S, bool), None, 0.9).solve(40)
    assert sweeps == sweeps_plain and np.array_equal(q.cpu().numpy(), q_plain.cpu().numpy())
    q_ref, sweeps_ref = robust_reference(mode, T, R, 0.9, 40)
    assert sweeps == sweeps_ref and np.array_equal(q.cpu().numpy(), q_ref)


@pytest.mark.parametrize("mode", ["deterministic", "stochastic"])
def test_robust_early_exit_returns_previous_iterate(mode):
    """vi_robust_kernel at gamma = 0.5 converges well before the iteration budget; like numpy it returns the iterate
    before the sweep that met np.allclose."""
    S, A = (3000, 4) if mode == "deterministic" else (100, 3)
    T, R = robust_models(mode, 3, S, A, seed=11)
    _, sweeps = robust_solve_and_compare(mode, T, R, 0.5, 200)
    assert sweeps < 200


# ------------------------------------------------------- non-finite MDPs ----
def test_three_state_mdp_with_infinite_rewards():
    """vi_sweep_row_kernel (A = 2, B = 1): the NaN of -inf + 0.9 * inf sits at the second action of state 0, after a
    finite first action; numpy's max returns NaN, and so must the segmented shuffle."""
    c = vi_cases.THREE_STATE
    T, R, term = c["transition"], c["reward"], c["terminal"]
    eng = make_engine("deterministic", T, R, term, None, 0.9)
    assert engine_selects_row_kernel(eng)
    iterates = sweep_by_sweep(eng, "deterministic", T, R, term, 0.9, 4)
    assert vi_cases.nan_after_a_number(iterates[1])
    q_ref, _ = solve_and_compare(eng, "deterministic", T, R, term, 0.9, 4)
    assert np.isnan(q_ref[:2]).all() and (q_ref[2] == np.inf).all()


NONFINITE = [("deterministic", 500, 4, 1, "row"), ("deterministic", 500, 3, 1, "gather"),
             ("sparse", 500, 4, 4, "row"), ("sparse", 300, 2, 8, "row"), ("sparse", 500, 3, 5, "gather"),
             ("stochastic", 150, 3, None, "dense"), ("stochastic", 264, 2, None, "dense")]


@pytest.mark.parametrize("gamma", [0.9, 0.0])
@pytest.mark.parametrize("mode,S,A,B,path", NONFINITE)
def test_nonfinite_mdp(mode, S, A, B, path, gamma):
    """Every sweep kernel on MDPs with +-inf rewards and zero probabilities (tests/vi_cases.py): NaN from
    -inf + gamma * inf, 0 * inf and, at gamma = 0, 0 * inf against an infinite V reaches the max over actions after a
    number.  "row" shapes take vi_sweep_row_kernel, "gather" shapes vi_sweep_gather_kernel, "dense" the dense kernels;
    sweep by sweep and through b2_vi_solve."""
    T, R, term, N = vi_cases.nonfinite_mdp(mode, S, A, B, seed=S + A + (B or 0))
    eng = make_engine(mode, T, R, term, N, gamma)
    if path != "dense":
        assert engine_selects_row_kernel(eng) == (path == "row")
    iterates = sweep_by_sweep(eng, mode, T, R, term, gamma, 6, nxt=N)
    if not (mode == "stochastic" and gamma == 0.0):
        # (at gamma = 0 a dense row meets every infinite V through 0 * inf: all its actions turn NaN in the same sweep)
        assert any(vi_cases.nan_after_a_number(q) for q in iterates)
    q_ref, _ = solve_and_compare(eng, mode, T, R, term, gamma, 6, nxt=N)
    assert np.isnan(q_ref).any()


@pytest.mark.parametrize("gamma", [0.9, 0.0])
@pytest.mark.parametrize("mode,M,S,A", [("deterministic", 3, 500, 3), ("deterministic", 2, 500, 1),
                                        ("stochastic", 2, 150, 3), ("stochastic", 3, 129, 2)])
def test_nonfinite_robust(mode, M, S, A, gamma):
    """vi_robust_kernel on models with +-inf rewards: np.min over the models returns NaN when one model is NaN, and
    when every model is (state 0 from the second sweep on); the kernel used to skip a NaN model and return +inf when
    all were.  Checked after each of 6 sweeps, V' = max_a Q' included."""
    from rl_agents_b200.engine.vi import RobustVIEngine
    T, R = vi_cases.nonfinite_models(mode, M, S, A, seed=S + M + A)
    eng = RobustVIEngine(mode, T, R, gamma=gamma)
    all_nan = False
    for k in range(1, 7):
        q_ref, sweeps_ref = robust_reference(mode, T, R, gamma, k)
        q, sweeps = eng.solve(k)
        assert sweeps == sweeps_ref == k
        assert same(q, q_ref) and same(eng.v[k & 1], q_ref.max(axis=-1)), k
        all_nan |= bool(np.isnan(q_ref[0]).all())
    assert all_nan


# ------------------------------------------------- np.allclose early exit ----
@pytest.mark.parametrize("nan", [False, True])
@pytest.mark.parametrize("mode,S,A,B", [("deterministic", 400, 4, 1), ("deterministic", 400, 3, 1),
                                        ("sparse", 400, 4, 2), ("sparse", 400, 3, 3)])
def test_allclose_exit_fires_on_equal_infinities_and_never_on_nan(mode, S, A, B, nan):
    """np.isclose(inf, inf) holds and np.isclose(nan, nan) does not: with forced +inf actions the fixed point is met
    early, as numpy meets it; one NaN state keeps every sweep violating, for the whole budget (register and gather
    kernels)."""
    T, R, term, N = vi_cases.forced_and_forbidden(mode, S, A, B, seed=S + A, nan=nan)
    eng = make_engine(mode, T, R, term, N, 0.5)
    q_ref, sweeps = solve_and_compare(eng, mode, T, R, term, 0.5, 80, nxt=N)
    assert np.isinf(q_ref).any() and np.isnan(q_ref).any() == nan
    assert (sweeps == 80) == nan


@pytest.mark.parametrize("nan", [False, True])
def test_robust_allclose_exit_fires_on_equal_infinities_and_never_on_nan(nan):
    """vi_robust_kernel: two models sharing the forced +inf rewards (so the min over models is +inf there too) stop
    early like numpy; a NaN state in both models keeps them running for the whole budget."""
    T1, R, _, _ = vi_cases.forced_and_forbidden("deterministic", 400, 3, 1, seed=1, nan=nan)
    T2, _, _, _ = vi_cases.forced_and_forbidden("deterministic", 400, 3, 1, seed=2, nan=nan)
    q_ref, sweeps = robust_solve_and_compare("deterministic", np.array([T1, T2]), np.array([R, R]), 0.5, 80)
    assert np.isinf(q_ref).any() and np.isnan(q_ref).any() == nan
    assert (sweeps == 80) == nan
