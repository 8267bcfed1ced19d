"""Pin the numpy comparator of value iteration (oracle.planners.value_iteration / robust_value_iteration) to the
UNMODIFIED reference agents (ValueIterationAgent, RobustValueIterationAgent) on the MDPs with infinite rewards of
tests/vi_cases.py: the same Q, NaN included, and the same number of Bellman operator applications.  So the device
kernels, tested against the comparator, follow the reference's NaN and infinity semantics: its max over actions and
min over models propagate NaN, and its np.allclose exit holds on equal infinities and never on NaN."""
import numpy as np
import pytest

from oracle import envs, planners, ref_loader
from tests import vi_cases

pytestmark = pytest.mark.skipif(not ref_loader.reference_available(), reason="needs the reference tree")


def counted(agent):
    """Count the agent's Bellman operator applications: the comparator's sweep count."""
    calls = [0]
    bellman = agent.bellman_expectation

    def wrapper(value):
        calls[0] += 1
        return bellman(value)
    agent.bellman_expectation = wrapper
    return calls


def reference_vi(mode, T, R, term, gamma, iterations, nxt=None):
    ref_loader.load_reference()
    from rl_agents.agents.dynamic_programming.value_iteration import ValueIterationAgent
    env = envs.FiniteMDPLite(T, R, term, mode=mode, nxt=nxt)
    with np.errstate(invalid="ignore", over="ignore"):
        agent = ValueIterationAgent(env, {"gamma": gamma, "iterations": iterations})
        calls = counted(agent)
        return agent.get_state_action_value(), calls[0]


def reference_robust_vi(mode, T, R, gamma, iterations):
    ref_loader.load_reference()
    from rl_agents.agents.dynamic_programming.robust_value_iteration import RobustValueIterationAgent
    models = [{"mode": mode, "transition": t, "reward": r} for t, r in zip(T, R)]
    with np.errstate(invalid="ignore", over="ignore"):
        agent = RobustValueIterationAgent(None, {"gamma": gamma, "iterations": iterations, "models": models})
        calls = counted(agent)
        return agent.get_state_action_value(), calls[0]


def assert_comparator_matches(mode, T, R, term, gamma, iterations, nxt=None):
    with np.errstate(invalid="ignore", over="ignore"):
        q, sweeps = planners.value_iteration(mode, T, R, term, gamma, iterations, nxt=nxt)
    q_ref, sweeps_ref = reference_vi(mode, T, R, term, gamma, iterations, nxt=nxt)
    assert sweeps == sweeps_ref
    assert np.array_equal(q, q_ref, equal_nan=True)
    return q, sweeps


def test_three_state_mdp():
    c = vi_cases.THREE_STATE
    q, _ = assert_comparator_matches("deterministic", c["transition"], c["reward"], c["terminal"], 0.9, 4)
    assert np.isnan(q[:2]).all() and (q[2] == np.inf).all()


@pytest.mark.parametrize("gamma", [0.9, 0.0])
@pytest.mark.parametrize("mode,S,A,B", [("deterministic", 60, 4, 1), ("deterministic", 60, 3, 1), ("sparse", 60, 4, 4),
                                        ("sparse", 60, 3, 5), ("stochastic", 40, 3, None)])
def test_nonfinite_mdp(mode, S, A, B, gamma):
    T, R, term, N = vi_cases.nonfinite_mdp(mode, S, A, B, seed=S + A + (B or 0))
    q, _ = assert_comparator_matches(mode, T, R, term, gamma, 6, nxt=N)
    assert np.isnan(q).any()


@pytest.mark.parametrize("gamma", [0.9, 0.0])
@pytest.mark.parametrize("mode,M,S,A", [("deterministic", 3, 60, 3), ("deterministic", 2, 60, 1),
                                        ("stochastic", 2, 40, 3)])
def test_nonfinite_robust(mode, M, S, A, gamma):
    T, R = vi_cases.nonfinite_models(mode, M, S, A, seed=S + M + A)
    with np.errstate(invalid="ignore", over="ignore"):
        q, sweeps = planners.robust_value_iteration(mode, T, R, gamma, 6)
    q_ref, sweeps_ref = reference_robust_vi(mode, T, R, gamma, 6)
    assert sweeps == sweeps_ref
    assert np.array_equal(q, q_ref, equal_nan=True)
    assert np.isnan(q[0]).all()


@pytest.mark.parametrize("nan", [False, True])
@pytest.mark.parametrize("mode,A,B", [("deterministic", 4, 1), ("sparse", 3, 3)])
def test_allclose_exit_on_infinities_and_nan(mode, A, B, nan):
    T, R, term, N = vi_cases.forced_and_forbidden(mode, 200, A, B, seed=7, nan=nan)
    q, sweeps = assert_comparator_matches(mode, T, R, term, 0.5, 80, nxt=N)
    assert np.isinf(q).any() and np.isnan(q).any() == nan
    assert (sweeps == 80) == nan
