"""Batched closed-loop episodes on finite MDPs: the device env step b2_finite_step (csrc/finite_step.cu) against the host
FiniteMDPEnv.step, and evaluation.run_batched_episodes(..., env="finite") against one drop-in agent per episode stepping
its own host FiniteMDPEnv.  Every comparison is exact: states, rewards as float64, done flags, actions, lengths and the
PCG64 words of every planner and env generator."""
import copy
import os

import numpy as np
import pytest

from tests.mdp_gape_stochastic_cases import MDPS

GOLDEN = np.load(os.path.join(os.path.dirname(__file__), "golden", "finite_mdps.npz"))


def mdp_spec(name):
    """name -> (mode, transition, reward, terminal, next) of a golden deterministic MDP or a stochastic case MDP."""
    if name in MDPS:
        m = MDPS[name]
        return m["mode"], m["transition"], m["reward"], m["terminal"], m["next"]
    return "deterministic", GOLDEN[name + "_T"], GOLDEN[name + "_R"], GOLDEN[name + "_term"], None


def make_env(name, state=0, seed=None):
    from rl_agents_b200.envs import FiniteMDPEnv
    mode, T, R, term, nxt = mdp_spec(name)
    return FiniteMDPEnv(T, R, term, mode=mode, nxt=nxt, state=state, seed=seed)


def words_of(gen):
    from rl_agents_b200.engine.mcts import pcg64_words
    return pcg64_words(gen)


# -- the step kernel --------------------------------------------------------------------------------------------------

class DeviceStep(object):
    """b2_finite_step on one MDP, for n episodes."""

    def __init__(self, env):
        import torch
        from rl_agents_b200 import _lib
        from rl_agents_b200.engine.tables import SampledFiniteTables
        self.torch, self._lib, self.lib = torch, _lib, _lib.load()
        self.tables = SampledFiniteTables(env.mdp, "cuda")

    def __call__(self, states, actions, alive, words):
        """-> (rc, states, reward, flags, bad_row, words) after one call; outputs of masked episodes keep a sentinel."""
        torch, _lib = self.torch, self._lib
        n = len(states)
        st = torch.as_tensor(np.asarray(states, np.int32), device="cuda")
        act = torch.as_tensor(np.asarray(actions, np.int32), device="cuda")
        al = torch.as_tensor(np.asarray(alive, np.uint8), device="cuda")
        w = torch.as_tensor(np.ascontiguousarray(words, np.uint64).view(np.int64), device="cuda")
        rew = torch.full((n,), -7.0, dtype=torch.float64, device="cuda")
        flg = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        bad = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        t = self.tables
        rc = self.lib.b2_finite_step(t.struct(), _lib.ptr(t.terminal), t.env_draws, _lib.ptr(st), _lib.ptr(act),
                                     _lib.ptr(al), _lib.ptr(w), _lib.ptr(rew), _lib.ptr(flg), _lib.ptr(bad), n,
                                     _lib.current_stream())
        return (rc, st.cpu().numpy(), rew.cpu().numpy(), flg.cpu().numpy(), bad.cpu().numpy(),
                w.cpu().numpy().view(np.uint64))


def host_step(env, state, action, gen):
    """FiniteMDPEnv.step from `state` with generator `gen` -> (next state, reward, done) or the ValueError raised."""
    env.mdp.state, env.np_random = int(state), gen
    try:
        s2, r, done, _, _ = env.step(int(action))
    except ValueError as e:
        return e
    return s2, r, done


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["large1", "trap", "loop", "garnet50", "dense6", "dup20", "term40", "unreached_bad20"])
def test_step_kernel_equals_host_step(name):
    """3000 episodes from random states, actions and generator seeds, chained for 6 steps with a random alive mask:
    every live episode equals FiniteMDPEnv.step bit for bit, generator words included; masked ones are not touched."""
    env = make_env(name)
    S, A = env.mdp.reward.shape
    n, rng = 3000, np.random.default_rng(17)
    reachable = S - 1 if name == "unreached_bad20" else S           # state 19 of unreached_bad20 has the NaN row
    states = rng.integers(0, reachable, n)
    gens = [np.random.default_rng(int(s)) for s in rng.integers(0, 2 ** 32, n)]
    words = np.stack([words_of(g) for g in gens])
    step = DeviceStep(env)
    done_seen = 0
    for _ in range(6):
        actions = rng.integers(0, A, n)
        alive = rng.uniform(size=n) < 0.8
        rc, st, rew, flg, bad, w = step(states, actions, alive, words)
        assert rc == 0
        for i in range(n):
            if not alive[i]:
                assert (st[i], rew[i], flg[i], bad[i]) == (states[i], -7.0, -7, -7)
                assert (w[i] == words[i]).all()
                continue
            s2, r, done = host_step(env, states[i], actions[i], gens[i])
            assert (st[i], rew[i].tobytes(), flg[i], bad[i]) == (s2, np.float64(r).tobytes(), int(done), -1), i
            assert (w[i] == words_of(gens[i])).all(), i
            done_seen += done
        states, words = st, w
    if name in ("trap", "term40"):
        assert done_seen > 0


@pytest.mark.gpu
def test_step_kernel_rejected_row_raises_numpys_error():
    """bad20's row (0, 1) is NaN: the step leaves the state and generator alone, reports the row, and the host raises
    numpy's own ValueError, message for message with FiniteMDPEnv.step; the other episodes step as usual."""
    env = make_env("bad20")
    step = DeviceStep(env)
    gens = [np.random.default_rng(s) for s in (3, 4)]
    words = np.stack([words_of(g) for g in gens])
    rc, st, rew, flg, bad, w = step([0, 0], [1, 2], [1, 1], words)
    assert rc == 0
    assert (st[0], rew[0], flg[0], bad[0]) == (0, 0.0, 0, 1) and (w[0] == words[0]).all()
    assert bad[1] == -1 and st[1] == host_step(env, 0, 2, gens[1])[0] and (w[1] == words_of(gens[1])).all()
    expected = host_step(env, 0, 1, np.random.default_rng(3))
    assert isinstance(expected, ValueError)
    with pytest.raises(ValueError) as e:
        step.tables.raise_rejected_row(int(bad[0]))
    assert str(e.value) == str(expected)


@pytest.mark.gpu
def test_step_kernel_refusals():
    """The C ABI refuses null pointers, an empty batch, a bad env_draws, missing tables, and a live episode's state or
    action outside the MDP -- without stepping any episode; a masked episode's ids are not read."""
    import torch
    from rl_agents_b200 import _lib
    env = make_env("garnet50")
    step = DeviceStep(env)
    lib, t = step.lib, step.tables
    words = np.stack([words_of(np.random.default_rng(s)) for s in range(3)])
    for states, actions, alive, what in (([0, -1, 2], [0, 0, 0], [1, 1, 1], "episode 1: state outside [0, 50)"),
                                         ([0, 50, 2], [0, 0, 0], [1, 1, 1], "episode 1: state outside [0, 50)"),
                                         ([0, 1, 2], [0, 0, 4], [1, 1, 1], "episode 2: action outside [0, 4)"),
                                         ([0, 1, 2], [-1, 0, 0], [1, 1, 1], "episode 0: action outside [0, 4)")):
        rc, st, rew, flg, bad, w = step(states, actions, alive, words)
        assert rc == 1
        assert lib.b2_last_error().decode() == "invalid argument: " + what
        assert (st == states).all() and (rew == -7.0).all() and (bad == -7).all() and (w == words).all()
    rc = step([0, 99, 2], [0, 9, 1], [1, 0, 1], words)[0]
    assert rc == 0                                           # episode 1 is masked: its ids are never read
    st = torch.zeros(2, dtype=torch.int32, device="cuda")
    buf = torch.zeros(2, dtype=torch.float64, device="cuda")
    act, flg, bad = (torch.zeros(2, dtype=torch.int32, device="cuda") for _ in range(3))
    u8 = torch.ones(2, dtype=torch.uint8, device="cuda")
    w = torch.zeros((2, 6), dtype=torch.int64, device="cuda")
    p = _lib.ptr
    base = dict(mdp=t.struct(), terminal=p(t.terminal), draws=1, states=p(st), actions=p(act), alive=p(u8), rng=p(w),
                reward=p(buf), flags=p(flg), bad=p(bad), n=2)

    def call(**over):
        a = dict(base, **over)
        return lib.b2_finite_step(a["mdp"], a["terminal"], a["draws"], a["states"], a["actions"], a["alive"], a["rng"],
                                  a["reward"], a["flags"], a["bad"], a["n"], _lib.current_stream())
    assert call() == 0
    torch.cuda.synchronize()
    no_cdf = t.struct()
    no_cdf.cdf = None
    wrong_shape = t.struct()
    wrong_shape.n_states = 0
    for over, msg in ((dict(mdp=None), "null pointer"), (dict(states=None), "null pointer"),
                      (dict(actions=None), "null pointer"), (dict(alive=None), "null pointer"),
                      (dict(reward=None), "null pointer"), (dict(flags=None), "null pointer"),
                      (dict(bad=None), "null pointer"), (dict(n=0), "n must be >= 1"),
                      (dict(terminal=None), "finite MDP tables missing"), (dict(mdp=no_cdf), "finite MDP tables missing"),
                      (dict(mdp=wrong_shape), "bad finite MDP shape"), (dict(draws=2), "env_draws must be 0 or 1"),
                      (dict(rng=None), "null pointer: env_rng is needed when the steps draw")):
        assert call(**over) == 1, over
        assert lib.b2_last_error().decode() == "invalid argument: " + msg, over
    assert call(draws=0, rng=None) == 0                      # a deterministic step reads no generator
    torch.cuda.synchronize()


# -- the batched harness against one agent per episode ---------------------------------------------------------------

DETERMINISTIC = ["large1", "trap", "loop"]
SAMPLED = ["garnet50", "dense6", "dup20", "term40"]
KL = {"upper_bound": {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)"},
      "continuation_type": "uniform"}
# planner -> (agent class path, budget, keywords, MDPs)
PLANNERS = {
    "opd": ("deterministic.DeterministicPlannerAgent", 40, {}, DETERMINISTIC),
    "gbop": ("state_aware.StateAwarePlannerAgent", 40, {}, DETERMINISTIC),
    "gbopd": ("graph_based.GraphBasedPlannerAgent", 40, {}, DETERMINISTIC),
    "brue": ("brue.BRUEAgent", 40, {}, DETERMINISTIC),
    "mcts": ("mcts.MCTSAgent", 40, {}, DETERMINISTIC + SAMPLED),
    "olop": ("olop.OLOPAgent", 40, KL, DETERMINISTIC + SAMPLED),
    "mdp_gape": ("mdp_gape.MDPGapEAgent", 40, {"max_next_states_count": 6}, DETERMINISTIC + SAMPLED),
    "sparse_sampling": ("sparse_sampling.SparseSamplingAgent", 0, {"horizon": 2, "C": 2}, DETERMINISTIC + SAMPLED),
    "mcts_dpw": ("mcts_dpw.MCTSDPWAgent", 40, {}, DETERMINISTIC + SAMPLED),
    "platypoos": ("platypoos.PlaTyPOOSAgent", 40, {"horizon": 3}, DETERMINISTIC + SAMPLED),
    "vi": (None, 30, {}, DETERMINISTIC + SAMPLED),
}
CASES = [(p, m) for p, spec in PLANNERS.items() for m in spec[3]]
N, STEPS, GAMMA, PLANNER_SEED, ENV_SEED = 24, 8, 0.8, 40, 900


def make_agent(planner, env, budget, kw):
    import importlib
    if planner == "vi":
        from rl_agents_b200.agents.dynamic_programming.value_iteration import ValueIterationAgent
        return ValueIterationAgent(env, {"gamma": GAMMA, "iterations": budget})
    module, cls = PLANNERS[planner][0].rsplit(".", 1)
    agent_cls = getattr(importlib.import_module("rl_agents_b200.agents.tree_search." + module), cls)
    return agent_cls(env, dict(copy.deepcopy(kw), budget=budget, gamma=GAMMA))


def agent_episodes(planner, name, starts):
    """One agent per episode on its own host FiniteMDPEnv -> dict of per-episode results, or the exception raised."""
    _, budget, kw, _ = PLANNERS[planner]
    out = {"actions": [], "rewards": [], "final_states": [], "planner_words": [], "env_words": []}
    for i, s0 in enumerate(starts):
        env = make_env(name, int(s0), seed=ENV_SEED + i)
        try:
            agent = make_agent(planner, env, budget, kw)
            agent.seed(PLANNER_SEED + i)
            acts, rews = [], []
            for _ in range(STEPS):
                a = int(agent.act(env.mdp.state))
                s2, r, done, _, _ = env.step(a)
                acts.append(a)
                rews.append(r)
                if done:
                    break
        except Exception as e:          # the harness must raise the same
            return e
        out["actions"].append(acts)
        out["rewards"].append(rews)
        out["final_states"].append(env.mdp.state)
        out["planner_words"].append(words_of(agent.planner.np_random) if planner != "vi" else None)
        out["env_words"].append(words_of(env.np_random))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("planner,name", CASES)
def test_batched_episodes_equal_per_episode_agents(planner, name):
    from rl_agents_b200.evaluation import run_batched_episodes
    _, budget, kw, _ = PLANNERS[planner]
    S = mdp_spec(name)[2].shape[0]
    starts = np.arange(N) % S
    expected = agent_episodes(planner, name, starts)
    run = lambda: run_batched_episodes(planner, list(range(N)), budget, GAMMA, max_steps=STEPS, env="finite",
                                       planner_seed=PLANNER_SEED, mdp=make_env(name), start_states=starts,
                                       env_seed=ENV_SEED, **copy.deepcopy(kw))
    if isinstance(expected, Exception):
        assert name == "trap", expected                       # trap's rewards span [-1, 1]
        with pytest.raises(type(expected)) as e:
            run()
        assert str(e.value) == str(expected)
        return
    out = run()
    assert not out["crashed"].any()
    for i in range(N):
        k = len(expected["actions"][i])
        assert out["lengths"][i] == k, i
        assert out["actions"][i, :k].tolist() == expected["actions"][i], i
        assert (out["actions"][i, k:] == -1).all()
        assert out["rewards"][i, :k].tobytes() == np.array(expected["rewards"][i], np.float64).tobytes(), i
        total = 0.0
        for r in expected["rewards"][i]:                        # sequentially, as the agent's caller adds them
            total += r
        assert out["returns"][i] == total, i
        assert out["final_states"][i] == expected["final_states"][i], i
        assert (out["env_words"][i] == expected["env_words"][i]).all(), i
        if planner != "vi":
            assert (out["planner_words"][i] == expected["planner_words"][i]).all(), i
    if name in ("term40", "trap"):
        assert len(set(out["lengths"].tolist())) > 1          # episodes end at different steps


def test_refusals():
    """Stochastic and sparse MDPs for the planners whose agents refuse them, and the GBOP planners on the scene envs:
    NotImplementedError before any device work."""
    from rl_agents_b200.evaluation import run_batched_episodes
    for planner in ("opd", "brue", "gbop", "gbopd"):
        for name in ("dense6", "garnet50"):
            with pytest.raises(NotImplementedError):
                run_batched_episodes(planner, [0, 1], 40, 0.8, env="finite", mdp=make_env(name))
    for planner in ("gbop", "gbopd"):
        for env in ("highway", "intersection"):
            with pytest.raises(NotImplementedError):
                run_batched_episodes(planner, [0], 40, 0.8, max_steps=1, env=env)
    with pytest.raises(ValueError):
        run_batched_episodes("opd", [0], 40, 0.8, max_steps=1, env="nowhere")
