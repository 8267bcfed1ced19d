"""Batched MCTS-DPW engine (device side of MCTSDPWAgent).

The host builds, once per engine and shared by every tree, the tables that keep the kernel bit-exact with no tolerance:
the action and state widening thresholds (the reference's own `k*N**alpha < m`, errors included), the exploration bonus
np.sqrt(np.log(N / n)) (CUDA's fp64 log is only faithfully rounded, which could flip a near-tie of the UCB index), the
closed-loop observation keys sha1(str(s))[:5], the sampled finite-MDP tables and gamma**d."""
import hashlib
import math

import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.mcts import policy_spec
from rl_agents_b200.engine.tables import SampledFiniteTables, gamma_tables, preference_tables, uniform_cdf_table
from rl_agents_b200.engine.tree_engine import TreeEngine

MAX_BONUS_BYTES = 64 << 20          # the exploration-bonus table: episodes (episodes + 1) / 2 doubles
# what the reference raises when a node has no child to select (random_argmax of an empty list, abstract.py:301) or
# to choose among (Generator.choice of an empty list, mcts_dpw.py:176)
EMPTY_ACTIONS_MESSAGE = "zero-size array to reduction operation maximum which has no identity"
EMPTY_STATES_MESSAGE = "a cannot be empty unless no samples are taken"


def obs_key(observation):
    """ChanceNode.get_child's key (mcts_dpw.py:173): sha1(str(observation))[:5] as a 20-bit integer."""
    return int(hashlib.sha1(str(observation).encode("UTF-8")).hexdigest()[:5], 16)


OPEN_LOOP_KEY = obs_key(None)


def observation_keys(n_states):
    """obs_key(s) for every finite state id s."""
    return np.array([obs_key(s) for s in range(n_states)], dtype=np.int32)


def widening_table(k, alpha, n_max, cap):
    """W[N], N in 0..n_max: the largest m <= cap for which `k*N**alpha < m` is false, -1 when there is none.  The
    predicate is false on a down-closed set of m, so a node with m children may widen iff m <= W[N].  The expression is
    the reference's (mcts_dpw.py:122, :175), evaluated in Python, so its errors are the reference's too (0 ** negative
    raises ZeroDivisionError; both tables are read at N = 0 on the first run)."""
    out = np.empty(n_max + 1, dtype=np.int32)
    for N in range(n_max + 1):
        x = k * N ** alpha
        if x != x or x >= cap:
            w = cap                     # NaN compares false with every m
        elif x < 0:
            w = -1
        else:
            w = min(int(math.floor(x)), cap)
        out[N] = w
    return out


def check_bonus_table(episodes):
    nbytes = 8 * episodes * (episodes + 1) // 2
    if nbytes > MAX_BONUS_BYTES:
        raise ValueError("MCTS-DPW's exploration-bonus table for %d episodes needs %.1f MiB, over the %d MiB cap "
                         "(at most %d episodes)" % (episodes, nbytes / 2 ** 20, MAX_BONUS_BYTES >> 20,
                                                    int((math.sqrt(1 + MAX_BONUS_BYTES) - 1) / 2)))


def bonus_table(episodes):
    """np.sqrt(np.log(N / n)) for 1 <= n <= N <= episodes, entry N (N - 1) / 2 + n - 1 (selection_strategy, :150).
    N / n is a correctly rounded division of two integers, as Python's int / int."""
    N = np.repeat(np.arange(1, episodes + 1, dtype=np.int64), np.arange(1, episodes + 1))
    n = np.arange(N.size, dtype=np.int64) - (N * (N - 1)) // 2 + 1
    return np.sqrt(np.log(N / n))


class MCTSDPWEngine(TreeEngine):
    """n_trees independent MCTS-DPW decisions per launch, each tree on its own numpy PCG64 stream."""

    def __init__(self, env_kind, n_trees, n_actions, episodes, horizon, gamma, temperature=1, k_action=3,
                 alpha_action=0.3, k_state=1, alpha_state=0.3, closed_loop=False, mdp=None,
                 rollout_policy="random_available", device="cuda"):
        # everything the configuration can get wrong is refused before any device work
        if env_kind not in (_lib.ENV_FINITE, _lib.ENV_HIGHWAY):
            raise NotImplementedError("MCTS-DPW runs on finite MDPs and HighwayLite")
        self.env_kind = env_kind
        self.n_actions, self.episodes, self.horizon = int(n_actions), int(episodes), int(horizon)
        if self.horizon < 1 or self.episodes < 1:
            raise ValueError("MCTS-DPW needs horizon >= 1 and episodes >= 1 (got %d, %d): the root would stay "
                             "childless and the reference's get_plan returns None" % (self.horizon, self.episodes))
        check_bonus_table(self.episodes)
        self.closed_loop = bool(closed_loop)
        self.capacity = 1 + 2 * self.episodes                 # a run adds at most a chance and a decision node
        rollout_id, rollout_action, rollout_ratio = policy_spec(rollout_policy)
        aw = widening_table(k_action, alpha_action, self.episodes, self.n_actions)
        sw = widening_table(k_state, alpha_state, self.episodes, self.episodes)
        super(MCTSDPWEngine, self).__init__(n_trees, _lib.MCTS_DPW_RESULT_WORDS, device)
        torch = self.torch
        self.gamma_pow = torch.as_tensor(gamma_tables(gamma, self.horizon)[0], device=self.device)
        self.cdf = torch.as_tensor(uniform_cdf_table(self.n_actions), device=self.device)
        self.pref_cdf = torch.as_tensor(preference_tables(self.n_actions, rollout_ratio)[1], device=self.device)
        self.action_widen = torch.as_tensor(aw, device=self.device)
        self.state_widen = torch.as_tensor(sw, device=self.device)
        self.bonus = torch.as_tensor(bonus_table(self.episodes), device=self.device)
        self.tables, self.terminal, self.obs_keys, env_draws, mdp_struct = None, None, None, 0, _lib.FiniteMDPSampled()
        if env_kind == _lib.ENV_FINITE:
            self.tables = SampledFiniteTables(mdp, self.device)
            self.terminal = self.tables.terminal
            self.obs_keys = torch.as_tensor(observation_keys(self.tables.n_states), device=self.device)
            env_draws, mdp_struct = self.tables.env_draws, self.tables.struct()
        self.cfg = _lib.MCTSDPWConfig(
            env_kind, self.n_trees, self.n_actions, self.episodes, self.horizon, self.capacity, rollout_id,
            rollout_action, int(self.closed_loop), OPEN_LOOP_KEY, env_draws, 0, float(temperature),
            self.gamma_pow.data_ptr(), self.cdf.data_ptr(), self.pref_cdf.data_ptr(), self.action_widen.data_ptr(),
            self.state_widen.data_ptr(), self.bonus.data_ptr(),
            self.obs_keys.data_ptr() if self.obs_keys is not None else None,
            self.terminal.data_ptr() if self.terminal is not None else None, mdp_struct)
        self.tree = _lib.MCTSDPWTree(*self._alloc_tree(_lib.MCTS_DPW_TREE_FIELDS, self.capacity))
        self.plan_buf = torch.empty(self.n_trees, dtype=torch.int8, device=self.device)

    def plan(self, root_states, rng_words):
        """root_states: [n_trees] state ids (finite) or [n_trees, 136] words (HighwayLite), on the device."""
        self._load_rng(rng_words)
        _lib.check(self.lib.b2_mcts_dpw_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.rng),
                                             _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def _check(self, res):
        """A sampled probability row that Generator.choice rejects raises its ValueError, as the reference's env step
        does; the other error words raise what the reference raises or a B2Error."""
        err = res[:, 4]
        bad = np.nonzero(err == 2)[0]
        if bad.size:
            self.tables.raise_rejected_row(int(res[bad[0], 5]))
        if (err == 3).any():
            raise ValueError(EMPTY_ACTIONS_MESSAGE)
        if (err == 4).any():
            raise ValueError(EMPTY_STATES_MESSAGE)
        if (err != 0).any():
            raise _lib.B2Error("MCTS-DPW node arena of %d nodes exhausted" % self.capacity)

    def tree_dict(self, tree=0):
        """The nodes of one tree in creation order: parent, first_child, next_sibling, count, kind (0 decision,
        1 chance), key (a chance node's action; a decision node's 20-bit observation key, -1 at the root), value."""
        n = int(self.result[tree, 0].item())
        out = {k: getattr(self, k)[tree, :n].cpu().numpy() for k in _lib.MCTS_DPW_TREE_FIELDS}
        if self.env_kind == _lib.ENV_HIGHWAY and self.closed_loop:
            dec = np.nonzero((out["kind"] == 0) & (out["parent"] >= 0))[0]
            out["key"][dec] = [obs_key(int(t)) for t in out["key"][dec]]      # the device keeps the step count t
        return out
