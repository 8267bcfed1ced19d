"""Host side shared by the tree engines: n_trees independent decisions per launch.

`TreeEngine`: the per-tree engines (MCTS, OLOP, MDP-GapE, BRUE, sparse sampling, GBOP-D), each tree on its own numpy
PCG64 stream, which the kernel advances in place.  `HostTieEngine`: the value-bound engines (OPD, its wavefront and
speculative variants, GBOP-T), whose greedy plan the device follows until a tie that the host breaks with the
planner's numpy generator."""
import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import gamma_tables, terminal_bonus_table

# node fields stored as int32; every other node field is float64
INT32_FIELDS = ("parent", "first_child", "next_sibling", "count", "meta", "kind", "key", "depth", "obs", "action",
                "flags", "state")


def decode_action(meta):
    """The incoming action in bits 0-7 of a node's meta word; 0xff (no incoming action: the root) -> -1."""
    action = (meta & 0xff).astype(int)
    action[action == 0xff] = -1
    return action


class TreeEngine(object):
    def __init__(self, n_trees, result_words, device, pcg64=True):
        """pcg64: allocate the per-tree PCG64 state the kernel advances (`rng`)."""
        import torch
        self.torch = torch
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.n_trees = int(n_trees)
        self.result = torch.empty((self.n_trees, result_words), dtype=torch.int32, device=self.device)
        if pcg64:
            self.rng = torch.empty((self.n_trees, _lib.PCG64_STATE_WORDS), dtype=torch.int64, device=self.device)

    def _alloc_tree(self, fields, capacity):
        """One [n_trees, capacity] node array per field name, set as an attribute; -> their data pointers."""
        torch = self.torch
        for n in fields:
            setattr(self, n, torch.empty((self.n_trees, capacity), device=self.device,
                                         dtype=torch.int32 if n in INT32_FIELDS else torch.float64))
        return [getattr(self, n).data_ptr() for n in fields]

    def _load_rng(self, rng_words):
        """rng_words: uint64 [n_trees, 6] (pcg64_words per tree)."""
        self.rng.copy_(self.torch.from_numpy(np.ascontiguousarray(rng_words).view(np.int64)))

    def _result(self):
        """Synchronise; -> the result words [n_trees, words] as a numpy array."""
        return self.result.cpu().numpy()

    def _check(self, res):
        """Raise what the reference raises for an error the result words report."""

    def _plans(self, res):
        """One [action] per tree: result word 3 (-1: no plan)."""
        return [[int(a)] for a in res[:, 3]]

    def finish(self):
        """Synchronise; -> (plans, result words [n_trees, words], PCG64 words after the search)."""
        res = self._result()
        self._check(res)
        return self._plans(res), res, self.rng.cpu().numpy().view(np.uint64)


class HostTieEngine(TreeEngine):
    """budget // n_actions expansions of n_actions children per tree (deterministic.py:118).  Result words: 4 a reward
    outside [0, 1], 5 the length of the device's plan, 6 the node where a tie stopped it (-1: none)."""
    TIE_WALKS = 1       # greedy walks from the tie node per tree; the last one is the plan's tail

    def __init__(self, n_trees, n_actions, budget, gamma, terminal_reward, device, gamma_pow_div=False):
        """gamma_pow_div: also build the gamma**d / (1 - gamma) table (the OPD kernels read it)."""
        super(HostTieEngine, self).__init__(n_trees, _lib.OPD_RESULT_WORDS, device, pcg64=False)
        torch = self.torch
        self.n_actions = int(n_actions)
        self.n_expansions = int(budget) // self.n_actions
        self.capacity = 1 + self.n_expansions * self.n_actions
        self.plan_capacity = self.n_expansions + 1
        gp, gd = gamma_tables(gamma, self.n_expansions + 2)
        self.gamma_pow = torch.as_tensor(gp, device=self.device)
        if gamma_pow_div:
            self.gamma_pow_div = torch.as_tensor(gd, device=self.device)
        self.terminal_bonus = torch.as_tensor(terminal_bonus_table(terminal_reward, gamma, self.n_expansions + 2),
                                              device=self.device)
        self.plan_buf = torch.empty((self.n_trees, self.plan_capacity), dtype=torch.int8, device=self.device)

    def _check(self, res):
        if (res[:, 4] != 0).any():
            raise ValueError("This planner assumes that all rewards are normalized in [0, 1]")  # deterministic.py:46-47

    def finish(self, np_randoms=None):
        """Synchronise; -> (plans, result words).  A tie in get_plan is broken on the host with the planner's RNG
        (np_randoms[tree]; default: a fresh generator) exactly as abstract.py:304-311 does."""
        res = self._result()
        self._check(res)
        plans_dev = self.plan_buf.cpu().numpy()
        plans = []
        for i in range(self.n_trees):
            plan = plans_dev[i, :res[i, 5]].astype(int).tolist()
            if res[i, 6] >= 0:
                rng = np_randoms[i] if np_randoms is not None else np.random.default_rng()
                for _ in range(self.TIE_WALKS):
                    tail = self._greedy_walk(i, int(res[i, 6]), rng)
                plan += tail
            plans.append(plan)
        return plans, res

    def _greedy_walk(self, tree, node, rng):
        """Down the children of highest value_lower from `node`, a tie broken by rng.choice; -> the actions."""
        fc = self.first_child[tree].cpu().numpy()
        meta = self.meta[tree].cpu().numpy()
        lower = self.lower[tree].cpu().numpy()
        plan = []
        while fc[node] >= 0:
            n = (meta[node] >> 8) & 0xff
            x = lower[fc[node]:fc[node] + n]
            indices = np.nonzero(x == np.amax(x))[0]
            node = fc[node] + int(rng.choice(indices))
            plan.append(int(meta[node] & 0xff))
        return plan
