"""Host side shared by the per-tree engines (MCTS, OLOP, MDP-GapE, BRUE, sparse sampling): n_trees independent
decisions per launch, each tree on its own numpy PCG64 stream, which the kernel advances in place."""
import numpy as np

from rl_agents_b200 import _lib

# node fields stored as int32; every other node field is float64
INT32_FIELDS = ("parent", "first_child", "next_sibling", "count", "meta", "kind", "key", "depth")


def decode_action(meta):
    """The incoming action in bits 0-7 of a node's meta word; 0xff (no incoming action: the root) -> -1."""
    action = (meta & 0xff).astype(int)
    action[action == 0xff] = -1
    return action


class TreeEngine(object):
    def __init__(self, n_trees, result_words, device):
        import torch
        self.torch = torch
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.n_trees = int(n_trees)
        self.result = torch.empty((self.n_trees, result_words), dtype=torch.int32, device=self.device)
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

    def _check(self, res):
        """Raise what the reference raises for an error the result words report."""

    def _plans(self, res):
        """One [action] per tree: result word 3 (-1: no plan)."""
        return [[int(a)] for a in res[:, 3]]

    def finish(self):
        """Synchronise; -> (plans, result words [n_trees, words], PCG64 words after the search)."""
        res = self.result.cpu().numpy()
        self._check(res)
        return self._plans(res), res, self.rng.cpu().numpy().view(np.uint64)
