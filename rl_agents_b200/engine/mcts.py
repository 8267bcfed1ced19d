"""Batched MCTS engine (device side of MCTSAgent).

A finite MDP in mode "deterministic" runs b2_mcts_plan / b2_mcts_plan_wave on FiniteTables; in mode "stochastic" or
"sparse" it runs b2_mcts_plan_sampled / b2_mcts_plan_wave_sampled on SampledFiniteTables.  The reference never reseeds
its env copies, so those take the live env's generator words (`env_words`), which every episode's copy starts from."""
import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.engine.tables import finite_model, gamma_tables, preference_tables, uniform_cdf_table
from rl_agents_b200.engine.tree_engine import TreeEngine, decode_action

POLICIES = {"random_available": 0, "random": 1, "preference": 2}


def policy_spec(policy):
    """"random" | "random_available" | ("preference", action, ratio) -> (kernel policy id, action, ratio)"""
    if isinstance(policy, (tuple, list)):
        kind, action, ratio = policy
        if kind != "preference":
            raise ValueError("Unknown policy type")
        return POLICIES[kind], int(action), ratio
    if policy not in ("random_available", "random"):
        raise ValueError("Unknown policy type")
    return POLICIES[policy], -1, 2


def pcg64_words(gen):
    """numpy Generator(PCG64) state -> the 6 x uint64 the kernel advances."""
    st = gen.bit_generator.state
    if st["bit_generator"] != "PCG64":
        raise ValueError("the planner RNG must be a numpy PCG64 Generator")
    s, inc = st["state"]["state"], st["state"]["inc"]
    m = (1 << 64) - 1
    return np.array([s >> 64, s & m, inc >> 64, inc & m, st["has_uint32"], st["uinteger"]], dtype=np.uint64)


def set_pcg64_words(gen, w):
    st = gen.bit_generator.state
    w = [int(x) for x in w]
    st["state"]["state"] = (w[0] << 64) | w[1]
    st["state"]["inc"] = (w[2] << 64) | w[3]
    st["has_uint32"], st["uinteger"] = w[4], w[5]
    gen.bit_generator.state = st


def reroot_arrays(arrays, n, action):
    """step_by_subtree (abstract.py:195-206): keep the sub-tree under the root's child `action`, re-indexed
    breadth first (children of a node stay contiguous and in order) with that child as node 0.
    arrays: dict of numpy arrays parent / first_child / count / meta / value / prior (first n entries valid).
    Returns (new arrays dict, number of kept nodes) -- (None, 0) when the action was never expanded.
    The specification of the device re-root b2_mcts_reroot (MCTSEngine.reroot)."""
    fc, meta = arrays["first_child"], arrays["meta"]
    root_child = -1
    if fc[0] >= 0:
        for c in range(fc[0], fc[0] + ((meta[0] >> 8) & 0xff)):
            if (meta[c] & 0xff) == action:
                root_child = c
    if root_child < 0:
        return None, 0
    order, new_parent = [root_child], [-1]
    head = 0
    new_first = []
    while head < len(order):
        old = order[head]
        k = (meta[old] >> 8) & 0xff if fc[old] >= 0 else 0
        new_first.append(len(order) if k else -1)
        for c in range(fc[old], fc[old] + k):
            order.append(c)
            new_parent.append(head)
        head += 1
    order = np.array(order)
    out = {"parent": np.array(new_parent, dtype=np.int32), "first_child": np.array(new_first, dtype=np.int32),
           "count": arrays["count"][order].copy(), "meta": arrays["meta"][order].copy(),
           "value": arrays["value"][order].copy(), "prior": arrays["prior"][order].copy()}
    out["meta"][0] = (out["meta"][0] & ~0xff) | 0xff          # the new root has no incoming action
    return out, len(order)


class MCTSEngine(TreeEngine):
    """n_trees independent MCTS decisions per launch; every tree consumes its
    own numpy PCG64 stream exactly as the reference planner would."""

    def __init__(self, env_kind, n_trees, n_actions, episodes, horizon, gamma, temperature, mdp=None,
                 rollout_policy="random_available", prior_policy="random_available", device="cuda", capacity=None):
        super(MCTSEngine, self).__init__(n_trees, _lib.MCTS_RESULT_WORDS, device)
        torch = self.torch
        rollout_id, rollout_action, rollout_ratio = policy_spec(rollout_policy)
        prior_id, prior_action, prior_ratio = policy_spec(prior_policy)
        self.n_actions = int(n_actions)
        self.episodes, self.horizon = int(episodes), int(horizon)
        self.capacity = max(int(capacity or 0), 1 + self.episodes * self.n_actions)
        gp, _ = gamma_tables(gamma, self.horizon + 1)
        self.gamma_pow = torch.as_tensor(gp, device=self.device)
        self.cdf = torch.as_tensor(uniform_cdf_table(self.n_actions), device=self.device)
        self.sampled, self.tables, finite_mdp = finite_model(env_kind, mdp, self.device)
        if self.sampled:
            self.env_rng = torch.empty((self.n_trees, _lib.PCG64_STATE_WORDS), dtype=torch.int64, device=self.device)
        self.tree = _lib.MCTSTree(*self._alloc_tree(_lib.MCTS_TREE_FIELDS, self.capacity))
        self._spare = None      # reroot's second arena
        self.pref_prior = torch.as_tensor(preference_tables(self.n_actions, prior_ratio)[0], device=self.device)
        self.pref_cdf = torch.as_tensor(preference_tables(self.n_actions, rollout_ratio)[1], device=self.device)
        self.cfg = _lib.MCTSConfig(env_kind, self.n_trees, self.n_actions, self.episodes, self.horizon, self.capacity,
                                   rollout_id, prior_id, float(temperature),
                                   self.gamma_pow.data_ptr(), self.cdf.data_ptr(),
                                   finite_mdp, prior_action, rollout_action, self.pref_prior.data_ptr(), self.pref_cdf.data_ptr(), None)
        self.resume = torch.zeros(self.n_trees, dtype=torch.int32, device=self.device)
        self.plan_buf = torch.empty((self.n_trees, max(self.horizon, 1)), dtype=torch.int8, device=self.device)

    def plan(self, root_states, rng_words, resume_nodes=None, env_words=None):
        """rng_words: uint64 [n_trees, 6] numpy (pcg64_words per tree).  resume_nodes: per-tree node counts of
        re-rooted sub-trees already in the arrays (see reroot), or None for fresh trees.  env_words (sampled MDPs
        only): uint64 [6] or [n_trees, 6], pcg64_words of the live env's generator that each tree's env copies start
        from."""
        self._load_rng(rng_words)
        if resume_nodes is None:
            self.cfg.resume_nodes = None
        else:
            self.resume.copy_(self.torch.as_tensor(np.asarray(resume_nodes, dtype=np.int32)))
            self.cfg.resume_nodes = self.resume.data_ptr()
        if self.sampled:
            if env_words is None:
                raise ValueError("MCTS on a stochastic finite MDP needs the env generator's words (env_words)")
            w = np.array(np.broadcast_to(np.asarray(env_words, dtype=np.uint64), (self.n_trees, _lib.PCG64_STATE_WORDS)))
            self.env_rng.copy_(self.torch.from_numpy(w.view(np.int64)))
            t = self.tables
            _lib.check(self.lib.b2_mcts_plan_sampled(
                self.cfg, t.struct(), _lib.ptr(t.terminal), t.env_draws, _lib.ptr(self.env_rng),
                _lib.ptr(root_states), self.tree, _lib.ptr(self.rng), _lib.ptr(self.plan_buf), _lib.ptr(self.result),
                _lib.current_stream()))
            return
        _lib.check(self.lib.b2_mcts_plan(self.cfg, _lib.ptr(root_states), self.tree, _lib.ptr(self.rng),
                                         _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def _check(self, res):
        if self.sampled:
            bad = np.nonzero(res[:, 3] == 1)[0]
            if bad.size:
                self.tables.raise_rejected_row(int(res[bad[0], 4]))

    def _plans(self, res):
        plans = self.plan_buf.cpu().numpy()
        return [plans[i, :res[i, 1]].astype(int).tolist() for i in range(self.n_trees)]

    def _arena(self):
        return tuple(getattr(self, k) for k in _lib.MCTS_TREE_FIELDS)

    def _use_arena(self, arena):
        for k, t in zip(_lib.MCTS_TREE_FIELDS, arena):
            setattr(self, k, t)
        self.tree = _lib.MCTSTree(*[t.data_ptr() for t in arena])

    def reroot(self, actions, sources=None, source=None):
        """step_strategy "subtree" for every tree in one launch (b2_mcts_reroot): tree j becomes the sub-tree of tree
        sources[j] (default j) of `source` (default this engine), as its last plan left it, under that tree's root
        child of action actions[j] -- reroot_arrays, on the device.  Re-rooting within this engine writes a spare
        arena, allocated on first use, and swaps it in; from another engine (the survivors of a batch gathered into a
        smaller one) it writes this engine's arena.
        -> kept, int32 numpy [n_trees]: the node counts to pass as plan(resume_nodes=...); 0 starts a new tree (the
        action is < 0 or was never expanded, or the sub-tree and this engine's episodes * n_actions new nodes would
        not fit), -1 reports a source index outside `source`'s trees."""
        torch = self.torch
        src = self if source is None else source
        if src is self:
            if self._spare is None:
                self._spare = tuple(torch.empty_like(t) for t in self._arena())
            dst = _lib.MCTSTree(*[t.data_ptr() for t in self._spare])
        else:
            dst = self.tree
        act = torch.as_tensor(np.asarray(actions, dtype=np.int32).reshape(self.n_trees), device=self.device)
        idx = None if sources is None else \
            torch.as_tensor(np.asarray(sources, dtype=np.int32).reshape(self.n_trees), device=self.device)
        _lib.check(self.lib.b2_mcts_reroot(src.tree, src.n_trees, src.capacity, _lib.ptr(src.result),
                                           _lib.MCTS_RESULT_WORDS, dst, self.n_trees, self.capacity, _lib.ptr(idx),
                                           _lib.ptr(act), self.episodes * self.n_actions, _lib.ptr(self.resume),
                                           _lib.current_stream()))
        if src is self:
            spare, self._spare = self._spare, self._arena()
            self._use_arena(spare)
        return self.resume.cpu().numpy()

    def tree_dict(self, tree=0):
        n = int(self.result[tree, 0].item())
        meta = self.meta[tree, :n].cpu().numpy()
        return {"parent": self.parent[tree, :n].cpu().numpy(), "action": decode_action(meta),
                "count": self.count[tree, :n].cpu().numpy(), "value": self.value[tree, :n].cpu().numpy(),
                "prior": self.prior[tree, :n].cpu().numpy(),
                "first_child": self.first_child[tree, :n].cpu().numpy(), "n_children": (meta >> 8) & 0xff}


class MCTSWaveEngine(object):
    """ONE MCTS decision searched by the whole GPU in waves of `width` episodes (b2_mcts_plan_wave);
    bit-identical with the specification oracle/planners.py::mcts_plan_wavefront."""

    def __init__(self, env_kind, n_actions, episodes, horizon, gamma, temperature, width, mdp=None, device="cuda",
                 max_ctas=0):
        import torch
        self.torch = torch
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.n_actions, self.episodes, self.horizon = int(n_actions), int(episodes), int(horizon)
        self.width = max(1, min(int(width), 1024))
        self.capacity = 1 + self.episodes * self.n_actions
        gp, _ = gamma_tables(gamma, self.horizon + 1)
        self.gamma_pow = torch.as_tensor(gp, device=self.device)
        self.sampled, self.tables, finite_mdp = finite_model(env_kind, mdp, self.device)
        if self.sampled:
            self.env_rng = torch.empty(_lib.PCG64_STATE_WORDS, dtype=torch.int64, device=self.device)
            self.rejected = torch.empty(2, dtype=torch.int32, device=self.device)
        i32 = torch.int32
        self.parent = torch.empty(self.capacity, dtype=i32, device=self.device)
        self.first_child = torch.empty(self.capacity, dtype=i32, device=self.device)
        self.count = torch.empty(self.capacity, dtype=i32, device=self.device)
        self.meta = torch.empty(self.capacity, dtype=i32, device=self.device)
        self.vsum = torch.empty(self.capacity, dtype=torch.int64, device=self.device)
        self.value = torch.empty(self.capacity, dtype=torch.float64, device=self.device)
        self.cfg = _lib.MCTSWaveConfig(env_kind, self.n_actions, self.episodes, self.horizon, self.capacity, self.width,
                                       0, 0, float(temperature), 0, self.gamma_pow.data_ptr(),
                                       finite_mdp, int(max_ctas), 0)
        self.tree = _lib.MCTSWaveTree(*[t.data_ptr() for t in (self.parent, self.first_child, self.count, self.meta,
                                                               self.vsum, self.value)])
        ws = self.lib.b2_mcts_wave_workspace_bytes(self.cfg)
        if ws < 0:
            raise _lib.B2Error("unsupported wavefront MCTS configuration")
        self.workspace = torch.empty(int(ws), dtype=torch.uint8, device=self.device)
        self.plan_buf = torch.empty(max(self.horizon, 1), dtype=torch.int8, device=self.device)
        self.result = torch.empty(_lib.MCTS_RESULT_WORDS, dtype=i32, device=self.device)

    def plan(self, root_state, seed, env_words=None):
        """root_state: int32 device tensor [1] (finite) or [136]; seed: the counter-based generator's seed;
        env_words (sampled MDPs only): uint64 [6], pcg64_words of the live env's generator."""
        assert root_state.dtype == self.torch.int32 and root_state.is_cuda and root_state.is_contiguous()
        self.cfg.seed = int(seed) & ((1 << 64) - 1)
        if self.sampled:
            if env_words is None:
                raise ValueError("MCTS on a stochastic finite MDP needs the env generator's words (env_words)")
            w = np.ascontiguousarray(np.asarray(env_words, dtype=np.uint64).reshape(-1))
            self.env_rng.copy_(self.torch.from_numpy(w.view(np.int64)))
            t = self.tables
            _lib.check(self.lib.b2_mcts_plan_wave_sampled(
                self.cfg, t.struct(), _lib.ptr(t.terminal), t.env_draws, _lib.ptr(self.env_rng), _lib.ptr(root_state),
                self.tree, _lib.ptr(self.workspace), _lib.ptr(self.plan_buf), _lib.ptr(self.result),
                _lib.ptr(self.rejected), _lib.current_stream()))
            return
        _lib.check(self.lib.b2_mcts_plan_wave(self.cfg, _lib.ptr(root_state), self.tree, _lib.ptr(self.workspace),
                                              _lib.ptr(self.plan_buf), _lib.ptr(self.result), _lib.current_stream()))

    def finish(self):
        res = self.result.cpu().numpy()
        if self.sampled:
            episode, row = self.rejected.cpu().numpy().tolist()
            if episode >= 0:
                self.tables.raise_rejected_row(row)
        return self.plan_buf.cpu().numpy()[:res[1]].astype(int).tolist(), res

    def tree_dict(self):
        meta = self.meta.cpu().numpy()
        return {"parent": self.parent.cpu().numpy(), "action": decode_action(meta), "count": self.count.cpu().numpy(),
                "first_child": self.first_child.cpu().numpy(), "n_children": (meta >> 8) & 0xff,
                "vsum": self.vsum.cpu().numpy(), "value": self.value.cpu().numpy()}

    def root_statistics(self):
        d = self.tree_dict()
        fc, n = int(d["first_child"][0]), int(d["n_children"][0])
        counts, values = np.zeros(self.n_actions), np.zeros(self.n_actions)
        for c in range(fc, fc + n):
            counts[d["action"][c]], values[d["action"][c]] = d["count"][c], d["value"][c]
        return counts, values
