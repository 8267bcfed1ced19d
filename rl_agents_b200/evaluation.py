"""Batched closed-loop evaluation of the planners on HighwayLite (of MCTS and OLOP on IntersectionLite, and of every
planner on finite MDPs, stepped by b2_finite_step): the
working version of the reference's disabled budget-sweep harness (scripts/planners_evaluation.py:287-289, SURVEY 8f
rank 4) in the shape the GPU wants -- all episodes advance in lock-step, every decision step is
ONE batched plan() launch over all live episodes and ONE batched env transition."""
import logging
import time

import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.envs import highway_lite, intersection_lite

logger = logging.getLogger(__name__)

# planners with an IntersectionLite model (b2_mcts_plan, b2_olop_plan)
INTERSECTION_PLANNERS = ("mcts", "olop")
# GBOP-T (StateAwarePlannerAgent) and GBOP-D (GraphBasedPlannerAgent): deterministic finite MDPs only
GBOP_PLANNERS = ("gbop", "gbopd")
# planners whose agents refuse a finite MDP in mode "stochastic" or "sparse"
DETERMINISTIC_ONLY_PLANNERS = ("opd", "brue") + GBOP_PLANNERS


def _np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def _keeps_subtrees(planner, kw):
    """Whether the episodes of `planner` keep their trees across decisions: keyword step_strategy "subtree" on "mcts",
    as MCTSAgent does.  Any other strategy than "reset" resets, with the warning the agents give."""
    strategy = kw.get("step_strategy", "reset")
    if planner == "mcts" and strategy == "subtree":
        return True
    if strategy != "reset":
        logger.warning("step strategy {} is not supported by the batched {} episodes: resetting".format(strategy,
                                                                                                        planner))
    return False


def run_batched_episodes(planner, seeds, budget, gamma, max_steps=40, device="cuda", planner_seed=0, env="highway",
                         **kw):
    """planner: "opd" | "mcts" | "olop" | "mdp_gape" (keywords: MDPGapEAgent config keys) | "brue" (keywords: BRUEAgent
    config keys) | "sparse_sampling" (keywords `horizon` and `C`, required as in SparseSamplingAgent's config; `budget`
    is unused) | "mcts_dpw" (keywords: MCTSDPWAgent config keys) | "platypoos" (keywords: PlaTyPOOSAgent config keys;
    the first action of each plan is played) | "vi" (ValueIterationAgent on the scenes' TTC-grid MDPs, `budget` = its
    `iterations`).  Every episode: scene make_scene(seed), replanning at every step (receding_horizon 1, step_strategy reset -- the reference
    defaults), until crash or `max_steps`.  "mcts" also takes step_strategy="subtree" (on every env): after each step
    every tree is re-rooted at its played action in one b2_mcts_reroot launch and the next search resumes from it, so
    episode i plays what MCTSAgent(env_i, {budget, gamma, step_strategy: "subtree"}) seeded planner_seed + i plays.
    env: "highway" (HighwayLite, every planner) or "intersection" (IntersectionLite scenes of
    envs.intersection_lite.make_scene stepped by b2_intersection_step, "mcts" and "olop" only; an episode also ends
    when the ego arrives or at the env's duration).  `crashed` is the ego's crash flag.
    env "finite": closed-loop episodes on a finite MDP, see run_finite_episodes (keywords `mdp`, `start_states`,
    `env_seed`).
    Returns dict(returns, lengths, crashed, decision_ms), with "subtree" also `resumed`: per episode, the decisions
    that resumed a kept sub-tree."""
    if env == "finite":
        return run_finite_episodes(planner, len(seeds), budget, gamma, max_steps=max_steps, device=device,
                                   planner_seed=planner_seed, **kw)
    if planner in GBOP_PLANNERS and env in ("highway", "intersection"):
        raise NotImplementedError("%r aggregates nodes by state id: it runs on finite MDPs only" % planner)
    import torch
    from rl_agents_b200.engine.mcts import MCTSEngine, pcg64_words, set_pcg64_words
    from rl_agents_b200.engine.olop import OLOPEngine
    from rl_agents_b200.engine.opd import OPDEngine
    from rl_agents_b200.agents.tree_search.mcts import allocation, subtree_capacity
    if env == "highway":
        env_kind, n_actions, make_scene = _lib.ENV_HIGHWAY, 5, highway_lite.make_scene
    elif env == "intersection":
        if planner not in INTERSECTION_PLANNERS:
            raise NotImplementedError("%r runs on HighwayLite only; IntersectionLite runs %s"
                                      % (planner, " and ".join(INTERSECTION_PLANNERS)))
        env_kind, n_actions, make_scene = _lib.ENV_INTERSECTION, intersection_lite.N_ACTIONS, intersection_lite.make_scene
    else:
        raise ValueError("unknown env %r" % env)
    subtree = _keeps_subtrees(planner, kw)
    lib = _lib.load()
    dev = torch.device(device)
    n = len(seeds)
    scenes = torch.from_numpy(np.stack([make_scene(s) for s in seeds])).to(dev)
    rngs = [_np_random(planner_seed + i) for i in range(n)]
    if planner == "opd":
        eng = OPDEngine(_lib.ENV_HIGHWAY, n, 5, budget, gamma, kw.get("terminal_reward", 0.0), device=dev)
    elif planner == "mcts":
        episodes, horizon = allocation(budget, gamma)
        from rl_agents_b200.agents.tree_search.mcts import MCTS
        # the reference's default temperature comes from the CLASS default gamma (mcts.py:120-127), not the configured one
        eng = MCTSEngine(env_kind, n, n_actions, episodes, horizon, gamma,
                         kw.get("temperature", MCTS.default_config()["temperature"]), device=dev,
                         capacity=subtree_capacity(episodes, horizon, n_actions) if subtree else None)
    elif planner == "olop":
        episodes, horizon = allocation(max(n_actions, budget), gamma)
        ub = kw.get("upper_bound", {"type": "kullback-leibler", "time": "global", "threshold": "2*np.log(time)"})
        eng = OLOPEngine(env_kind, n, n_actions, episodes, horizon, gamma, ub, kw.get("continuation_type", "uniform"),
                         device=dev)
    elif planner == "mdp_gape":
        # MDPGapEAgent's completed config (mdp_gape.py:20-40) with budget / gamma and any keyword overriding it
        from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapE, budget_allocation
        from rl_agents_b200.engine.mdp_gape import MDPGapEEngine
        cfg = MDPGapE.default_config()
        MDPGapE.rec_update(cfg, dict(kw, budget=budget, gamma=gamma))
        episodes, horizon = budget_allocation(cfg, 5)
        eng = MDPGapEEngine(_lib.ENV_HIGHWAY, n, 5, episodes, horizon, gamma, cfg["upper_bound"], cfg["accuracy"],
                            cfg["confidence"], cfg["continuation_type"], cfg["max_next_states_count"], device=dev)
    elif planner == "brue":
        # BRUEAgent's completed config (OLOP's defaults, brue.py:19-22) with budget / gamma and any keyword overriding it
        from rl_agents_b200.agents.tree_search.brue import BRUE
        from rl_agents_b200.engine.brue import BRUEEngine
        cfg = BRUE.default_config()
        BRUE.rec_update(cfg, dict(kw, budget=budget, gamma=gamma))
        horizon = cfg["horizon"] if "horizon" in cfg else allocation(max(5, budget), gamma)[1]
        eng = BRUEEngine(_lib.ENV_HIGHWAY, n, 5, budget, horizon, gamma, device=dev)
    elif planner == "sparse_sampling":
        from rl_agents_b200.engine.sparse_sampling import SparseSamplingEngine
        eng = SparseSamplingEngine(_lib.ENV_HIGHWAY, n, 5, kw["horizon"], kw["C"], gamma, device=dev)
    elif planner == "mcts_dpw":
        # MCTSDPWAgent's completed planner config (mcts_dpw.py:20-54) with budget / gamma and any keyword overriding it
        from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPW, MCTSDPWAgent
        from rl_agents_b200.engine.mcts_dpw import MCTSDPWEngine
        cfg = MCTSDPWAgent.default_config()
        MCTSDPWAgent.rec_update(cfg, dict(kw, budget=budget, gamma=gamma))
        pcfg = MCTSDPW.default_config()
        MCTSDPW.rec_update(pcfg, cfg)
        episodes, horizon = (pcfg["episodes"], pcfg["horizon"]) if pcfg["horizon"] else allocation(budget, gamma)
        eng = MCTSDPWEngine(_lib.ENV_HIGHWAY, n, 5, episodes, horizon, gamma, pcfg["temperature"], pcfg["k_action"],
                            pcfg["alpha_action"], pcfg["k_state"], pcfg["alpha_state"],
                            closed_loop=pcfg["closed_loop"],
                            rollout_policy=MCTSDPWAgent.policy_factory(pcfg["rollout_policy"]), device=dev)
    elif planner == "platypoos":
        # PlaTyPOOSAgent's completed planner config (h_max from the budget unless "horizon" is given)
        from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOS
        from rl_agents_b200.engine.platypoos import PlaTyPOOSEngine, horizon_of
        cfg = PlaTyPOOS.default_config()
        PlaTyPOOS.rec_update(cfg, dict(kw, budget=budget, gamma=gamma))
        horizon = cfg["horizon"] if "horizon" in cfg else horizon_of(budget, 5)
        eng = PlaTyPOOSEngine(_lib.ENV_HIGHWAY, n, 5, horizon, gamma, device=dev)
    elif planner == "vi":
        from rl_agents_b200.engine.ttc_vi import HighwayTTCVI
        eng = HighwayTTCVI(gamma, budget, device=dev)
    else:
        raise ValueError("unknown planner %r" % planner)
    returns = np.zeros(n)
    lengths = np.zeros(n, dtype=int)
    alive = np.ones(n, dtype=bool)
    crashed = np.zeros(n, dtype=bool)
    rew = torch.empty(n, dtype=torch.float32, device=dev)
    flg = torch.empty(n, dtype=torch.int32, device=dev)
    actions_log = []
    t_plan = 0.0
    kept, resumed = None, np.zeros(n, dtype=int)
    for step in range(max_steps):
        if not alive.any():
            break
        t0 = time.perf_counter()
        if subtree and step:
            # MCTS.step_tree: every tree re-rooted at its played action (-1 after an empty plan: a new tree)
            kept = eng.reroot([p[0] if p else -1 for p in plans])
            resumed += alive & (kept > 0)
        if planner == "opd":
            eng.plan(scenes)
            plans, _ = eng.finish(rngs)
        elif planner == "vi":
            plans = [[int(a)] for a in eng.solve(scenes, want_q=False)["action"].cpu().numpy()]
        else:
            words = np.stack([pcg64_words(g) for g in rngs])
            if kept is None:
                eng.plan(scenes, words)
            else:
                eng.plan(scenes, words, kept)
            plans, _, words = eng.finish()
            for g, w in zip(rngs, words):
                set_pcg64_words(g, w)
        t_plan += time.perf_counter() - t0
        act = np.array([p[0] if p else 1 for p in plans], dtype=np.int32)      # empty plan: IDLE
        actions_log.append(act.copy())
        step = lib.b2_highway_step if env == "highway" else lib.b2_intersection_step
        _lib.check(step(_lib.ptr(scenes), _lib.ptr(torch.from_numpy(act).to(dev)), _lib.ptr(rew), _lib.ptr(flg), None, n,
                        _lib.current_stream()))
        r, f = rew.cpu().numpy(), flg.cpu().numpy()
        returns += np.where(alive, r, 0.0)
        lengths += alive
        done = (f & 3) != 0
        if env == "highway":
            crashed |= alive & ((f & 1) != 0)
        else:       # IntersectionLite also terminates on arrival: the crash is bit 1 of the ego's flags word
            crashed |= alive & ((scenes[:, 48].cpu().numpy() & 2) != 0)
        alive &= ~done
    out = {"returns": returns, "lengths": lengths, "crashed": crashed, "actions": np.array(actions_log).T,
           "decision_ms": 1e3 * t_plan / max(len(actions_log), 1), "n": n}
    if subtree:
        out["resumed"] = resumed        # per episode: the decisions that resumed a kept sub-tree
    return out


def _completed_config(agent_cls, planner_cls, kw, budget, gamma):
    """The planner config of agent_cls(env, dict(kw, budget=budget, gamma=gamma)): the agent's defaults updated with
    the keywords, then the planner's defaults updated with that."""
    cfg = agent_cls.default_config()
    agent_cls.rec_update(cfg, dict(kw, budget=budget, gamma=gamma))
    pcfg = planner_cls.default_config()
    planner_cls.rec_update(pcfg, cfg)
    return pcfg


def _finite_engine_factory(planner, mdp, n_actions, budget, gamma, kw, dev):
    """-> make(n_trees): the engine of `planner` on the finite MDP `mdp` with its drop-in agent's completed config."""
    from rl_agents_b200.agents.tree_search.mcts import MCTS, MCTSAgent, allocation
    E, A = _lib.ENV_FINITE, n_actions
    if planner == "opd":
        from rl_agents_b200.agents.tree_search.deterministic import (DeterministicPlannerAgent,
                                                                     OptimisticDeterministicPlanner)
        from rl_agents_b200.engine.opd import OPDEngine
        c = _completed_config(DeterministicPlannerAgent, OptimisticDeterministicPlanner, kw, budget, gamma)
        return lambda m: OPDEngine(E, m, A, budget, gamma, c.get("terminal_reward", 0), mdp=mdp, device=dev,
                                   keys_in_smem=c.get("keys_in_smem", True))
    if planner == "gbop":
        from rl_agents_b200.agents.tree_search.state_aware import StateAwarePlanner, StateAwarePlannerAgent
        from rl_agents_b200.engine.gbop import GBOPEngine
        c = _completed_config(StateAwarePlannerAgent, StateAwarePlanner, kw, budget, gamma)
        return lambda m: GBOPEngine(m, A, budget, gamma, mdp, c.get("terminal_reward", 0), c["backup_aggregated_nodes"],
                                    c["prune_suboptimal_leaves"], c["accuracy"], device=dev)
    if planner == "gbopd":
        from rl_agents_b200.agents.tree_search.graph_based import GraphBasedPlanner, GraphBasedPlannerAgent
        from rl_agents_b200.engine.gbop import GBOPDEngine
        c = _completed_config(GraphBasedPlannerAgent, GraphBasedPlanner, kw, budget, gamma)
        return lambda m: GBOPDEngine(m, A, budget, gamma, mdp, c["accuracy"], c["sampling_timeout"], device=dev)
    if planner == "brue":
        from rl_agents_b200.agents.tree_search.brue import BRUE, BRUEAgent
        from rl_agents_b200.engine.brue import BRUEEngine
        c = _completed_config(BRUEAgent, BRUE, kw, budget, gamma)
        horizon = c["horizon"] if "horizon" in c else allocation(max(A, budget), gamma)[1]
        return lambda m: BRUEEngine(E, m, A, budget, horizon, gamma, mdp=mdp, device=dev)
    if planner == "mcts":
        from rl_agents_b200.agents.tree_search.mcts import subtree_capacity
        from rl_agents_b200.engine.mcts import MCTSEngine
        c = _completed_config(MCTSAgent, MCTS, kw, budget, gamma)
        episodes, horizon = (c["episodes"], c["horizon"]) if c["horizon"] else allocation(budget, gamma)
        capacity = subtree_capacity(episodes, horizon, A) if c["step_strategy"] == "subtree" else None
        return lambda m: MCTSEngine(E, m, A, episodes, horizon, gamma, c["temperature"], mdp=mdp,
                                    rollout_policy=MCTSAgent.policy_factory(c["rollout_policy"]),
                                    prior_policy=MCTSAgent.policy_factory(c["prior_policy"]), device=dev,
                                    capacity=capacity)
    if planner == "olop":
        from rl_agents_b200.agents.tree_search.olop import OLOP, OLOPAgent
        from rl_agents_b200.engine.olop import OLOPEngine
        c = _completed_config(OLOPAgent, OLOP, kw, budget, gamma)
        episodes, horizon = (c["episodes"], c["horizon"]) if "horizon" in c else allocation(max(A, budget), gamma)
        return lambda m: OLOPEngine(E, m, A, episodes, horizon, gamma, c["upper_bound"], c["continuation_type"],
                                    mdp=mdp, device=dev)
    if planner == "mdp_gape":
        from rl_agents_b200.agents.tree_search.mdp_gape import MDPGapE, MDPGapEAgent, budget_allocation
        from rl_agents_b200.engine.mdp_gape import MDPGapEEngine
        c = _completed_config(MDPGapEAgent, MDPGapE, kw, budget, gamma)
        episodes, horizon = (c["episodes"], c["horizon"]) if "horizon" in c else budget_allocation(c, A)
        return lambda m: MDPGapEEngine(E, m, A, episodes, horizon, gamma, c["upper_bound"], c["accuracy"],
                                       c["confidence"], c["continuation_type"], c["max_next_states_count"], mdp=mdp,
                                       device=dev)
    if planner == "sparse_sampling":
        from rl_agents_b200.engine.sparse_sampling import EMPTY_ROOT_MESSAGE, SparseSamplingEngine
        if kw["horizon"] == 0:
            raise ValueError(EMPTY_ROOT_MESSAGE)            # SparseSampling.plan: a childless root
        return lambda m: SparseSamplingEngine(E, m, A, kw["horizon"], kw["C"], gamma, mdp=mdp, device=dev)
    if planner == "mcts_dpw":
        from rl_agents_b200.agents.tree_search.mcts_dpw import MCTSDPW, MCTSDPWAgent
        from rl_agents_b200.engine.mcts_dpw import MCTSDPWEngine
        c = _completed_config(MCTSDPWAgent, MCTSDPW, kw, budget, gamma)
        episodes, horizon = (c["episodes"], c["horizon"]) if c["horizon"] else allocation(budget, gamma)
        return lambda m: MCTSDPWEngine(E, m, A, episodes, horizon, gamma, c["temperature"], c["k_action"],
                                       c["alpha_action"], c["k_state"], c["alpha_state"], closed_loop=c["closed_loop"],
                                       rollout_policy=MCTSDPWAgent.policy_factory(c["rollout_policy"]), mdp=mdp,
                                       device=dev)
    if planner == "platypoos":
        from rl_agents_b200.agents.tree_search.platypoos import PlaTyPOOS, PlaTyPOOSAgent
        from rl_agents_b200.engine.platypoos import PlaTyPOOSEngine, check_plannable, horizon_of
        c = _completed_config(PlaTyPOOSAgent, PlaTyPOOS, kw, budget, gamma)
        horizon = c["horizon"] if "horizon" in c else horizon_of(budget, A)
        check_plannable(horizon, A, True)
        return lambda m: PlaTyPOOSEngine(E, m, A, horizon, gamma, mdp=mdp, device=dev)
    raise ValueError("unknown planner %r" % planner)


def run_finite_episodes(planner, n_episodes, budget, gamma, mdp, start_states=None, env_seed=0, max_steps=40,
                        device="cuda", planner_seed=0, **kw):
    """Closed-loop episodes on a finite MDP in any mode, in lock step: per decision step ONE batched plan() over the
    live episodes and ONE b2_finite_step over all of them (FiniteMDPEnv.step on the device).

    mdp: a FiniteMDPEnv, or any env adapters.describe takes for a finite MDP.  Episode i starts at start_states[i]
    (default: the MDP's `state`); its env generator is np.random.default_rng(env_seed + i), the one
    FiniteMDPEnv(seed=env_seed + i) holds, and its planner generator that of agent.seed(planner_seed + i).  Each
    episode plays what its planner's drop-in agent, built with dict(kw, budget=budget, gamma=gamma), would act and
    ends when done (terminal[state the action is taken in]) or at `max_steps`.  With "mcts" and step_strategy="subtree"
    every live tree is re-rooted at its played action after each step (b2_mcts_reroot), into a new engine holding the
    survivors' trees only when episodes have ended, and the next search resumes from it.
    planner: "opd", "gbop" (GBOP-T), "gbopd" (GBOP-D) and "brue" on deterministic MDPs (NotImplementedError otherwise,
    as their agents refuse); "mcts", "olop", "mdp_gape", "sparse_sampling", "mcts_dpw" and "platypoos" in every mode;
    "vi" (ValueIterationAgent, `budget` = its `iterations`).  A reached row that Generator.choice rejects raises its
    ValueError.
    Returns dict(returns, lengths, crashed (all False), actions and rewards [n_episodes, steps] (-1 and 0 once an
    episode has ended), final_states, planner_words and env_words (PCG64 words [n_episodes, 6] at the end),
    decision_ms (host time per plan step), step_ms (device time per b2_finite_step call), n)."""
    import torch
    from rl_agents_b200.engine.mcts import pcg64_words, set_pcg64_words
    from rl_agents_b200.engine.tables import SampledFiniteTables
    from rl_agents_b200.envs.adapters import describe
    d = describe(mdp)
    if d.kind != _lib.ENV_FINITE:
        raise ValueError("env 'finite' needs a finite-MDP env (got %r)" % type(mdp).__name__)
    if planner in DETERMINISTIC_ONLY_PLANNERS and d.mdp.mode != "deterministic":
        raise NotImplementedError("%r plans on deterministic finite MDPs only (got mode %r)" % (planner, d.mdp.mode))
    subtree = _keeps_subtrees(planner, kw)
    lib = _lib.load()
    dev = torch.device(device)
    n, A = int(n_episodes), d.n_actions
    start = np.full(n, d.root[0]) if start_states is None else np.asarray(start_states)
    if start.shape != (n,) or (start < 0).any() or (start >= d.mdp.reward.shape[0]).any():
        raise ValueError("start_states must hold one state id of the MDP per episode")
    if planner == "vi":
        from rl_agents_b200.engine.vi import VIEngine
        m = d.mdp
        q = VIEngine(m.mode, m.transition, m.reward, m.terminal, nxt=getattr(m, "next", None), gamma=gamma,
                     device=dev).solve(budget)[0].cpu().numpy()
    else:
        make = _finite_engine_factory(planner, d.mdp, A, budget, gamma, kw, dev)
    tables = SampledFiniteTables(d.mdp, dev)
    states = torch.as_tensor(start.astype(np.int32), device=dev)
    env_rng = torch.as_tensor(np.stack([pcg64_words(np.random.default_rng(env_seed + i)) for i in range(n)])
                              .view(np.int64), device=dev)
    rngs = [_np_random(planner_seed + i) for i in range(n)]
    rew = torch.empty(n, dtype=torch.float64, device=dev)
    flg = torch.empty(n, dtype=torch.int32, device=dev)
    bad = torch.empty(n, dtype=torch.int32, device=dev)
    returns, lengths, alive = np.zeros(n), np.zeros(n, dtype=int), np.ones(n, dtype=bool)
    actions, rewards = np.full((n, max_steps), -1), np.zeros((n, max_steps))
    eng, events, t_plan, steps = None, [], 0.0, 0
    planned, kept, resumed = None, None, np.zeros(n, dtype=int)     # "subtree": the episodes of the last plan
    for step in range(max_steps):
        live = np.nonzero(alive)[0]
        if not live.size:
            break
        t0 = time.perf_counter()
        if planner == "vi":
            act_live = np.argmax(q[states.cpu().numpy()[live]], axis=1)       # ValueIterationAgent.act
        else:
            if eng is None or eng.n_trees != live.size:     # an engine per live-episode count
                old, eng = eng, make(live.size)
                if subtree and old is not None:             # the survivors' trees, gathered and re-rooted
                    kept = eng.reroot(act[live], np.searchsorted(planned, live), source=old)
                del old
            elif subtree and planned is not None:           # MCTS.step_tree, every tree in one launch
                kept = eng.reroot(act[live])
            if kept is not None:
                resumed[live] += kept > 0
            planned = live
            live_d = torch.as_tensor(live, device=dev)
            roots = states.index_select(0, live_d).contiguous()
            if planner in ("opd", "gbop"):
                eng.plan(roots)
                plans, _ = eng.finish([rngs[i] for i in live])
            else:
                words = np.stack([pcg64_words(rngs[i]) for i in live])
                if planner == "mcts":       # MCTSAgent.plan: the resumed sub-trees and the live env generator's words
                    eng.plan(roots, words, kept,
                             env_rng.index_select(0, live_d).cpu().numpy().view(np.uint64) if eng.sampled else None)
                else:
                    eng.plan(roots, words)
                plans, _, words = eng.finish()
                for i, w in zip(live, words):
                    set_pcg64_words(rngs[i], w)
            act_live = [p[0] for p in plans]
        t_plan += time.perf_counter() - t0
        act = np.zeros(n, dtype=np.int32)
        act[live] = act_live
        mask = np.zeros(n, dtype=np.uint8)
        mask[live] = 1
        act_d, mask_d = torch.from_numpy(act).to(dev), torch.from_numpy(mask).to(dev)
        events.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
        events[-1][0].record()
        _lib.check(lib.b2_finite_step(tables.struct(), _lib.ptr(tables.terminal), tables.env_draws, _lib.ptr(states),
                                      _lib.ptr(act_d), _lib.ptr(mask_d), _lib.ptr(env_rng), _lib.ptr(rew),
                                      _lib.ptr(flg), _lib.ptr(bad), n, _lib.current_stream()))
        events[-1][1].record()
        r, f, b = rew.cpu().numpy(), flg.cpu().numpy(), bad.cpu().numpy()
        rejected = live[b[live] >= 0]
        if rejected.size:
            tables.raise_rejected_row(int(b[rejected[0]]))
        returns[live] += r[live]
        rewards[live, step] = r[live]
        actions[live, step] = act[live]
        lengths[live] += 1
        alive[live] = (f[live] & 1) == 0
        steps += 1
    step_ms = sum(a.elapsed_time(b) for a, b in events)
    out = {"returns": returns, "lengths": lengths, "crashed": np.zeros(n, dtype=bool), "actions": actions[:, :steps],
           "rewards": rewards[:, :steps], "final_states": states.cpu().numpy(),
           "planner_words": np.stack([pcg64_words(g) for g in rngs]), "env_words": env_rng.cpu().numpy().view(np.uint64),
           "decision_ms": 1e3 * t_plan / max(steps, 1), "step_ms": step_ms / max(steps, 1), "n": n}
    if subtree:
        out["resumed"] = resumed        # per episode: the decisions that resumed a kept sub-tree
    return out
