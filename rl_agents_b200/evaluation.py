"""Batched closed-loop evaluation of the planners on HighwayLite (and of MCTS and OLOP on IntersectionLite): the
working version of the reference's disabled budget-sweep harness (scripts/planners_evaluation.py:287-289, SURVEY 8f
rank 4) in the shape the GPU wants -- all episodes advance in lock-step, every decision step is
ONE batched plan() launch over all live episodes and ONE batched env transition."""
import time

import numpy as np

from rl_agents_b200 import _lib
from rl_agents_b200.envs import highway_lite, intersection_lite

# planners with an IntersectionLite model (b2_mcts_plan, b2_olop_plan)
INTERSECTION_PLANNERS = ("mcts", "olop")


def _np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def run_batched_episodes(planner, seeds, budget, gamma, max_steps=40, device="cuda", planner_seed=0, env="highway",
                         **kw):
    """planner: "opd" | "mcts" | "olop" | "mdp_gape" (keywords: MDPGapEAgent config keys) | "brue" (keywords: BRUEAgent
    config keys) | "sparse_sampling" (keywords `horizon` and `C`, required as in SparseSamplingAgent's config; `budget`
    is unused) | "mcts_dpw" (keywords: MCTSDPWAgent config keys) | "platypoos" (keywords: PlaTyPOOSAgent config keys;
    the first action of each plan is played) | "vi" (ValueIterationAgent on the scenes' TTC-grid MDPs, `budget` = its
    `iterations`).  Every episode: scene make_scene(seed), replanning at every step (receding_horizon 1, step_strategy reset -- the reference
    defaults), until crash or `max_steps`.
    env: "highway" (HighwayLite, every planner) or "intersection" (IntersectionLite scenes of
    envs.intersection_lite.make_scene stepped by b2_intersection_step, "mcts" and "olop" only; an episode also ends
    when the ego arrives or at the env's duration).  `crashed` is the ego's crash flag.
    Returns dict(returns, lengths, crashed, decision_ms)."""
    import torch
    from rl_agents_b200.engine.mcts import MCTSEngine, pcg64_words, set_pcg64_words
    from rl_agents_b200.engine.olop import OLOPEngine
    from rl_agents_b200.engine.opd import OPDEngine
    from rl_agents_b200.agents.tree_search.mcts import allocation
    if env == "highway":
        env_kind, n_actions, make_scene = _lib.ENV_HIGHWAY, 5, highway_lite.make_scene
    elif env == "intersection":
        if planner not in INTERSECTION_PLANNERS:
            raise NotImplementedError("%r runs on HighwayLite only; IntersectionLite runs %s"
                                      % (planner, " and ".join(INTERSECTION_PLANNERS)))
        env_kind, n_actions, make_scene = _lib.ENV_INTERSECTION, intersection_lite.N_ACTIONS, intersection_lite.make_scene
    else:
        raise ValueError("unknown env %r" % env)
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
                         kw.get("temperature", MCTS.default_config()["temperature"]), device=dev)
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
    for step in range(max_steps):
        if not alive.any():
            break
        t0 = time.perf_counter()
        if planner == "opd":
            eng.plan(scenes)
            plans, _ = eng.finish(rngs)
        elif planner == "vi":
            plans = [[int(a)] for a in eng.solve(scenes, want_q=False)["action"].cpu().numpy()]
        else:
            eng.plan(scenes, np.stack([pcg64_words(g) for g in rngs]))
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
    return {"returns": returns, "lengths": lengths, "crashed": crashed, "actions": np.array(actions_log).T,
            "decision_ms": 1e3 * t_plan / max(len(actions_log), 1), "n": n}
