"""GPU tests of DROP on IntersectionLite (b2_opd_plan_wave with B2_ENV_INTERSECTION and n_models = M): the kernel and
DiscreteRobustPlannerAgent against the unmodified reference's goldens (tests/golden/golden_drop_intersection.json) and
against oracle.planners.robust_plan at every wave width, on route hypotheses made by the product env's
`set_route_at_intersection`; and the refusals that stay."""
import json

import numpy as np
import pytest

from oracle import intersection as oit
from oracle import planners
from oracle.intersection_routes import IntersectionLiteRoutes
from tests import intersection_scenes as isc
from tests.util import load_golden

pytestmark = pytest.mark.gpu
G = load_golden("golden_drop_intersection.json")


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def f64_hex(x):
    return np.asarray(x, dtype="<f8").tobytes().hex()


def model_words(words, chains):
    """The product env's models: one preprocessed copy of IntersectionLiteEnv(words) per chain (robust.py:66)."""
    from rl_agents_b200.agents.common.factory import preprocess_env
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv
    env = IntersectionLiteEnv(np.array(words, dtype=np.int32))
    return np.stack([preprocess_env(env, chain).words for chain in chains])


def oracle_models(words, args):
    env = IntersectionLiteRoutes(oit.IntersectionLiteState.unpack(np.array(words, dtype=np.int32)))
    return [env.set_route_at_intersection(a) for a in args]


def chains(args):
    return [[{"method": "set_route_at_intersection", "args": a}] for a in args]


def run_engine(words, budget, gamma, width, terminal_reward=0.0, seed=0):
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.engine.opd import OPDWaveEngine
    eng = OPDWaveEngine(_lib.ENV_INTERSECTION, 3, budget, gamma, width, terminal_reward, n_models=len(words))
    eng.plan(torch.tensor(words, dtype=torch.int32, device="cuda"))
    rng = np_random(seed)
    plans, res = eng.finish([rng])
    return plans[0], eng.tree_dict(0), rng, res


def assert_same_tree(d, t):
    assert d["parent"].tolist() == t.parent and d["action"].tolist() == t.action and d["count"].tolist() == t.count
    assert f64_hex(d["lower"]) == f64_hex(t.lower) and f64_hex(d["upper"]) == f64_hex(t.upper)


@pytest.mark.parametrize("name", sorted(G["cases"]))
def test_kernel_equals_the_reference_golden(name):
    g = G["cases"][name]
    c = g["config"]
    words = model_words(g["words"], c["models"])
    plan, d, rng, _ = run_engine(words, c["budget"], c["gamma"], 1, c.get("terminal_reward", 0), g["seed"])
    tr = g["tree"]
    assert plan == g["plan"]
    assert d["parent"].tolist() == tr["parent"] and d["action"].tolist() == tr["action"]
    assert d["count"].tolist() == tr["count"]
    assert f64_hex(d["lower"]) == tr["lower"] and f64_hex(d["upper"]) == tr["upper"]
    assert rng_state(rng) == g["rng_state"]


# (route hypotheses, wave width, budget, scene family and index, terminal_reward)
ORACLE_CASES = [
    ((1,), 1, 600, ("phases", 3), 0.0),
    ((0, 2), 8, 1500, ("arrival", 5), 0.3),
    ((0, 1, 2), 64, 3000, ("crossing", 4), 0.0),
    ((0, 1, 2), 1, 900, ("full", 1), 0.0),
    ((0, 1, 2), 8, 2000, ("stale", 2), 0.0),
    ((2, "random"), 64, 300, ("ties", 0), 0.5),
    ((0, 1, 2, "random", 5, -1, 4, "random"), 8, 600, ("blocked", 2), 0.0),
    ((2, 1, 0, "random", 1, 2, 0, 3), 64, 1200, ("wrap", 1), 0.2),
    ((0, 1, 2, "random", 0, 1, 2, 0), 1, 300, ("arrival", 13), 0.0),
]


@pytest.mark.parametrize("args,width,budget,scene,terminal_reward", ORACLE_CASES,
                         ids=["M%d_w%d_b%d_%s%d" % (len(c[0]), c[1], c[2], c[3][0], c[3][1]) for c in ORACLE_CASES])
def test_kernel_equals_robust_plan(args, width, budget, scene, terminal_reward):
    words = isc.family(scene[0])[scene[1]].pack()
    gamma = 0.9
    plan, d, rng, res = run_engine(model_words(words, chains(args)), budget, gamma, width, terminal_reward, seed=5)
    orng = np_random(5)
    oplan, t = planners.robust_plan(oracle_models(words, args), budget, gamma, terminal_reward, orng, width=width)
    assert plan == oplan
    assert_same_tree(d, t)
    assert int(res[0, 7]) == len(t.waves)
    assert rng_state(rng) == rng_state(orng)


def test_identical_models_give_the_one_model_tree():
    words = isc.family("crossing")[1].pack()
    p1, d1, _, _ = run_engine(model_words(words, chains((1,))), 900, 0.9, 8)
    for m in (2, 3, 8):
        pm, dm, _, _ = run_engine(model_words(words, chains((1,) * m)), 900, 0.9, 8)
        assert pm == p1
        for k in ("parent", "action", "count", "depth", "first_child", "n_children", "done"):
            assert np.array_equal(dm[k], d1[k]), k
        assert f64_hex(dm["lower"]) == f64_hex(d1["lower"]) and f64_hex(dm["upper"]) == f64_hex(d1["upper"])


def test_agent_from_routes_behaviours_plans_as_the_reference():
    """DiscreteRobustPlannerAgent built from the shipped routes_behaviours.json with `__class__` switched, on an
    IntersectionLiteEnv: the plan, tree and RNG words of the reference (the change_vehicles entries are skipped)."""
    from rl_agents_b200.agents.robust.robust import DiscreteRobustPlannerAgent
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv
    shipped = dict(G["routes_behaviours"], __class__="<class '%s.%s'>" % (DiscreteRobustPlannerAgent.__module__,
                                                                          DiscreteRobustPlannerAgent.__name__))
    for name in ("routes_behaviours_s0", "routes_behaviours_s1", "routes_behaviours_s2"):
        g = G["cases"][name]
        env = IntersectionLiteEnv(np.array(g["words"], dtype=np.int32))
        agent = DiscreteRobustPlannerAgent(env, json.loads(json.dumps(shipped)))
        agent.seed(g["seed"])
        assert agent.plan(env.observation()) == g["plan"], name
        assert rng_state(agent.planner.np_random) == g["rng_state"]
        d = agent.planner.last_tree.tree_dict(0)
        assert d["parent"].tolist() == g["tree"]["parent"] and f64_hex(d["lower"]) == g["tree"]["lower"]
        assert env.words.tolist() == g["words"]                  # the models are copies


def test_agent_wavefront_and_random_hypotheses():
    """`wavefront: K` through the agent equals robust_plan at width K; a "random" chain follows the spec's hash."""
    from rl_agents_b200.agents.robust.robust import DiscreteRobustPlannerAgent
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv
    words = isc.family("phases")[6].pack()
    args = ("random", 0, 2)
    for width in (1, 8, 64):
        env = IntersectionLiteEnv(words)
        agent = DiscreteRobustPlannerAgent(env, {"budget": 600, "gamma": 0.9, "wavefront": width,
                                                 "models": chains(args)})
        agent.seed(3)
        plan, t = planners.robust_plan(oracle_models(words, args), 600, 0.9, 0.0, np_random(3), width=width)
        assert agent.plan(env.observation()) == plan
        assert_same_tree(agent.planner.last_tree.tree_dict(0), t)


def test_refusals_still_hold():
    import torch
    from rl_agents_b200 import _lib
    from rl_agents_b200.agents.robust.robust import DiscreteRobustPlanner
    from rl_agents_b200.engine.opd import OPDSpeculativeEngine, OPDWaveEngine
    from rl_agents_b200.envs import HighwayLiteEnv
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv
    words = model_words(oit.make_intersection_state(0).pack(), chains((0, 1, 2)))
    root = torch.tensor(words, dtype=torch.int32, device="cuda")
    # more than 8 models: the engine, and the C ABI behind it
    with pytest.raises(ValueError, match="at most 8 models"):
        OPDWaveEngine(_lib.ENV_INTERSECTION, 3, 60, 0.9, 1, n_models=9)
    eng = OPDWaveEngine(_lib.ENV_INTERSECTION, 3, 60, 0.9, 1, n_models=8)
    eng.cfg.n_models = 9
    with pytest.raises(_lib.B2Error, match="n_models must be in 0..8"):
        eng.plan(torch.tensor(np.concatenate([words] * 3), dtype=torch.int32, device="cuda"))
    # models of different env kinds
    planner = DiscreteRobustPlanner(None, {"budget": 60, "gamma": 0.9})
    with pytest.raises(ValueError, match="share the env kind"):
        planner.plan([IntersectionLiteEnv(words[0]), HighwayLiteEnv(seed=0)], None)
    # IntersectionLite with another action count, joint or not
    for n_actions in (2, 5):
        for m in (0, 3):
            eng = OPDWaveEngine(_lib.ENV_INTERSECTION, n_actions, 60, 0.9, 1, n_models=m)
            with pytest.raises(_lib.B2Error, match="IntersectionLite has 3 actions"):
                eng.plan(root if m else root[0].contiguous())
    # the speculative kernel stays plain OPD
    spec = OPDSpeculativeEngine(_lib.ENV_INTERSECTION, 3, 60, 0.9, 8)
    spec.cfg.n_models = 3
    with pytest.raises(_lib.B2Error, match="n_models = 0"):
        spec.plan(root)
