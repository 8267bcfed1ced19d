"""DROP on IntersectionLite route hypotheses, without a GPU: the golden generator reproduces its JSON, the oracle's
robust_plan equals every golden of the unmodified reference (tree, bounds, plan and RNG words), and the product's and
the oracle's `set_route_at_intersection` agree word for word (docs/INTERSECTION_LITE_SPEC.md, "Route hypotheses")."""
import filecmp
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import intersection as oit
from oracle import planners, ref_loader
from oracle.intersection_routes import IntersectionLiteRoutes, set_route_at_intersection
from tests import intersection_scenes as isc
from tests.util import load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
G = load_golden("golden_drop_intersection.json")
ARGS = (0, 1, 2, 5, -1, "random")


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def f64(hexstr):
    return np.frombuffer(bytes.fromhex(hexstr), dtype="<f8")


def oracle_models(g):
    """The models the config's chains make from the case's scene (the drop-in's preprocess_env, as robust.py:66)."""
    from rl_agents_b200.agents.common.factory import preprocess_env
    env = IntersectionLiteRoutes(oit.IntersectionLiteState.unpack(np.array(g["words"], dtype=np.int32)))
    return [preprocess_env(env, chain) for chain in g["config"]["models"]]


def all_scenes():
    out = [oit.make_intersection_state(s) for s in range(8)]
    for name in isc.FAMILY_NAMES:
        out.extend(isc.family(name))
    return out


@pytest.mark.skipif(not ref_loader.reference_available(), reason="needs the reference tree")
def test_golden_generator_reproduces_its_json(tmp_path):
    out = tmp_path / "golden.json"
    subprocess.run([sys.executable, os.path.join(GOLDEN, "make_golden_drop_intersection.py"), "--out", str(out)],
                   check=True, cwd=ROOT, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    assert filecmp.cmp(str(out), os.path.join(GOLDEN, "golden_drop_intersection.json"), shallow=False)


def test_golden_cases_cover_what_they_are_named_for():
    shipped = G["routes_behaviours"]
    assert shipped["budget"] == 20 and shipped["gamma"] == 0.9
    assert [[p["method"] for p in chain] for chain in shipped["models"]] == \
        [["set_route_at_intersection", "change_vehicles"]] * 3
    assert [chain[0]["args"] for chain in shipped["models"]] == [0, 1, 2]
    cases = G["cases"]
    for name in ("routes_behaviours_s0", "routes_behaviours_s1", "routes_behaviours_s2"):
        assert cases[name]["config"] == shipped
    assert {len(cases[n]["config"]["models"]) for n in ("m2_s3_b200", "m2_s3_b600")} == {2}
    assert {len(cases[n]["config"]["models"]) for n in ("m3_s4_b200", "m3_s4_b600")} == {3}
    assert any(c["config"].get("terminal_reward", 0) > 0 for c in cases.values())
    assert cases["si0_s1_b200"]["words"][129] == 0 and cases["si2_s2_b200"]["words"][129] == 2
    assert sorted(cases["si0_s1_b200"]["tree"]["action"][1:3]) == [oit.A_IDLE, oit.A_FASTER]
    assert sorted(cases["si2_s2_b200"]["tree"]["action"][1:3]) == [oit.A_SLOWER, oit.A_IDLE]
    assert cases["t12_s7_b200"]["words"][128] == 12
    assert any(chain[0]["args"] == "random" for c in cases.values() for chain in c["config"]["models"])


@pytest.mark.parametrize("name", sorted(G["cases"]))
def test_robust_plan_equals_the_reference_golden(name):
    g = G["cases"][name]
    c = g["config"]
    rng = np_random(g["seed"])
    plan, t = planners.robust_plan(oracle_models(g), c["budget"], c["gamma"], c.get("terminal_reward", 0), rng)
    tr = g["tree"]
    assert plan == g["plan"]
    assert t.parent == tr["parent"] and t.action == tr["action"] and t.count == tr["count"]
    assert np.array_equal(np.array(t.lower), f64(tr["lower"])) and np.array_equal(np.array(t.upper), f64(tr["upper"]))
    assert rng_state(rng) == g["rng_state"]


def test_golden_trees_reach_crashes_and_arrivals():
    """The family cases are there for their terminal nodes: some model crashes or arrives inside the tree."""
    for name in ("arrival4_b300", "full0_b300", "crossing1_b300", "ties4_b300", "arrival0_random_b200"):
        g = G["cases"][name]
        c = g["config"]
        _, t = planners.robust_plan(oracle_models(g), c["budget"], c["gamma"], c.get("terminal_reward", 0),
                                    np_random(g["seed"]))
        assert any(any(d) for d in t.done), name


@pytest.mark.parametrize("arg", ARGS, ids=[str(a) for a in ARGS])
def test_product_and_oracle_set_route_agree_word_for_word(arg):
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv
    changed = 0
    for st in all_scenes():
        words = st.pack()
        env = IntersectionLiteEnv(words)
        out = env.set_route_at_intersection(arg)
        ref = set_route_at_intersection(st, arg).pack()
        assert np.array_equal(out.words, ref)
        assert np.array_equal(env.words, words) and out is not env
        assert np.array_equal(IntersectionLiteRoutes(st).set_route_at_intersection(arg).state.pack(), ref)
        changed += int(not np.array_equal(ref, words))
    assert changed > 0


@pytest.mark.parametrize("arg", ARGS, ids=[str(a) for a in ARGS])
def test_set_route_rewrites_only_the_approach(arg):
    for st in all_scenes():
        before = st.pack()
        out = set_route_at_intersection(st, arg)
        assert np.array_equal(st.pack(), before)                       # the receiver is unchanged
        after = out.pack()
        route = after[32:48]
        eligible = ((st.flags & 1) != 0) & (st.s < oit.APPROACH)
        eligible[0] = False
        assert np.array_equal(np.delete(after, np.arange(33, 48)), np.delete(before, np.arange(33, 48)))
        assert np.array_equal(route[~eligible], st.route[~eligible])   # ego, s >= 40 and absent slots
        assert np.array_equal(route // 3, st.route // 3)
        if arg != "random":
            assert np.all(route[eligible] % 3 == arg % 3)
        for k in np.nonzero(eligible)[0]:
            if arg == "random":
                h = ((st.t * 16 + int(k)) * 2654435761 + st.spawn_seq * 40503) % 2 ** 32
                assert route[k] % 3 == (h >> 16) % 3


def test_random_routes_vary_with_the_decision_time():
    differ = 0
    for st in all_scenes():
        later = st.copy()
        later.t += 1
        differ += int(not np.array_equal(set_route_at_intersection(st, "random").route,
                                         set_route_at_intersection(later, "random").route))
    assert differ > 0


@pytest.mark.parametrize("bad", [1.0, "left", "Random", None, True, [0], np.float32(2)])
def test_bad_arguments_raise_value_error(bad):
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv
    st = oit.make_intersection_state(0)
    with pytest.raises(ValueError):
        set_route_at_intersection(st, bad)
    with pytest.raises(ValueError):
        IntersectionLiteEnv(st.pack()).set_route_at_intersection(bad)


def test_numpy_integer_arguments_are_integers():
    from rl_agents_b200.envs.intersection_lite import IntersectionLiteEnv
    st = oit.make_intersection_state(1)
    for arg in (np.int32(2), np.int64(-2)):
        ref = set_route_at_intersection(st, int(arg)).pack()
        assert np.array_equal(set_route_at_intersection(st, arg).pack(), ref)
        assert np.array_equal(IntersectionLiteEnv(st.pack()).set_route_at_intersection(arg).words, ref)
