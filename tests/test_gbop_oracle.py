"""Pin the GBOP-T and GBOP-D restatements (oracle/planners.py: state_aware_plan, graph_based_plan) to
tests/golden/golden_gbop.json, recorded from the UNMODIFIED reference by tests/golden/make_golden_gbop.py: plan,
state values / node bounds and the planner RNG's position, exactly.  Also count the backup queue entries the
searches need, the number the device kernels' queues must hold (one entry per FIFO pop, in the same order)."""
import sys

import numpy as np
import pytest

from oracle import envs as oenvs
from oracle import planners
from tests.util import load_golden

G = load_golden("golden_gbop.json")


def np_random(seed):
    return np.random.Generator(np.random.PCG64(np.random.SeedSequence(seed)))


def rng_state(rng):
    st = rng.bit_generator.state
    return {"state": str(st["state"]["state"]), "inc": str(st["state"]["inc"]),
            "has_uint32": int(st["has_uint32"]), "uinteger": int(st["uinteger"])}


def env(name):
    m = G["mdps"][name]
    return oenvs.FiniteMDPLite(m["T"], m["R"], m["term"], state=0)


def gbopt(g, rng=None):
    c = g["config"]
    return planners.state_aware_plan(env(g["mdp"]), 0, c["budget"], c["gamma"], rng or np_random(g["seed"]),
                                     terminal_reward=c.get("terminal_reward", 0.0))


def gbopd(g, rng=None):
    c = g["config"]
    return planners.graph_based_plan(oenvs.LegacyStepEnv(env(g["mdp"])), 0, c["budget"], c["gamma"],
                                     rng or np_random(g["seed"]), g["accuracy"], g["sampling_timeout"])


def max_queue_entries(planner, run):
    """Call run(), which runs the oracle function `planner` (its backups are `queue = [...]; while queue:
    queue.pop(0) ...`), and count the pops of each backup's queue list; -> (run's result, the most entries one
    backup put through its queue).  Only the calls made directly in planner's own code are watched
    (sys.monitoring), and every call site that is not a list pop is switched off after its first call, so the
    oracle runs unmodified and at nearly full speed."""
    mon = sys.monitoring
    tool = mon.PROFILER_ID
    mon.use_tool_id(tool, "gbop queue count")
    current, counts = [None], []

    def on_call(code, offset, callable_, arg0):
        if callable_ is not list.pop:
            return mon.DISABLE
        if arg0 is not current[0]:           # a new backup binds a new queue list
            current[0] = arg0
            counts.append(0)
        counts[-1] += 1

    try:
        mon.register_callback(tool, mon.events.CALL, on_call)
        mon.set_local_events(tool, planner.__code__, mon.events.CALL)
        out = run()
    finally:
        mon.set_local_events(tool, planner.__code__, 0)
        mon.register_callback(tool, mon.events.CALL, None)
        mon.free_tool_id(tool)
        mon.restart_events()
    return out, max(counts)


@pytest.mark.parametrize("key", sorted(G["gbopt"]))
def test_state_aware_oracle_matches_the_reference(key):
    g = G["gbopt"][key]
    rng = np_random(g["seed"])
    plan, t, state_values, leaves = gbopt(g, rng)
    assert plan == g["plan"]
    # the reference materialises a default entry wherever it reads a bound (a defaultdict): compare the full table
    default = 1 / (1 - g["config"]["gamma"])
    S = len(G["mdps"][g["mdp"]]["T"])
    assert all(state_values.get(s, default) == g["state_values"].get(str(s), default) for s in range(S))
    assert set(map(str, state_values)) <= set(g["state_values"])
    assert len(leaves) == g["n_leaves"] and len(set(t.obs)) == g["n_states"]
    assert sum(t.depth[leaf] for leaf in leaves) == g["leaf_depth_sum"]
    assert sum(t.lower[leaf] for leaf in leaves) == g["leaf_lower_sum"]
    assert rng_state(rng) == g["rng_state"]          # get_plan's two walks consume the same draws


@pytest.mark.parametrize("key", sorted(G["gbopd"]))
def test_graph_based_oracle_matches_the_reference(key):
    g = G["gbopd"][key]
    assert g["accuracy"] == 0              # the reference's set-ordered parent pushes only reach a fixed point there
    rng = np_random(g["seed"])
    plan, nodes = gbopd(g, rng)
    assert plan == g["plan"]
    assert {str(s): [n["lower"], n["upper"], n["expanded"]] for s, n in sorted(nodes.items())} == g["nodes"]
    assert rng_state(rng) == g["rng_state"]


def test_golden_cases_cover_what_they_are_named_for():
    gt, gd = G["gbopt"], G["gbopd"]
    assert gt["quantized6_b90_g0.9"]["tied"] and not gt["loop_b1000_g0.9"]["tied"]
    assert set(np.unique(G["mdps"]["quantized6"]["R"])) == {0.0, 0.5}
    term = G["mdps"]["large1_term4"]["term"]
    assert sum(term) >= 4 and gt["large1_term4_tr0.3_b400_g0.85"]["config"]["terminal_reward"] == 0.3
    # trap: rewards -1 that GBOP-D accepts, and a tie-break draw in most sampling steps
    assert min(map(min, G["mdps"]["trap"]["R"])) == -1.0
    assert gd["trap_b500_g0.9_acc0"]["rng_state"] != rng_state(np_random(gd["trap_b500_g0.9_acc0"]["seed"]))


def test_state_aware_oracle_raises_the_references_error():
    e = G["errors"]["gbopt_trap_b100_g0.9"]
    with pytest.raises(ValueError) as info:
        planners.state_aware_plan(env("trap"), 0, 100, 0.9, np_random(0))
    assert str(info.value) == e["message"]


def test_loop_backups_outgrow_the_first_device_queue_sizes():
    """One backup of each loop search needs more queue entries than the engines allocate first (GBOPEngine:
    64 x node capacity, GBOPDEngine: 256 x states), so the device searches of the GPU regression tests must grow
    their queues to plan what the reference plans."""
    g = G["gbopt"]["loop_b1000_g0.9"]
    (plan, _, _, _), entries = max_queue_entries(planners.state_aware_plan, lambda: gbopt(g))
    assert plan == g["plan"]
    A = len(G["mdps"]["loop"]["R"][0])
    capacity = 1 + (g["config"]["budget"] // A) * A
    assert entries > 64 * capacity, entries
    g = G["gbopd"]["loop_b500_g0.9_acc0"]
    (plan, _), entries = max_queue_entries(planners.graph_based_plan, lambda: gbopd(g))
    assert plan == g["plan"]
    assert entries > 256 * len(G["mdps"]["loop"]["T"]), entries


def test_queue_count_sees_every_backup():
    """The counter on a smaller search: the largest backup of budget 600 on loop puts 1053 entries through its
    queue, within GBOPEngine's first queue (64 x 601 nodes)."""
    g = dict(G["gbopt"]["loop_b1000_g0.9"], config={"budget": 600, "gamma": 0.9})
    _, entries = max_queue_entries(planners.state_aware_plan, lambda: gbopt(g))
    assert entries == 1053
