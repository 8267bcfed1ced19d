"""Deterministic IntersectionLite scene families for the step-path tests, and a census of the paths a trajectory
reaches.

The generator of `oracle.intersection.make_intersection_state` makes one kind of scene: the ego at s = 10 on its
approach, up to 8 others on the approaches, spawn clock 0.  Trajectories from such scenes never reach several paths
of `il::step`: the ego's arrival (and a crash in the same step), exact front ties, a spawn that finds every slot
taken or takes a slot freed in the same sub-step, a blocker exactly at the entry's clear distance, positions exactly
at the spec's thresholds, the spawn counter's wrap -- and since every scene starts at spawn clock 0, the two scenes
of a warp always spawn on the same sub-step.  Each family below is built to reach some of them, and `census` counts,
on the numpy oracle, how often a trajectory does -- so that a GPU test that passes is known to have exercised the
path.

Every scene stays inside the state domain of docs/INTERSECTION_LITE_SPEC.md: slot 0 is the ego on route 0, routes
0..11, speed index 0..2, spawn clock 0..22, spawn_seq 0..2^31 - 1, finite words.
"""
import functools
from collections import Counter

import numpy as np

from oracle import intersection as oit

f32 = np.float32
V = oit.V_SLOTS
N_DECISIONS = 13
SEQ_MAX = 0x7fffffff

PATHS = ("arrival", "arrive_crash", "front_tie", "spawn", "blocked", "spawn_full", "spawn_freed", "clear_edge",
         "crossing_hit", "box_crossing_hit", "lane_hit", "box_lane_pair", "ego_crash", "yield", "depart_left",
         "depart_straight", "depart_right", "seq_wrap", "odd_action")

LEN = [f32(x) for x in oit.LEN]
PRIO_END = [f32((oit.APPROACH + b) + oit.PRIO_PAST) for b in oit.BOX]
ARC_END = [f32(oit.APPROACH + oit.ARC_LEFT), f32(oit.APPROACH + oit.ARC_RIGHT)]


# ------------------------------------------------------------------------------------------------ scene helpers ----
def blank(ego_s=10.0, ego_v=4.5, si=1, clock=0, seq=0, t=0):
    st = oit.IntersectionLiteState()
    st.s, st.v = np.zeros(V, f32), np.zeros(V, f32)
    st.route, st.flags = np.zeros(V, np.int32), np.zeros(V, np.int32)
    st.s[0], st.v[0], st.flags[0] = f32(ego_s), f32(ego_v), 1
    st.t, st.speed_index, st.spawn_clock, st.spawn_seq, st.arrived = int(t), int(si), int(clock), int(seq), 0
    return st


def put(st, slot, route, s, v, crashed=False):
    st.s[slot], st.v[slot], st.route[slot], st.flags[slot] = f32(s), f32(v), int(route), 1 | (2 if crashed else 0)


def ulp_step(x, n):
    """x moved by n units in the last place (positive finite x)"""
    return np.array([f32(x).view(np.int32) + n], np.int32).view(f32)[0]


def spawn_route(k):
    """The route the spawn with counter k picks (spec: h = k * 2654435761 + 40503 mod 2^32, (h >> 16) mod 12)."""
    return int((((int(k) * 2654435761 + 40503) & 0xffffffff) >> 16) % oit.N_ROUTES)


def seq_for_entry(entry, start=0):
    """The first spawn counter >= start whose spawn comes in on `entry`."""
    k = int(start)
    while spawn_route(k) // 3 != entry:
        k += 1
    return k


def spawn_substeps(clock):
    """The sub-steps of the next decision on which a scene at spawn clock `clock` spawns."""
    return frozenset(sub for sub in range(oit.SUBSTEPS) if (int(clock) + sub + 1) % oit.SPAWN_PERIOD == 0)


# ------------------------------------------------------------------------------------------------------ families ----
def phases_scenes():
    """Generator scenes with the spawn clock at every value 0..22, ordered so that scenes 2i and 2i + 1 are 11 apart:
    the two scenes of every warp spawn on different sub-steps at every decision."""
    clocks = [c for i in range(11) for c in (i, i + 11)] + [22]
    out = []
    for i, c in enumerate(clocks):
        st = oit.make_intersection_state(900 + i, n_others=(8, 12, 5)[i % 3])
        st.spawn_clock = c
        out.append(st)
    return out


def arrival_scenes():
    """The ego past its arc, within one or two decisions of its route's end, at every speed index; in some scenes a
    stopped, crashed vehicle on the route that shares the ego's exit (E straight, westward on y = 2) near the end, so
    that the crashed ego still rolls past its end: it arrives and crashes in the same step."""
    out = []
    for si in range(3):
        for d, others in ((1.5, False), (5.0, True), (9.0, False), (14.0, True)):
            st = blank(ego_s=LEN[0] - f32(d), ego_v=max(4.5 * si, 2.0), si=si, clock=(7 * si + int(d)) % 23,
                       seq=40 + si)
            if others:
                put(st, 1, 4, 30.0, 8.0)
                put(st, 2, 7, 20.0, 7.0)
                put(st, 3, 11, 60.0, 8.5)
            out.append(st)
    for si, d, s_hit in ((1, 6.0, 88.0), (2, 6.0, 89.5), (2, 9.0, 90.5), (1, 4.0, 91.5), (2, 3.0, 91.0),
                         (2, 12.0, 91.9)):
        st = blank(ego_s=LEN[0] - f32(d), ego_v=4.5 * si, si=si, clock=3 * si, seq=77)
        put(st, 2, 10, s_hit, 0.0, crashed=True)
        out.append(st)
    return out


def _full_scene(entry, clock, freed):
    """15 others present, none of them within ENTRY_CLEAR of the spawn's entry; `freed`: slot 5 is at its route's end
    and leaves on the spawn sub-step, so the spawn takes the slot it has just freed."""
    st = blank(ego_s=20.0, ego_v=4.5, clock=clock, seq=seq_for_entry(entry, 1000 + 37 * entry))
    slots_per_entry = [0, 0, 0, 0]
    slots_per_entry[0] = 1                                     # the ego
    positions = (16.0, 23.0, 30.0, 62.0, 72.0, 82.0)
    for k in range(1, V):
        route = (5 * k + entry) % oit.N_ROUTES
        e = route // 3
        s = positions[slots_per_entry[e] % len(positions)]
        slots_per_entry[e] += 1
        put(st, k, route, s, 6.0 + (k % 4))
    if freed:
        route = st.route[5]
        st.s[5], st.v[5] = ulp_step(LEN[route % 3], -8), f32(8.0)
    return st


def full_scenes():
    out = []
    for entry in range(4):
        out.append(_full_scene(entry, 22, False))
        out.append(_full_scene(entry, 22, True))
        out.append(_full_scene(entry, 10, False))
    return out


def blocked_scenes():
    """At the spawn sub-step (the first), a stopped, crashed vehicle one ulp below, exactly at, or one ulp above
    ENTRY_CLEAR on the entry the spawn counter picks; every turn of every entry."""
    out = []
    for entry in range(4):
        for n, off in enumerate((-1, 0, 1)):
            st = blank(ego_s=20.0, ego_v=4.5, clock=22, seq=seq_for_entry(entry, 50 + 11 * entry + n))
            put(st, 1 + n, 3 * entry + (n + entry) % 3, ulp_step(oit.ENTRY_CLEAR, off), 0.0, crashed=True)
            put(st, 6, 3 * ((entry + 1) % 4) + 1, 24.0, 7.0)
            put(st, 9, 3 * ((entry + 2) % 4) + 2, 66.0, 8.0)
            out.append(st)
    return out


def ties_scenes():
    """Exact s ties between two front candidates of a follower, with different speeds (so the tie decides its IDM):
    two vehicles on the follower's route, or one on its route and one of the same entry on another route, still on the
    approach; the lower slot is either one.  Every entry."""
    out = []
    for entry in range(4):
        for kind in range(2):
            for low_first in (True, False):
                st = blank(ego_s=3.0 if entry else 2.0, ego_v=4.5, clock=5 * entry + kind, seq=300 + entry)
                r = 3 * entry + 1
                other = r if kind == 0 else 3 * entry + (0 if low_first else 2)
                a, b = (3, 7) if low_first else (7, 3)
                put(st, a, r, 30.0, 8.5)
                put(st, b, other, 30.0, 1.0)
                put(st, 5, r, 16.0, 7.0)                    # the follower
                put(st, 11, 3 * ((entry + 2) % 4), 18.0, 6.5)
                out.append(st)
    return out


def boundaries_scenes():
    """Vehicles one ulp either side of, and exactly at, each threshold of the spec, stopped so that the first
    sub-step's post-integration tests see the exact value too: the yielder's window (YIELD_FROM, STOP_LINE), the
    priority window (PRIO_FROM, the three PRIO_END), APPROACH, the arc ends and the route lengths (the ego's too)."""
    out = []
    cases = []
    # (threshold, route of the vehicle at it, partner: route, s, v)
    cases += [(oit.YIELD_FROM, 1, (4, 30.0, 7.0)), (oit.STOP_LINE, 1, (7, 40.0, 7.0))]     # a yielder at the edge
    cases += [(oit.PRIO_FROM, 4, (1, 20.0, 5.0))]                                           # priority vehicles
    cases += [(PRIO_END[0], 3, (1, 20.0, 5.0)), (PRIO_END[1], 7, (2, 20.0, 5.0)), (PRIO_END[2], 11, (1, 20.0, 5.0))]
    cases += [(oit.APPROACH, 6, (7, 36.0, 6.0)), (oit.APPROACH, 2, (1, 37.0, 0.0))]         # same entry, behind
    cases += [(ARC_END[0], 9, (10, 50.0, 7.0)), (ARC_END[1], 5, (4, 55.0, 7.0))]
    cases += [(LEN[0], 3, (3, 80.0, 8.0)), (LEN[1], 7, (7, 80.0, 8.0)), (LEN[2], 11, (11, 78.0, 8.0))]
    for i, (b, route, (pr, ps, pv)) in enumerate(cases):
        for off in (-1, 0, 1):
            st = blank(ego_s=4.0, ego_v=4.5, clock=(3 * i + off) % 23, seq=500 + i)
            put(st, 2 + (i % 3), route, ulp_step(b, off), 0.0)
            put(st, 8, pr, ps, pv)
            out.append(st)
    for off in (-1, 0, 1):                                  # the ego at its route's end, stopped at speed index 0
        st = blank(ego_s=ulp_step(LEN[0], off), ego_v=0.0, si=0, clock=4, seq=610)
        put(st, 3, 5, 20.0, 7.0)
        out.append(st)
    return out


def _crossing_candidates(entry, turn):
    a_route = 3 * entry + turn
    for rb in range(oit.N_ROUTES):
        if rb // 3 == entry:
            continue
        for sa, sb in ((38.0, 38.0), (38.0, 36.0), (36.0, 38.0), (39.5, 35.0), (35.0, 39.5)):
            st = blank(ego_s=2.0, ego_v=4.5, clock=(entry + 5 * turn) % 23, seq=700 + rb)
            put(st, 4, a_route, sa, 8.0)
            put(st, 9, rb, sb, 8.0)
            yield st


def _box_crossing(st):
    """Does a crossing-path collision (disc test) happen inside the box within one IDLE decision?"""
    found = []

    def obs(hit, lane, present, **_):
        box = _in_box(st_copy.route, st_copy.s)
        for i in range(V):
            for j in range(i + 1, V):
                if hit[i, j] and not lane[i, j] and box[i] and box[j]:
                    found.append((i, j))
    st_copy = st.copy()
    oit.intersection_step(st_copy, oit.A_IDLE, on_substep=obs)
    return bool(found)


def crossing_scenes():
    """Pairs of other vehicles on conflicting routes, timed to meet inside the box (found by running the oracle), for
    every entry and both arcs; and a vehicle just inside the box next to one of its entry's still on the approach
    (less than 5 m apart in s, more than 3.5 m apart on the ground: no collision)."""
    out = []
    for entry in range(4):
        for turn in (0, 2):
            n = 0
            for st in _crossing_candidates(entry, turn):
                if _box_crossing(st):
                    out.append(st)
                    n += 1
                    if n == 2:
                        break
            assert n == 2, (entry, turn)
    for entry in range(4):
        st = blank(ego_s=2.0 if entry else 20.0, ego_v=4.5, clock=entry, seq=800 + entry)
        put(st, 3, 3 * entry, 40.5, 2.0)
        put(st, 6, 3 * entry + 1, 36.5, 0.0)
        out.append(st)
    return out


def wrap_scenes():
    """spawn_seq a few steps below 2^31 - 1: the counter wraps to 0 within the trajectory."""
    out = []
    for i, (k, clock) in enumerate(((0, 22), (1, 5), (2, 15), (3, 0), (0, 9), (4, 20))):
        st = oit.make_intersection_state(950 + i)
        st.spawn_seq, st.spawn_clock = SEQ_MAX - k, clock
        out.append(st)
    return out


def stale_scenes():
    """Absent slots whose s, v and route words are not zero (and some with a stale crash bit): within ENTRY_CLEAR of
    the spawn's entry, just ahead of a present vehicle on its route, next to the ego; and vehicles that start
    crashed."""
    out = []
    for i in range(10):
        rng = np.random.default_rng(960 + i)
        st = oit.make_intersection_state(960 + i, n_others=6)
        st.spawn_clock = (22, 11, 3)[i % 3]
        spawn_entry = spawn_route(st.spawn_seq) // 3
        present = np.nonzero(st.flags & 1)[0]
        absent = [k for k in range(1, V) if not st.flags[k] & 1]
        for j, a in enumerate(absent):
            if j % 3 == 0:
                st.route[a], st.s[a] = 3 * spawn_entry + j % 3, f32(rng.uniform(0.0, 13.0))
            else:
                p = present[rng.integers(len(present))]
                st.route[a], st.s[a] = st.route[p], f32(st.s[p] + rng.uniform(0.5, 4.0))
            st.v[a] = f32(rng.uniform(0.5, 9.0))
            st.flags[a] = 2 if j % 4 == 1 else 0
        for p in present[1:][i % 2::3]:
            st.flags[p] = 3
        out.append(st)
    return out


_FAMILIES = {"phases": phases_scenes, "arrival": arrival_scenes, "full": full_scenes, "blocked": blocked_scenes,
             "ties": ties_scenes, "boundaries": boundaries_scenes, "crossing": crossing_scenes, "wrap": wrap_scenes,
             "stale": stale_scenes}
FAMILY_NAMES = tuple(_FAMILIES)


@functools.lru_cache(maxsize=None)
def _family_words(name):
    return tuple(tuple(s.pack().tolist()) for s in _FAMILIES[name]())


def family(name):
    """Fresh states of a family (deterministic)."""
    return [oit.IntersectionLiteState.unpack(np.array(w, np.int32)) for w in _family_words(name)]


# -------------------------------------------------------------------------------------------------- trajectories ----
def available(state):
    si = state.speed_index
    return [oit.A_IDLE] + ([oit.A_FASTER] if si < 2 else []) + ([oit.A_SLOWER] if si > 0 else [])


def avail_mask(state):
    return sum(1 << a for a in available(state))


class ActionStream(object):
    """Actions from a fixed RNG over the available ones; one in six is an action the scene does not offer: SLOWER at
    speed index 0, FASTER at 2, or the out-of-range 7 (all three leave the speed index alone)."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)

    def __call__(self, state):
        if self.rng.uniform() < 1.0 / 6.0:
            odd = [7] + ([oit.A_SLOWER] if state.speed_index == 0 else []) + \
                  ([oit.A_FASTER] if state.speed_index == 2 else [])
            return int(odd[self.rng.integers(len(odd))])
        av = available(state)
        return int(av[self.rng.integers(len(av))])


def _in_box(route, s):
    return (s >= oit.APPROACH) & (s < (oit.APPROACH + np.array([oit.BOX[t] for t in route % 3], f32)))


def _census_step(state, action, counts):
    ego_was, arrived_was = bool(state.flags[0] & 2), bool(state.arrived)
    if action not in available(state):
        counts["odd_action"] += 1
    subs = []

    def obs(**kw):
        d = {k: (np.array(v, copy=True) if isinstance(v, np.ndarray) else v) for k, v in kw.items()}
        d["s"], d["route"], d["flags"] = state.s.copy(), state.route.copy(), state.flags.copy()
        subs.append(d)
    r, term, trunc = oit.intersection_step(state, action, on_substep=obs)
    for d in subs:
        present, s_f = d["present"], d["s_front"]
        for i in np.nonzero(present & d["has_front"])[0]:
            counts["front_tie"] += int((s_f[i] == s_f[i].min()).sum() > 1)
        counts["yield"] += int((d["yields"] & present).sum())
        hit, lane, s = d["hit"], d["lane"], d["s"]
        entry = d["route"] // 3
        box = _in_box(d["route"], s)
        for i in range(V):
            for j in range(i + 1, V):
                if hit[i, j]:
                    counts["lane_hit" if lane[i, j] else "crossing_hit"] += 1
                    if not lane[i, j] and box[i] and box[j]:
                        counts["box_crossing_hit"] += 1
                # a vehicle just in the box and one of its entry on the approach: not a shared lane
                if (present[i] and present[j] and entry[i] == entry[j] and d["route"][i] != d["route"][j]
                        and (s[i] < oit.APPROACH) != (s[j] < oit.APPROACH) and abs(float(s[i] - s[j])) < oit.LENGTH):
                    counts["box_lane_pair"] += 1
        for k in np.nonzero(d["left"])[0]:
            counts[("depart_left", "depart_straight", "depart_right")[d["route"][k] % 3]] += 1
        sp = d["spawn"]
        if sp is not None:
            counts["seq_wrap"] += int(sp["seq"] == SEQ_MAX)
            pres = (d["flags"] & 1) != 0
            if sp["slot"] > 0:
                pres[sp["slot"]] = False          # as it was before the spawn
            on_entry = pres & (d["route"] // 3 == sp["route"] // 3)
            counts["clear_edge"] += int(bool((on_entry & (s == oit.ENTRY_CLEAR)).any()))
            if not sp["clear"]:
                counts["blocked"] += 1
            elif sp["slot"] < 0:
                counts["spawn_full"] += 1
            else:
                counts["spawn"] += 1
                counts["spawn_freed"] += int(bool(d["left"][sp["slot"]]))
    if bool(state.flags[0] & 2) and not ego_was:
        counts["ego_crash"] += 1
    if state.arrived and not arrived_was:
        counts["arrival"] += 1
        counts["arrive_crash"] += int(bool(state.flags[0] & 2))
    return r, term, trunc


def oracle_trajectory(state, n_decisions=N_DECISIONS, seed=0, counts=None):
    """Steps a copy of `state` n times with ActionStream(seed) on the numpy oracle.  Returns (actions, words
    [n + 1, 136] (the start state first), rewards f32 [n], flags [n] (bit0 terminated, bit1 truncated), avail [n]
    (available-action mask of each new state)).  With `counts` (a Counter), adds the census of the paths reached."""
    s = state.copy()
    pick = ActionStream(seed)
    acts, words, rews, flags, avail = [], [s.pack()], [], [], []
    for _ in range(n_decisions):
        a = pick(s)
        if counts is None:
            r, term, trunc = oit.intersection_step(s, a)
        else:
            r, term, trunc = _census_step(s, a, counts)
        acts.append(a)
        words.append(s.pack())
        rews.append(f32(r))
        flags.append((1 if term else 0) | (2 if trunc else 0))
        avail.append(avail_mask(s))
    return (np.array(acts, np.int32), np.stack(words), np.array(rews, np.float32), np.array(flags, np.int32),
            np.array(avail, np.int32))


@functools.lru_cache(maxsize=None)
def _family_runs(name, n_decisions):
    runs, counts = [], []
    for i, s in enumerate(family(name)):
        c = Counter()
        runs.append(oracle_trajectory(s, n_decisions, seed=i, counts=c))
        counts.append(c)
    return runs, counts


def family_trajectories(name, n_decisions=N_DECISIONS):
    """Oracle trajectories of every scene of a family (scene i uses ActionStream(i))."""
    return _family_runs(name, n_decisions)[0]


def census(name, n_decisions=N_DECISIONS):
    """Counter of the paths the family's trajectories reach (keys: PATHS)."""
    total = sum(_family_runs(name, n_decisions)[1], Counter())
    return Counter({k: total[k] for k in PATHS})


def divergent_pairs(words):
    """words [n_scenes, n_decisions + 1, 136] of a batch in warp order: the number of warps (scenes 2g, 2g + 1) whose
    two scenes spawn on different sub-steps in at least one decision."""
    n = 0
    for g in range(0, len(words) - 1, 2):
        a, b = words[g], words[g + 1]
        n += any(spawn_substeps(a[k][130]) != spawn_substeps(b[k][130]) for k in range(len(a) - 1))
    return n
