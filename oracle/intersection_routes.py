"""Route hypotheses on IntersectionLite -- numpy statement of `set_route_at_intersection` (docs/INTERSECTION_LITE_SPEC.md,
"Route hypotheses") on IntersectionLiteState (TEST INFRASTRUCTURE).

`IntersectionLiteRoutes` is oracle.intersection.IntersectionLite with the method the reference's preprocess_env
(rl_agents/agents/common/factory.py:97-116) looks up on `env.unwrapped`, so that the unmodified
DiscreteRobustPlannerAgent builds its route-hypothesis models from it.  `step` is unchanged.  Kept apart from
oracle/intersection.py, which stays as it is.
"""
import numpy as np

from oracle.intersection import APPROACH, V_SLOTS, IntersectionLite

N_TURNS = 3                         # left, straight, right: route = 3 * entry + turn


def set_route_at_intersection(st, _to):
    """-> a new IntersectionLiteState: `st` (left untouched) with every present slot k >= 1 still on its approach
    (s_k < 40) on the turn `_to` of its own entry.  `_to`: an integer (mod 3, as upstream's `_to % len(...)`) or
    "random": in ascending slot order, h = ((t * 16 + k) * 2654435761 + spawn_seq * 40503) mod 2^32,
    turn = (h >> 16) mod 3.  Anything else raises ValueError."""
    if isinstance(_to, str) and _to == "random":
        turn = None
    elif isinstance(_to, (int, np.integer)) and not isinstance(_to, (bool, np.bool_)):
        turn = int(_to) % N_TURNS
    else:
        raise ValueError("set_route_at_intersection takes an integer turn or \"random\", got %r" % (_to,))
    out = st.copy()
    for k in range(1, V_SLOTS):
        if not (int(out.flags[k]) & 1) or not (out.s[k] < APPROACH):
            continue
        if turn is None:
            h = ((int(out.t) * 16 + k) * 2654435761 + int(out.spawn_seq) * 40503) & 0xffffffff
            k_turn = (h >> 16) % N_TURNS
        else:
            k_turn = turn
        out.route[k] = N_TURNS * (int(out.route[k]) // N_TURNS) + k_turn
    return out


class IntersectionLiteRoutes(IntersectionLite):
    """IntersectionLite with `set_route_at_intersection(_to)`: returns a planning copy (the receiver is unchanged, as
    upstream returns `env_copy`)."""

    def set_route_at_intersection(self, _to):
        return IntersectionLiteRoutes(set_route_at_intersection(self.state, _to))

    def __deepcopy__(self, memo):
        return IntersectionLiteRoutes(self.state.copy())
