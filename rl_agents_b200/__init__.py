"""rl_agents_b200 -- H100-native batched tree-search and value-iteration engine
behind the rl-agents plugin surface (agent_factory / AbstractAgent / JSON
config).  Select it by pointing `__class__` in an agent JSON at e.g.

    "<class 'rl_agents_b200.agents.tree_search.deterministic.DeterministicPlannerAgent'>"

All planning runs in hand-written sm_90a CUDA (csrc/ -> libb2planner.so)
reached through the C ABI in include/b2_planner.h; there is no CPU fallback.
"""
__version__ = "0.1.0"
