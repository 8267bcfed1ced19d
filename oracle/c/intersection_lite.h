/* IntersectionLite in plain C -- TEST INFRASTRUCTURE (oracle/), not product code.
 * Third statement of docs/INTERSECTION_LITE_SPEC.md (after oracle/intersection.py in numpy and
 * rl_agents_b200/csrc/intersection_lite.cuh in CUDA), in the numpy statement's operation order; literal
 * O(V^2) scans, scalar fp32, compiled with -ffp-contract=off. */
#ifndef B2_ORACLE_INTERSECTION_LITE_H
#define B2_ORACLE_INTERSECTION_LITE_H
#include <stdint.h>

#define IL_V 16
#define IL_WORDS 136

typedef struct {
    float s[IL_V], v[IL_V];
    int32_t route[IL_V], flags[IL_V];
    int32_t pad[64];
    int32_t t, si, spawn_clock, spawn_seq, arrived, pad2[3];
} il_state;   /* exactly the 136-word layout */

int il_available_actions(const il_state* s, int* actions);   /* IDLE, FASTER, SLOWER order; returns the count */
/* one decision step in place; returns the reward; *flags: bit0 terminated, bit1 truncated */
float il_step(il_state* s, int action, int* flags);
void il_step_batch(int32_t* words, const int32_t* actions, float* rewards, int32_t* flags, int n);
#endif
