/* HighwayLite in plain C -- TEST INFRASTRUCTURE (oracle/), not product code.
 * Third statement of docs/HIGHWAY_LITE_SPEC.md (after oracle/envs.py in numpy and
 * rl_agents_b200/csrc/highway_lite.cuh in CUDA); literal O(V^2) scans, scalar fp32, compiled
 * with -ffp-contract=off so that every operation is a single IEEE binary32 operation. */
#ifndef B2_ORACLE_HIGHWAY_LITE_H
#define B2_ORACLE_HIGHWAY_LITE_H
#include <stdint.h>

#define HL_V 16
#define HL_WORDS 136
#define HL_LANES 4

typedef struct {
    float x[HL_V], y[HL_V], h[HL_V], v[HL_V], ts[HL_V], timer[HL_V];
    int32_t tgt[HL_V], flags[HL_V];
    int32_t t, si, pad[6];
} hl_state;   /* exactly the 136-word layout */

int hl_available_actions(const hl_state* s, int* actions);   /* children order; returns the count */
/* one decision step in place; returns the reward; *flags: bit0 terminated, bit1 truncated */
float hl_step(hl_state* s, int action, int* flags);

/* shared with the IntersectionLite statement (intersection_lite.c): the spec's polynomials sin_p / cos_p and
 * not_zero, whose constants hl_init builds once (every exported entry point calls it) */
void hl_init(void);
float sin_p(float x);
float cos_p(float x);
float not_zero(float x);
#endif
