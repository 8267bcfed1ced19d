/* See intersection_lite.h.  Follows docs/INTERSECTION_LITE_SPEC.md section by section, in the operation order of
 * oracle/intersection.py::intersection_step. */
#include "intersection_lite.h"

#include <math.h>
#include <string.h>

#include "highway_lite.h"   /* sin_p / cos_p / not_zero */

enum { IL_SLOWER = 0, IL_IDLE = 1, IL_FASTER = 2 };
#define IL_SUBSTEPS 15
#define IL_DURATION 13
#define IL_ROUTES 12
#define IL_SPAWN_PERIOD 23

static const float APPROACH = 40.0f, EXIT = 40.0f, BOX_STRAIGHT = 12.0f, LENGTH = 5.0f, HIT_D2 = 12.25f, ACC_MAX = 6.0f;
static const float OTHER_TS = 9.0f, STOP_LINE = 38.0f, YIELD_FROM = 15.0f, PRIO_FROM = 25.0f, PRIO_PAST = 4.0f;
static const float ENTRY_CLEAR = 14.0f, SPAWN_SPEED = 8.0f, SPEED_STEP = 4.5f;
/* HighwayLite's IDM parameters (docs/HIGHWAY_LITE_SPEC.md), which the spec reuses */
static const float SPEED_LIMIT = 30.0f, COMFORT_ACC_MAX = 3.0f, D0 = 10.0f, TAU = 1.5f;

/* constants that are results of fp32 expressions: built once, in fp32 */
static float DT, KP_A, PI_F, TWO_SQRT_AB, BOX[3], LEN[3];
static int g_init = 0;

static void il_init(void) {
    if (g_init) return;
    hl_init();
    volatile float one = 1.0f;
    DT = one / 15.0f;
    KP_A = one / 0.6f;
    PI_F = (float)3.141592653589793;
    TWO_SQRT_AB = 2.0f * sqrtf(15.0f);
    BOX[0] = 4.0f * PI_F;
    BOX[1] = BOX_STRAIGHT;
    BOX[2] = 2.0f * PI_F;
    for (int t = 0; t < 3; ++t) LEN[t] = (APPROACH + BOX[t]) + EXIT;
    g_init = 1;
}

static float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
/* floor division and modulo by 3, as numpy's // and % on the route words */
static int entry_of(int r) { return r >= 0 ? r / 3 : -((2 - r) / 3); }
static int turn_of(int r) { return r - 3 * entry_of(r); }

static void position(int route, float s, float* wx, float* wy) {
    const int turn = turn_of(route), entry = entry_of(route);
    float x = 2.0f, y = -46.0f + s;
    const float u = s - APPROACH;
    if (turn == 0 && s >= APPROACH) {          /* left: radius 8 about (-6, -6) */
        const float th = u * 0.125f;
        const float lx = -6.0f + 8.0f * cos_p(th), ly = -6.0f + 8.0f * sin_p(th);
        const float ul = u - BOX[0];
        const int past = u >= BOX[0];
        x = past ? -6.0f - ul : lx;
        y = past ? 2.0f : ly;
    } else if (turn == 2 && s >= APPROACH) {   /* right: radius 4 about (6, -6) */
        const float th = u * 0.25f;
        const float rx = 6.0f - 4.0f * cos_p(th), ry = -6.0f + 4.0f * sin_p(th);
        const float ur = u - BOX[2];
        const int past = u >= BOX[2];
        x = past ? 6.0f + ur : rx;
        y = past ? -2.0f : ry;
    }
    /* entries: S as is, W rotated clockwise, N by 180 degrees, E counter-clockwise */
    *wx = entry == 0 ? x : (entry == 1 ? y : (entry == 2 ? -x : -y));
    *wy = entry == 0 ? y : (entry == 1 ? -x : (entry == 2 ? -y : x));
}

static float idm(float v, int has_front, float d, float v_f) {
    const float ts = fminf(fmaxf(OTHER_TS, 0.0f), SPEED_LIMIT);
    const float ratio = fmaxf(v, 0.0f) / fabsf(not_zero(ts));
    const float r2 = ratio * ratio, r4 = r2 * r2;
    const float acc = COMFORT_ACC_MAX * (1.0f - r4);
    const float gap = (D0 + v * TAU) + (v * (v - v_f)) / TWO_SQRT_AB;
    const float q = gap / not_zero(d);
    return has_front ? acc - COMFORT_ACC_MAX * (q * q) : acc;
}

int il_available_actions(const il_state* s, int* actions) {
    int n = 0;
    actions[n++] = IL_IDLE;
    if (s->si < 2) actions[n++] = IL_FASTER;
    if (s->si > 0) actions[n++] = IL_SLOWER;
    return n;
}

float il_step(il_state* s, int action, int* flags_out) {
    il_init();
    if (action == IL_FASTER) s->si = s->si + 1 < 2 ? s->si + 1 : 2;
    else if (action == IL_SLOWER) s->si = s->si - 1 > 0 ? s->si - 1 : 0;
    const float ts0 = SPEED_STEP * (float)s->si;
    for (int sub = 0; sub < IL_SUBSTEPS; ++sub) {
        int present[IL_V], entry[IL_V], turn[IL_V];
        float acc[IL_V];
        for (int i = 0; i < IL_V; ++i) {
            present[i] = (s->flags[i] & 1) != 0;
            entry[i] = entry_of(s->route[i]);
            turn[i] = turn_of(s->route[i]);
        }
        /* front vehicle (same route, or same entry while it is still on the approach; smallest s, ties: smallest
         * slot), IDM, yield to priority traffic, clip, the ego's speed control, crashed vehicles */
        for (int i = 0; i < IL_V; ++i) {
            int front = -1;
            for (int j = 0; j < IL_V; ++j) {
                const int same_lane = s->route[j] == s->route[i] || (entry[j] == entry[i] && s->s[j] < APPROACH);
                if (present[j] && j != i && same_lane && s->s[j] > s->s[i] && (front < 0 || s->s[j] < s->s[front]))
                    front = j;
            }
            float a = idm(s->v[i], front >= 0, front >= 0 ? s->s[front] - s->s[i] : 0.0f, front >= 0 ? s->v[front] : 0.0f);
            int prio = 0;
            for (int j = 0; j < IL_V; ++j)
                if (present[j] && entry[j] != entry[i] && s->route[j] > s->route[i] && s->s[j] > PRIO_FROM &&
                    s->s[j] < (APPROACH + BOX[turn[j]]) + PRIO_PAST)
                    prio = 1;
            const int yields = s->s[i] > YIELD_FROM && s->s[i] < STOP_LINE && prio;
            const float a_y = idm(s->v[i], 1, STOP_LINE - s->s[i], 0.0f);
            if (yields) a = fminf(a, a_y);
            a = clampf(a, -ACC_MAX, ACC_MAX);
            if (i == 0) a = KP_A * (ts0 - s->v[0]);
            if (s->flags[i] & 2) a = -s->v[i];
            acc[i] = a;
        }
        /* integrate */
        for (int i = 0; i < IL_V; ++i) {
            if (!present[i]) continue;
            const float ns = s->s[i] + s->v[i] * DT;
            const float nv = fmaxf(s->v[i] + acc[i] * DT, 0.0f);
            s->s[i] = ns;
            s->v[i] = nv;
        }
        /* collisions on the new positions (presence as at the start of the sub-step) */
        float x[IL_V], y[IL_V];
        int hit[IL_V];
        for (int i = 0; i < IL_V; ++i) position(s->route[i], s->s[i], &x[i], &y[i]);
        for (int i = 0; i < IL_V; ++i) {
            hit[i] = 0;
            for (int j = 0; j < IL_V; ++j) {
                if (!(present[i] && present[j] && j != i)) continue;
                const int lane = s->route[j] == s->route[i] ||
                                 (entry[j] == entry[i] && s->s[j] < APPROACH && s->s[i] < APPROACH);
                const float dx = x[j] - x[i], dy = y[j] - y[i];
                const float d2 = dx * dx + dy * dy;
                if (lane ? fabsf(s->s[j] - s->s[i]) < LENGTH : d2 < HIT_D2) hit[i] = 1;
            }
        }
        for (int i = 0; i < IL_V; ++i)
            if (hit[i]) s->flags[i] |= 2;
        /* end of route: others leave, the ego has arrived */
        for (int i = 0; i < IL_V; ++i) {
            if (!(present[i] && s->s[i] >= LEN[turn[i]])) continue;
            if (i == 0) s->arrived = 1;
            else s->flags[i] = 0;
        }
        /* deterministic spawning */
        s->spawn_clock += 1;
        if (s->spawn_clock >= IL_SPAWN_PERIOD) {
            s->spawn_clock = 0;
            const uint32_t k = (uint32_t)s->spawn_seq;
            s->spawn_seq = (int32_t)((k + 1u) & 0x7fffffffu);
            const uint32_t h = k * 2654435761u + 40503u;
            const int route = (int)((h >> 16) % (uint32_t)IL_ROUTES);
            int clear = 1, slot = -1;
            for (int j = 0; j < IL_V; ++j)
                if ((s->flags[j] & 1) && entry_of(s->route[j]) == route / 3 && s->s[j] < ENTRY_CLEAR) clear = 0;
            for (int j = IL_V - 1; j >= 1; --j)
                if (!(s->flags[j] & 1)) slot = j;
            if (clear && slot > 0) {
                s->s[slot] = 0.0f;
                s->v[slot] = SPAWN_SPEED;
                s->route[slot] = route;
                s->flags[slot] = 1;
            }
        }
    }
    s->t += 1;
    const int crashed0 = (s->flags[0] & 2) != 0;
    float r;
    if (crashed0) {
        r = 0.0f;
    } else if (s->arrived) {
        r = 1.0f;
    } else {
        const float sc = clampf((s->v[0] - 7.0f) * 0.5f, 0.0f, 1.0f);
        r = (5.0f + sc) / 6.0f;
    }
    /* the words outside the layout are zero after a step, as the other statements write them */
    memset(s->pad, 0, sizeof(s->pad));
    memset(s->pad2, 0, sizeof(s->pad2));
    *flags_out = (crashed0 || s->arrived ? 1 : 0) | (s->t >= IL_DURATION ? 2 : 0);
    return r;
}

void il_step_batch(int32_t* words, const int32_t* actions, float* rewards, int32_t* flags, int n) {
    for (int i = 0; i < n; ++i) rewards[i] = il_step((il_state*)(words + (size_t)i * IL_WORDS), actions[i], &flags[i]);
}
