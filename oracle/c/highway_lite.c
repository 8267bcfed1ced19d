/* See highway_lite.h.  Follows docs/HIGHWAY_LITE_SPEC.md section by section. */
#include "highway_lite.h"

#include <math.h>
#include <string.h>

static const float LANE_W = 4.0f, LENGTH = 5.0f, WIDTH = 2.0f, HALF_LENGTH = 2.5f;
static const float MAX_SPEED = 40.0f, SPEED_LIMIT = 30.0f, ACC_MAX = 6.0f, COMFORT_ACC_MAX = 3.0f;
static const float D0 = 10.0f, TAU = 1.5f, LANE_CHANGE_DELAY = 1.0f, MOBIL_MAX_BRAKING = -2.0f;
static const float ON_LANE_MARGIN = 3.0f, SPEED_LO = 20.0f, SPEED_RANGE = 10.0f;
#define HL_SUBSTEPS 15
#define HL_DURATION 40

/* constants that are results of fp32 expressions or decimal literals: built once, in fp32 */
static float DT, KP_A, KP_HEADING, KP_LATERAL, PI_F, TWO_PI, HALF_PI, QUARTER_PI_SIN, S_BETA_MAX, TWO_SQRT_AB,
    MOBIL_MIN_GAIN, EPS, LAT_DEADBAND, HEADING_DEADBAND;
static float ASIN_C[10], SIN_C[5], COS_C[6];
static int g_init = 0;

void hl_init(void) {
    if (g_init) return;
    volatile float one = 1.0f;
    DT = one / 15.0f;
    KP_A = one / 0.6f;
    KP_HEADING = one / 0.2f;
    KP_LATERAL = one / 0.6f;
    PI_F = (float)3.141592653589793;
    TWO_PI = 2.0f * PI_F;
    HALF_PI = (float)(3.141592653589793 / 2);
    QUARTER_PI_SIN = (float)0.70710678;
    S_BETA_MAX = (float)0.65465367;
    TWO_SQRT_AB = 2.0f * sqrtf(15.0f);
    MOBIL_MIN_GAIN = (float)0.2;
    EPS = (float)0.01;
    LAT_DEADBAND = (float)1e-9;
    HEADING_DEADBAND = (float)1e-12;
    const double a[10] = {0.16666667, 0.075, 0.044642857, 0.030381944, 0.022372159,
                          0.017352764, 0.01396484, 0.011551816, 0.0097616, 0.0083903};
    const double sn[5] = {-1.0 / 6, 1.0 / 120, -1.0 / 5040, 1.0 / 362880, -1.0 / 39916800};
    const double cs[6] = {-0.5, 1.0 / 24, -1.0 / 720, 1.0 / 40320, -1.0 / 3628800, 1.0 / 479001600};
    for (int i = 0; i < 10; ++i) ASIN_C[i] = (float)a[i];
    for (int i = 0; i < 5; ++i) SIN_C[i] = (float)sn[i];
    for (int i = 0; i < 6; ++i) COS_C[i] = (float)cs[i];
    g_init = 1;
}

static float poly(float z, const float* c, int n) {
    float acc = c[n - 1];
    for (int i = n - 2; i >= 0; --i) acc = c[i] + z * acc;
    return acc;
}
static float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
static float asin_p(float u) { const float z = u * u; return u * (1.0f + z * poly(z, ASIN_C, 10)); }
float sin_p(float x) { x = clampf(x, -HALF_PI, HALF_PI); const float z = x * x; return x * (1.0f + z * poly(z, SIN_C, 5)); }
float cos_p(float x) { x = clampf(x, -HALF_PI, HALF_PI); const float z = x * x; return 1.0f + z * poly(z, COS_C, 6); }
float not_zero(float x) { return fabsf(x) > EPS ? x : (x >= 0.0f ? EPS : -EPS); }
static int lane_of(float y) { return (int)clampf(rintf(y / LANE_W), 0.0f, (float)(HL_LANES - 1)); }

static float idm(float v, float ts, int has_front, float x, float xf, float vf) {
    const float tsc = clampf(ts, 0.0f, SPEED_LIMIT);
    const float ratio = fmaxf(v, 0.0f) / fabsf(not_zero(tsc));
    const float r2 = ratio * ratio, r4 = r2 * r2;
    float acc = COMFORT_ACC_MAX * (1.0f - r4);
    if (has_front) {
        const float d = xf - x;
        const float gap = (D0 + v * TAU) + (v * (v - vf)) / TWO_SQRT_AB;
        const float q = gap / not_zero(d);
        acc = acc - COMFORT_ACC_MAX * (q * q);
    }
    return acc;
}

/* front / rear of vehicle i on the lane centred at lane_y (spec section 4, tie rules by index) */
static void neighbours(const hl_state* s, int i, float lane_y, int* front, int* rear) {
    *front = -1;
    *rear = -1;
    for (int j = 0; j < HL_V; ++j) {
        if (j == i || !(s->flags[j] & 1)) continue;
        if (!(fabsf(s->y[j] - lane_y) <= ON_LANE_MARGIN)) continue;
        if (s->x[j] >= s->x[i]) {
            if (*front < 0 || s->x[j] <= s->x[*front]) *front = j;
        } else {
            if (*rear < 0 || s->x[j] > s->x[*rear]) *rear = j;
        }
    }
}

int hl_available_actions(const hl_state* s, int* actions) {
    const int cur = lane_of(s->y[0]);
    int n = 0;
    actions[n++] = 1;
    if (cur > 0) actions[n++] = 0;
    if (cur < HL_LANES - 1) actions[n++] = 2;
    if (s->si < 2) actions[n++] = 3;
    if (s->si > 0) actions[n++] = 4;
    return n;
}

float hl_step(hl_state* s, int action, int* flags_out) {
    hl_init();
    if (action == 3 || action == 4) {
        int k = (int)clampf(rintf(((s->v[0] - SPEED_LO) / SPEED_RANGE) * 2.0f), 0.0f, 2.0f);
        k = action == 3 ? k + 1 : k - 1;
        k = k < 0 ? 0 : (k > 2 ? 2 : k);
        s->si = k;
        s->ts[0] = 20.0f + 5.0f * (float)k;
    } else if (action == 0) {
        s->tgt[0] = s->tgt[0] - 1 < 0 ? 0 : s->tgt[0] - 1;
    } else if (action == 2) {
        s->tgt[0] = s->tgt[0] + 1 > HL_LANES - 1 ? HL_LANES - 1 : s->tgt[0] + 1;
    }
    for (int sub = 0; sub < HL_SUBSTEPS; ++sub) {
        hl_state n = *s;   /* synchronous update: decisions read s, results go to n */
        for (int i = 0; i < HL_V; ++i) {
            if (!(s->flags[i] & 1)) continue;
            const int crashed = (s->flags[i] & 2) != 0, is_idm = i > 0;
            const int cur = lane_of(s->y[i]);
            const float cur_y = (float)cur * LANE_W;
            int tgt = s->tgt[i];
            float timer = s->timer[i];
            const int active = !crashed && is_idm;
            int f0, r0;
            neighbours(s, i, cur_y, &f0, &r0);
            const float self_a = idm(s->v[i], s->ts[i], f0 >= 0, s->x[i], f0 >= 0 ? s->x[f0] : 0.0f, f0 >= 0 ? s->v[f0] : 0.0f);
            if (active && cur != tgt) {              /* abort rule */
                for (int j = 0; j < HL_V; ++j) {
                    if (j == i || !(s->flags[j] & 1)) continue;
                    const float d = s->x[j] - s->x[i];
                    const float gap = (D0 + s->v[i] * TAU) + (s->v[i] * (s->v[i] - s->v[j])) / TWO_SQRT_AB;
                    if (lane_of(s->y[j]) != s->tgt[i] && s->tgt[j] == s->tgt[i] && d > 0.0f && d < gap) {
                        tgt = cur;
                        break;
                    }
                }
            } else if (active && timer > LANE_CHANGE_DELAY) {   /* MOBIL */
                timer = 0.0f;
                for (int side = -1; side <= 1; side += 2) {
                    const int lane = cur + side;
                    if (lane < 0 || lane >= HL_LANES || !(fabsf(s->v[i]) >= 1.0f)) continue;
                    int f, r;
                    neighbours(s, i, (float)lane * LANE_W, &f, &r);
                    const float foll = r >= 0 ? idm(s->v[r], s->ts[r], 1, s->x[r], s->x[i], s->v[i]) : 0.0f;
                    const float pred = idm(s->v[i], s->ts[i], f >= 0, s->x[i], f >= 0 ? s->x[f] : 0.0f, f >= 0 ? s->v[f] : 0.0f);
                    const float jerk = pred - self_a;
                    if (!(foll < MOBIL_MAX_BRAKING) && !(jerk < MOBIL_MIN_GAIN)) tgt = lane;
                }
            }
            /* steering */
            float lat = s->y[i] - (float)tgt * LANE_W;
            if (fabsf(lat) < LAT_DEADBAND) lat = 0.0f;
            const float lat_speed_cmd = -(KP_LATERAL * lat);
            const float nzv = not_zero(s->v[i]);
            const float u = clampf(lat_speed_cmd / nzv, -QUARTER_PI_SIN, QUARTER_PI_SIN);
            float dh = asin_p(u) - s->h[i];
            if (dh > PI_F) dh = dh - TWO_PI;
            if (dh < -PI_F) dh = dh + TWO_PI;
            if (fabsf(dh) < HEADING_DEADBAND) dh = 0.0f;
            const float rate = KP_HEADING * dh;
            float sb = clampf((HALF_LENGTH / nzv) * rate, -S_BETA_MAX, S_BETA_MAX);
            /* acceleration */
            float acc = self_a;
            if (cur != tgt) {
                int ft, rt;
                neighbours(s, i, (float)tgt * LANE_W, &ft, &rt);
                acc = fminf(acc, idm(s->v[i], s->ts[i], ft >= 0, s->x[i], ft >= 0 ? s->x[ft] : 0.0f, ft >= 0 ? s->v[ft] : 0.0f));
            }
            acc = clampf(acc, -ACC_MAX, ACC_MAX);
            if (i == 0) acc = KP_A * (s->ts[0] - s->v[0]);
            /* kinematics */
            if (crashed) { sb = 0.0f; acc = -s->v[i]; }
            if (s->v[i] > MAX_SPEED) acc = fminf(acc, MAX_SPEED - s->v[i]);
            if (s->v[i] < -MAX_SPEED) acc = fmaxf(acc, -MAX_SPEED - s->v[i]);
            const float cb = sqrtf(1.0f - sb * sb), sh = sin_p(s->h[i]), ch = cos_p(s->h[i]);
            const float c_hb = ch * cb - sh * sb, s_hb = sh * cb + ch * sb;
            n.x[i] = s->x[i] + (s->v[i] * c_hb) * DT;
            n.y[i] = s->y[i] + (s->v[i] * s_hb) * DT;
            n.h[i] = s->h[i] + ((s->v[i] * sb) / HALF_LENGTH) * DT;
            n.v[i] = s->v[i] + acc * DT;
            n.timer[i] = is_idm ? timer + DT : timer;
            n.tgt[i] = tgt;
        }
        /* collisions on the new positions */
        for (int i = 0; i < HL_V; ++i)
            for (int j = 0; j < HL_V; ++j)
                if (i != j && (n.flags[i] & 1) && (n.flags[j] & 1) && fabsf(n.x[i] - n.x[j]) < LENGTH &&
                    fabsf(n.y[i] - n.y[j]) < WIDTH)
                    n.flags[i] |= 2;
        *s = n;
    }
    const int crashed0 = (s->flags[0] & 2) != 0;
    const float lane_r = (float)s->tgt[0] / (float)(HL_LANES - 1);
    const float fs = s->v[0] * cos_p(s->h[0]);
    const float sc = clampf((fs - SPEED_LO) / SPEED_RANGE, 0.0f, 1.0f);
    float r = (crashed0 ? -1.0f : 0.0f) + 0.1f * lane_r;
    r = r + 0.4f * sc;
    r = (r + 1.0f) / 1.5f;
    if (!(s->y[0] >= -2.0f && s->y[0] <= 14.0f)) r = 0.0f;
    s->t += 1;
    *flags_out = (crashed0 ? 1 : 0) | (s->t >= HL_DURATION ? 2 : 0);
    return r;
}

/* ---------------------------------------------------------------------------------------------------------------
 * ValueIterationAgent on a HighwayLite scene (docs/HIGHWAY_LITE_SPEC.md section 9): the time-to-collision grid MDP of
 * `env.unwrapped.to_finite_mdp()` and the reference agent's fixed point on it
 * (rl_agents/agents/dynamic_programming/value_iteration.py:17,29-35,42-73).  Third statement, after
 * oracle/envs.py::highway_finite_mdp (+ oracle/planners.py::value_iteration) and rl_agents_b200/csrc/ttc_vi.cu; explicit
 * tables, literal loops.  TEST INFRASTRUCTURE.
 * ------------------------------------------------------------------------------------------------------------- */
#define TTC_H 3
#define TTC_T 10
enum { A_LEFT = 0, A_IDLE = 1, A_RIGHT = 2, A_FASTER = 3, A_SLOWER = 4 };
#define TTC_S (TTC_H * HL_LANES * TTC_T)
#define TTC_A 5

static int ttc_clip(int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); }
static int ttc_cell(int h, int i, int j) { return (ttc_clip(h, TTC_H - 1) * HL_LANES + ttc_clip(i, HL_LANES - 1)) * TTC_T + ttc_clip(j, TTC_T - 1); }
static int ttc_lane(float y) { return ttc_clip((int)rintf(y / 4.0f), HL_LANES - 1); }

/* grid [3][4][10] of costs 0 / 0.5 / 1 */
void hl_ttc_grid(const hl_state* s, double* grid) {
    hl_init();
    for (int c = 0; c < TTC_S; ++c) grid[c] = 0.0;
    const double margin = (double)LENGTH / 2 + (double)LENGTH / 2;
    const double points[3][2] = {{0.0, 1.0}, {-margin, 0.5}, {margin, 0.5}};
    for (int h = 0; h < TTC_H; ++h) {
        const double ego_speed = 20.0 + 5.0 * h;
        for (int k = 1; k < HL_V; ++k) {
            if (!(s->flags[k] & 1)) continue;
            if (ego_speed == (double)s->v[k]) continue;
            const float dh = s->h[k] - s->h[0];
            const double projected = (double)s->v[k] * (double)cos_p(dh);
            const double diff = ego_speed - projected;
            const double nz = fabs(diff) > 0.01 ? diff : (diff >= 0 ? 0.01 : -0.01);
            const int lane = ttc_lane(s->y[k]);
            for (int p = 0; p < 3; ++p) {
                const double distance = ((double)s->x[k] - (double)s->x[0]) + points[p][0];
                const double ttc = distance / nz;
                if (ttc < 0) continue;
                const double tq[2] = {floor(ttc), ceil(ttc)};        /* int(ttc), int(ceil(ttc)) for ttc >= 0 */
                for (int q = 0; q < 2; ++q) {
                    if (tq[q] >= 0 && tq[q] < TTC_T) {
                        double* g = &grid[(h * HL_LANES + lane) * TTC_T + (int)tq[q]];
                        if (points[p][1] > *g) *g = points[p][1];
                    }
                }
            }
        }
    }
}

/* q_out [120][5]; returns the number of sweeps; *state = mdp.state, *action = argmax_a Q[state] */
int hl_ttc_value_iteration(const int32_t* words, double gamma, int iterations, double rtol, double atol, double* q_out,
                           int32_t* state, int32_t* action) {
    const hl_state* s = (const hl_state*)words;
    static double grid[TTC_S], reward[TTC_S][TTC_A], q[TTC_S][TTC_A], nq[TTC_S][TTC_A], v[TTC_S];
    static int transition[TTC_S][TTC_A], terminal[TTC_S];
    hl_ttc_grid(s, grid);
    const double action_reward[TTC_A] = {0.0, 0.0, 0.0, 0.0, 0.0};      /* lane_change_reward = 0 */
    for (int h = 0; h < TTC_H; ++h)
        for (int i = 0; i < HL_LANES; ++i)
            for (int j = 0; j < TTC_T; ++j) {
                const int c = (h * HL_LANES + i) * TTC_T + j;
                const double state_reward = (-1.0 * grid[c] + 0.1 * ((double)i / (HL_LANES - 1))) + 0.4 * ((double)h / (TTC_H - 1));
                terminal[c] = grid[c] == 1.0 || j == TTC_T - 1;
                for (int a = 0; a < TTC_A; ++a) {
                    int nh = h, ni = i;
                    if (a == A_LEFT) ni = i - 1;
                    else if (a == A_RIGHT) ni = i + 1;
                    else if (a == A_FASTER && j == 0) nh = h + 1;
                    else if (a == A_SLOWER && j == 0) nh = h - 1;
                    transition[c][a] = ttc_cell(nh, ni, j + 1);
                    reward[c][a] = state_reward + action_reward[a];
                    q[c][a] = 0.0;
                }
            }
    int sweeps = 0;
    for (int it = 0; it < iterations; ++it) {
        ++sweeps;
        for (int c = 0; c < TTC_S; ++c) {
            double m = q[c][0];
            for (int a = 1; a < TTC_A; ++a) m = q[c][a] > m ? q[c][a] : m;
            v[c] = m;
        }
        int close = 1;
        for (int c = 0; c < TTC_S; ++c)
            for (int a = 0; a < TTC_A; ++a) {
                const double next_v = terminal[c] ? 0.0 : v[transition[c][a]];
                nq[c][a] = reward[c][a] + gamma * next_v;
                if (!(fabs(q[c][a] - nq[c][a]) <= atol + rtol * fabs(nq[c][a]))) close = 0;
            }
        if (close) break;                               /* the previous iterate is returned (:71-72) */
        memcpy(q, nq, sizeof(q));
    }
    memcpy(q_out, q, sizeof(q));
    const int s0 = ttc_cell(s->si, ttc_lane(s->y[0]), 0);
    int best = 0;
    for (int a = 1; a < TTC_A; ++a)
        if (q[s0][a] > q[s0][best]) best = a;
    *state = s0;
    *action = best;
    return sweeps;
}

/* n scenes one after the other (the CPU data point beside b2_highway_ttc_vi) */
void hl_ttc_value_iteration_batch(const int32_t* words, int n, double gamma, int iterations, int32_t* actions) {
    static double q[TTC_S][TTC_A];
    int32_t st;
    for (int e = 0; e < n; ++e)
        hl_ttc_value_iteration(words + (int64_t)e * HL_WORDS, gamma, iterations, 1e-5, 1e-8, &q[0][0], &st, &actions[e]);
}
