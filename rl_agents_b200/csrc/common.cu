#include <stdarg.h>

#include "common.cuh"

namespace b2 {
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int sm_count() {
    int dev = 0, n = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
}

int check_env_kind(int env_kind, int n_actions) {
    if (env_kind == B2_ENV_FINITE) return B2_OK;
    if (env_kind != B2_ENV_HIGHWAY) {
        set_error("unknown env_kind %d", env_kind);
        return B2_ERR_INVALID;
    }
    B2_REQUIRE(n_actions == B2_HW_ACTIONS, "HighwayLite has 5 actions");
    return B2_OK;
}

int check_lane_env(int env_kind, int n_actions, const b2_finite_mdp& mdp) {
    if (env_kind == B2_ENV_FINITE) {
        B2_REQUIRE(mdp.transition && mdp.reward && mdp.terminal, "finite MDP tables missing");
        B2_REQUIRE(mdp.n_actions == n_actions, "mdp.n_actions != n_actions");
    }
    return check_env_kind(env_kind, n_actions);
}

int check_lane_env_il(int env_kind, int n_actions, const b2_finite_mdp& mdp) {
    if (env_kind == B2_ENV_INTERSECTION) {
        B2_REQUIRE(n_actions == B2_IL_ACTIONS, "IntersectionLite has 3 actions");
        return B2_OK;
    }
    return check_lane_env(env_kind, n_actions, mdp);
}

int check_sampled_mdp(const b2_finite_mdp_sampled& mdp, int n_actions, const uint8_t* terminal, bool needs_terminal) {
    B2_REQUIRE(mdp.cdf && mdp.next && mdp.reward && mdp.row_ok && (terminal || !needs_terminal),
               "finite MDP tables missing");
    B2_REQUIRE(mdp.n_actions == n_actions && mdp.n_states > 0 && mdp.n_next >= 1, "bad finite MDP shape");
    return B2_OK;
}

int check_sampled_entry(int env_kind, const b2_finite_mdp_sampled& mdp, int n_actions, const uint8_t* terminal,
                        int32_t env_draws) {
    B2_REQUIRE(env_kind == B2_ENV_FINITE, "env_kind must be B2_ENV_FINITE");
    if (check_sampled_mdp(mdp, n_actions, terminal, true) != B2_OK) return B2_ERR_INVALID;
    B2_REQUIRE(env_draws == 0 || env_draws == 1, "env_draws must be 0 or 1");
    return B2_OK;
}
}  // namespace b2

extern "C" const char* b2_last_error(void) { return b2::g_err; }
extern "C" int b2_version(void) { return 100; }

extern "C" int b2_device_info(int* sms, int* cc_major, int* cc_minor, char* name, int name_len) {
    int dev = 0;
    B2_CUDA_CHECK(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    B2_CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
    if (sms) *sms = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    if (name && name_len > 0) {
        strncpy(name, prop.name, name_len - 1);
        name[name_len - 1] = 0;
    }
    return B2_OK;
}
