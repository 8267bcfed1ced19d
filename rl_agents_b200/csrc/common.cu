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
