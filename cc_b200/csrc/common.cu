// common.cu - error plumbing of the C ABI (include/ccb200.h).
#include "ccb_common.cuh"
#include <cstdarg>
#include <cstdlib>

namespace ccb {

static thread_local char g_err[512] = "";
long long g_launches = 0;
thread_local const char* g_last_conv = "";

int pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("CCB_PDL");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v;
}

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: CUDA error: %s", what, cudaGetErrorString(e));
        return CCB_ERR_LAUNCH;
    }
    return CCB_OK;
}

}  // namespace ccb

extern "C" const char* ccb_last_error_string(void) { return ccb::g_err; }
extern "C" int ccb_version(void) { return 101; }
extern "C" const char* ccb_debug_last_conv_kernel(void) { return ccb::g_last_conv; }
extern "C" long long ccb_launch_count(void) { return ccb::g_launches; }
extern "C" int ccb_is_simulator(void) {
#ifdef CCB_CPU_SIM
    return 1;
#else
    return 0;
#endif
}
