// common.cpp -- thread-local error message + misc C-ABI entry points (hp_last_error, hp_version).
#include "common.h"
#include "../../include/hyperpose_b200.h"

namespace hpb {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* get_error() { return g_err; }
}

extern "C" {
const char* hp_last_error(void) { return hpb::get_error(); }
const char* hp_version(void) { return "hyperpose_b200 0.1 (sm_90a)"; }
int hp_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}
}
