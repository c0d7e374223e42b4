// error plumbing + library-level C ABI
#include "common.cuh"

namespace rqb {
static thread_local std::string g_err;
thread_local int64_t g_launches = 0;
void set_error(const std::string& msg) { g_err = msg; }
int fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}
}  // namespace rqb

extern "C" {
const char* rqb200_last_error(void) { return rqb::g_err.c_str(); }
int rqb200_version(void) { return 118; }
int rqb200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
}
