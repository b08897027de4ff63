// abi.cu -- error reporting, launch counter, device facts.
#include "common.cuh"

namespace qk {
static thread_local std::string g_err;
std::atomic<int64_t> g_launches{0};

void set_err(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
}
int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;      // H100 SXM
    if (!cached[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}
const char* last_err() { return g_err.c_str(); }
}  // namespace qk

extern "C" {
const char* qk_last_error(void) { return qk::last_err(); }
int qk_version(void) { return QK_VERSION; }
int64_t qk_launch_count(void) { return qk::g_launches.load(); }
int qk_sm_count(void) { return qk::sm_count(); }
}
