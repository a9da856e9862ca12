// bx_api.cu -- library-level entry points (error string, version, device probe).
#include <stdarg.h>
#include <string.h>

#include "bx_common.cuh"

static thread_local char g_err[512] = "";
unsigned long long g_bx_launches = 0;

void bx_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

BX_API const char *bx_last_error(void) { return g_err; }

BX_API int bx_version(void) { return 200; }

BX_API unsigned long long bx_launch_count(void) { return g_bx_launches; }

BX_API int bx_device_sm_count(void) {
    static int cache[BX_MAX_DEVICES] = {};      // per device ordinal (0 = not queried yet)
    int dev = 0, n = 0;
    BX_CUDA(cudaGetDevice(&dev));
    if (dev >= 0 && dev < BX_MAX_DEVICES && cache[dev]) return cache[dev];
    BX_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    if (dev >= 0 && dev < BX_MAX_DEVICES) cache[dev] = n;
    return n;
}
