// bx_common.cuh -- shared helpers of the bufferx_b200 CUDA library (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/bufferx_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "bufferx_b200 is written for sm_90a (H100)"
#endif

#define BX_API extern "C" __attribute__((visibility("default")))

void bx_set_error(const char *fmt, ...);
extern unsigned long long g_bx_launches;  // kernels launched by this library since load (host-side count)

#define BX_REQUIRE(cond, ...)            \
    do {                                 \
        if (!(cond)) {                   \
            bx_set_error(__VA_ARGS__);   \
            return BX_ERR_INVALID_ARG;   \
        }                                \
    } while (0)

#define BX_CUDA(expr)                                                                          \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            bx_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return BX_ERR_CUDA;                                                                \
        }                                                                                      \
    } while (0)

#define BX_LAUNCH_CHECK()                                                                      \
    do {                                                                                       \
        ++g_bx_launches;                                                                       \
        cudaError_t _e = cudaGetLastError();                                                   \
        if (_e != cudaSuccess) {                                                               \
            bx_set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
            return BX_ERR_CUDA;                                                                \
        }                                                                                      \
    } while (0)

static inline cudaStream_t bx_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) and the SM count are PER-DEVICE: one flag / value per device ordinal,
// so a process that drives several GPUs configures each of them (a plain `static bool` configured only the first).
constexpr int BX_MAX_DEVICES = 64;
struct BxPerDevice {
    size_t v[BX_MAX_DEVICES];   // 0 = not configured yet on that device; otherwise the configured value
};
// true when `want` exceeds what this device has been configured with (and records it)
static inline bool bx_needs_attr(BxPerDevice &f, size_t want = 1) {
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= BX_MAX_DEVICES) return true;
    if (f.v[d] >= want) return false;
    f.v[d] = want;
    return true;
}

#define BX_FULL 0xffffffffu

__device__ __forceinline__ int bx_lane() { return threadIdx.x & 31; }

// squared distance with the frozen evaluation order ((dx*dx)+(dy*dy))+(dz*dz); the translation
// units that use it are compiled with -fmad=false so no FMA contraction can happen.
__device__ __forceinline__ float bx_d2(float dx, float dy, float dz) { return ((dx * dx) + (dy * dy)) + (dz * dz); }

// exclusive block scan of one int per thread (blockDim.x <= 1024, multiple of 32); returns the
// exclusive prefix, *total gets the block total.  `sh` needs 33 ints.
__device__ __forceinline__ int bx_block_exscan(int v, int *sh, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(BX_FULL, inc, o);
        if (lane >= o) inc += n;
    }
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int w = lane < nw ? sh[lane] : 0;
        int winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int n = __shfl_up_sync(BX_FULL, winc, o);
            if (lane >= o) winc += n;
        }
        sh[lane] = winc - w;             // exclusive warp offsets
        if (lane == 31) sh[32] = winc;   // total
    }
    __syncthreads();
    const int res = sh[warp] + inc - v;
    *total = sh[32];
    __syncthreads();
    return res;
}
