// bx_splits.cuh -- the fixed-order split reductions of the training kernels (bx_train_step.cu, bx_train_desc.cu).
// A reduction over samples x positions writes BX_TS_SPLITS per-block partials (each block sums with block_sum), then
// sum_splits_kernel adds them in split order, one thread per output: no floating-point atomics, bit-identical across runs.
#pragma once
#include "bx_common.cuh"

namespace {

constexpr int TS_THREADS = 256;   // threads of every block that reduces with block_sum

// in-block fixed-order tree reduction of NV doubles per thread; thread 0 ends with the block totals in sh[i * TS_THREADS]
template <int NV>
__device__ __forceinline__ void block_sum(double (&v)[NV], double *sh) {
    const int t = threadIdx.x;
#pragma unroll
    for (int i = 0; i < NV; ++i) sh[i * TS_THREADS + t] = v[i];
    __syncthreads();
    for (int s = TS_THREADS / 2; s > 0; s >>= 1) {
        if (t < s) {
#pragma unroll
            for (int i = 0; i < NV; ++i) sh[i * TS_THREADS + t] += sh[i * TS_THREADS + t + s];
        }
        __syncthreads();
    }
}

// out[l] = sum over splits of partial[split][l], in split order
__global__ void sum_splits_kernel(const double *__restrict__ partial, int nsplit, long long L, double *__restrict__ out) {
    const long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= L) return;
    double s = 0.0;
    for (int i = 0; i < nsplit; ++i) s += partial[(size_t)i * L + l];
    out[l] = s;
}

inline int blocks_for(long long n, int t) { return (int)((n + t - 1) / t); }

}  // namespace
