// bx_dp.cu -- the cross-rank mean of one sharded training step (driver.train_sharded, DESIGN.md §8).
//
// Every rank gathers the same [W, n+1] fp32 matrix of records (gradients, BatchNorm buffers, contribution flag) and
// runs this kernel on it, so every rank computes the same bits: each element is summed in float64 in ascending rank
// order over the contributing rows, divided once by their count and rounded once to fp32.  The additions and the
// division are spelled __dadd_rn / __ddiv_rn, and the unit is compiled with -fmad=false, so nothing is reordered or
// contracted.
#include "bx_common.cuh"

namespace {

constexpr int DP_THREADS = 256;
constexpr long long DP_MAX_BLOCKS = 4096;

__global__ void __launch_bounds__(DP_THREADS)
dp_mean_kernel(const float *__restrict__ g, int W, long long n, float *__restrict__ out, int32_t *__restrict__ count) {
    const long long stride = n + 1;
    int cnt = 0;
    for (int r = 0; r < W; ++r) cnt += g[(long long)r * stride + n] != 0.0f;
    if (blockIdx.x == 0 && threadIdx.x == 0) *count = cnt;
    if (cnt == 0) return;
    const double denom = (double)cnt;
    for (long long i = (long long)blockIdx.x * DP_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * DP_THREADS) {
        double s = 0.0;
        bool first = true;
        for (int r = 0; r < W; ++r) {
            const float *row = g + (long long)r * stride;
            if (row[n] == 0.0f) continue;
            const double v = (double)row[i];
            s = first ? v : __dadd_rn(s, v);      // start from the first contributor: one rank is the identity, -0 included
            first = false;
        }
        out[i] = __double2float_rn(__ddiv_rn(s, denom));
    }
}

}  // namespace

BX_API int bx_dp_mean(const float *gathered, int W, long long n, float *out, int32_t *count, void *stream) {
    BX_REQUIRE(gathered != nullptr && out != nullptr && count != nullptr, "bx_dp_mean: null pointer");
    BX_REQUIRE(W >= 1, "bx_dp_mean: W = %d, needs at least one rank", W);
    BX_REQUIRE(n >= 0, "bx_dp_mean: n = %lld must be >= 0", n);
    long long blocks = (n + DP_THREADS - 1) / DP_THREADS;
    blocks = blocks < 1 ? 1 : (blocks > DP_MAX_BLOCKS ? DP_MAX_BLOCKS : blocks);
    dp_mean_kernel<<<(unsigned)blocks, DP_THREADS, 0, bx_stream(stream)>>>(gathered, W, n, out, count);
    BX_LAUNCH_CHECK();
    return 0;
}
