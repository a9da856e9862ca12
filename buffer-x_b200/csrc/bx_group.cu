// bx_group.cu -- channel-first gathers of the pointnet2 layouts (pointnet2_ops gather_operation / grouping_operation).
//
// out[b][c][k] = features[b][c][idx[b][k]] over features [B,C,N] and int32 idx [B,K]: gather_operation is K = M,
// grouping_operation is idx [B,M,S] read as K = M*S (its output [B,C,M,S] is the same memory).  An index outside [0,N)
// yields NaN instead of a read outside the cloud.  One thread per output element; consecutive threads take consecutive k,
// so the stores and the index reads coalesce.
#include "bx_common.cuh"

namespace {

__global__ void gather_channels_kernel(const float *__restrict__ features, int C, int N, const int *__restrict__ idx, int K,
                                       size_t total, float *__restrict__ out) {
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const size_t k = e % K, bc = e / K, b = bc / C;
    const int i = idx[b * K + k];
    out[e] = (i >= 0 && i < N) ? features[bc * N + i] : __int_as_float(0x7fc00000);
}

}  // namespace

BX_API int bx_gather_channels(const float *features, int B, int C, int N, const int32_t *idx, int K, float *out, void *stream) {
    BX_REQUIRE(B >= 0 && C >= 0 && N >= 0 && K >= 0, "bx_gather_channels: negative size");
    const size_t total = (size_t)B * C * K;
    if (total == 0) return BX_OK;
    BX_REQUIRE(features && idx && out, "bx_gather_channels: null pointer");
    gather_channels_kernel<<<(unsigned)((total + 255) / 256), 256, 0, bx_stream(stream)>>>(features, C, N, idx, K, total, out);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
