// bx_svd.cu -- batched 3x3 singular value decomposition (torch_batch_svd.svd, utils/common.py:715 cal_Z_axis).
//
// One thread per matrix, everything in fp64 registers: the one-sided Jacobi of bx_svd3.cuh (U and V orthonormal for every
// input: rank deficient, zero, isotropic or with a negative determinant; A not assumed symmetric; signs of singular vectors
// unspecified, as in cuSOLVER).  fp32 in, fp32 out: A = U diag(S) V^T.
#include "bx_common.cuh"
#include "bx_svd3.cuh"

namespace {

__global__ void svd3_kernel(const float *__restrict__ A, int B, float *__restrict__ U, float *__restrict__ S,
                            float *__restrict__ V) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= B) return;
    double w[3][3], v[3][3], sv[3], u[3][3];   // w[j] = column j of A
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int r = 0; r < 3; ++r) w[j][r] = (double)A[(size_t)m * 9 + 3 * r + j];
    bx_svd3_fp64(w, u, sv, v);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        S[(size_t)m * 3 + j] = (float)sv[j];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            U[(size_t)m * 9 + 3 * r + j] = (float)u[j][r];
            V[(size_t)m * 9 + 3 * r + j] = (float)v[j][r];
        }
    }
}

}  // namespace

BX_API int bx_svd3(const float *A, int B, float *U, float *S, float *V, void *stream) {
    BX_REQUIRE(B >= 0, "bx_svd3: B=%d < 0", B);
    if (B == 0) return BX_OK;
    BX_REQUIRE(A && U && S && V, "bx_svd3: null pointer");
    svd3_kernel<<<(B + 127) / 128, 128, 0, bx_stream(stream)>>>(A, B, U, S, V);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
