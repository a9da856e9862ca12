// bx_conv.cu -- a9 attention pooling and the factorised first CostNet layer.
//
// bx_pool_desc replaces pool_layer / avg-pool / F.normalize of the descriptor network (models/patch_embedder.py:32-39,
// 80-83): one CTA per patch turns the last Cylindrical_Net activation into the unit descriptor and the unit-normalised
// equivariant map.
// bx_costvol_ab computes the first CostNet layer (models/patchnet.py:196) over the cost volume of models/BUFFERX.py:51-65
// in factorised form: two small convolutions of the source / target equivariant maps, from which the next layer's loader
// regenerates the activation (the COSTAB loaders of bx_conv_tc.cu and bx_conv_sd.cu), so the cost volume is never
// materialised.  CUDA-core fp32 arithmetic with fp32 accumulation.
#include "bx_common.cuh"

namespace {

// ---- a9: attention pooling ------------------------------------------------------------------------
// one CTA per patch; thread = spatial position (S <= 160).
constexpr int POOL_T = 160;

__global__ void __launch_bounds__(POOL_T)
pool_desc_kernel(const float *__restrict__ x, int K, int C, int S, int channels_last, const float *__restrict__ w1,
                 const float *__restrict__ b1, const float *__restrict__ w2, const float *__restrict__ b2,
                 float *__restrict__ desc, float *__restrict__ equi, const int *__restrict__ d_K) {
    __shared__ float sw1[32 * 16], sb1[16], sw2[16], sb2;
    if (d_K && (int)blockIdx.x >= *d_K) return;            // beyond the device-side count: the whole CTA, before any barrier
    __shared__ float xw[32][POOL_T + 1];
    __shared__ float fsum[32];
    const int k = blockIdx.x, tid = threadIdx.x;
    for (int i = tid; i < 32 * 16; i += POOL_T) sw1[i] = w1[i];
    if (tid < 16) { sb1[tid] = b1[tid]; sw2[tid] = w2[tid]; }
    if (tid == 0) sb2 = b2[0];
    __syncthreads();
    const float *xp = x + (size_t)k * C * S;
    float xv[32];
    float att = 0.0f;
    if (tid < S) {
        float h[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) h[j] = sb1[j];
        float nrm = 0.0f;
        if (channels_last) {   // x: [K][32/4][S][4] (tensor-core conv output, channel-blocked)
            const float4 *x4 = reinterpret_cast<const float4 *>(xp) + tid;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 v = __ldg(x4 + (size_t)q * S);
                xv[4 * q] = v.x; xv[4 * q + 1] = v.y; xv[4 * q + 2] = v.z; xv[4 * q + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int c = 0; c < 32; ++c) xv[c] = xp[(size_t)c * S + tid];
        }
#pragma unroll
        for (int c = 0; c < 32; ++c) {
            nrm = fmaf(xv[c], xv[c], nrm);
#pragma unroll
            for (int j = 0; j < 16; ++j) h[j] = fmaf(xv[c], sw1[c * 16 + j], h[j]);
        }
        float a = sb2;
#pragma unroll
        for (int j = 0; j < 16; ++j) a = fmaf(fmaxf(h[j], 0.0f), sw2[j], a);
        att = fmaxf(a, 0.0f);
        const float inv = 1.0f / fmaxf(sqrtf(nrm), 1e-12f);
        float *ep = equi + (size_t)k * C * S;
#pragma unroll
        for (int c = 0; c < 32; ++c) ep[(size_t)c * S + tid] = xv[c] * inv;
    }
#pragma unroll
    for (int c = 0; c < 32; ++c) xw[c][tid] = (tid < S) ? xv[c] * att : 0.0f;
    __syncthreads();
    // per-channel mean over positions: warp w reduces channels w, w+5, ...
    const int lane = tid & 31, warp = tid >> 5;
    for (int c = warp; c < 32; c += POOL_T / 32) {
        float s = 0.0f;
        for (int i = lane; i < POOL_T; i += 32) s += xw[c][i];
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(BX_FULL, s, o);
        if (lane == 0) fsum[c] = s / (float)S;
    }
    __syncthreads();
    if (tid < 32) {
        float v = fsum[tid];
        float n2 = v * v;
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) n2 += __shfl_xor_sync(BX_FULL, n2, o);
        desc[(size_t)k * 32 + tid] = v / fmaxf(sqrtf(n2), 1e-12f);
    }
}

// ---- factorised first CostNet layer ---------------------------------------------------------------------
// The cost volume is V[c][n][k][l] = d1[c][1+k][(l-n) mod 20] - d2[c][1+k][l] (models/BUFFERX.py:51-65) and the first
// CostNet layer (patchnet.py:196, valid 3x3x3, BN folded, ReLU) is linear in it before the ReLU, so
//     out0[co][n][k][l] = relu( A[co][k][(l-n) mod 20] - B[co][k][l] )
//     A[co][k][m] = bias[co] + sum_{c,dk,e} Wa[c][dk][e][co] * d1[c][1+k+dk][(m+e-2) mod 20],  Wa[..e..] = sum_{dl-dn = e-2} w
//     B[co][k][l] =            sum_{c,dk,dl} Wb[c][dk][dl][co] * d2[c][1+k+dk][l+dl],           Wb       = sum_{dn} w
// : 60 + 54 output positions per match instead of 972 (27 MMAC -> 1.4 MMAC per match).  The next layer's loader
// (BX_GEOM_COSTAB) regenerates out0 from A and B, so neither the 256 KB cost volume nor the 124 KB first activation
// of a match is ever written.  One CTA per match; d1/d2 rows 1..5 staged in shared memory, weights through L1.
constexpr int AB_T = 512;            // two matches at a time, 256 threads each
constexpr int AB_WA = 32 * 3 * 5 * 32, AB_WB = 32 * 3 * 3 * 32;
constexpr int AB_SMEM = (AB_WA + AB_WB + 2 * 2 * 3200) * (int)sizeof(float);

// Persistent CTAs (one per SM): the 98 KB of factor weights stay in shared memory; every thread owns 8 output channels
// at two positions of one match (one weight fetch feeds 16 FMAs).  A and B are written channel-blocked
// ([32/4][positions][4]) so that the consumer (BX_GEOM_COSTAB loader) reads them with 16-byte loads.
__global__ void __launch_bounds__(AB_T, 1)
costvol_ab_kernel(const float *__restrict__ equi_s, const float *__restrict__ equi_t, const int *__restrict__ s_mids,
                  const int *__restrict__ t_mids, const int *__restrict__ d_M, const float *__restrict__ wa,
                  const float *__restrict__ wb, const float *__restrict__ bias, float *__restrict__ A, float *__restrict__ B) {
    extern __shared__ __align__(16) float ab_smem[];
    float *swa = ab_smem, *swb = swa + AB_WA, *sd = swb + AB_WB;   // sd: [half(2)][d1 | d2][32][100]
    const int M = *d_M;
    const int tid = threadIdx.x, half = tid >> 8, ht = tid & 255;
    if ((int)blockIdx.x * 2 >= M) return;
    for (int i = tid; i < AB_WA / 4; i += AB_T) reinterpret_cast<float4 *>(swa)[i] = __ldg(reinterpret_cast<const float4 *>(wa) + i);
    for (int i = tid; i < AB_WB / 4; i += AB_T) reinterpret_cast<float4 *>(swb)[i] = __ldg(reinterpret_cast<const float4 *>(wb) + i);
    float *d1 = sd + half * 6400, *d2 = d1 + 3200;
    for (int m0 = (int)blockIdx.x * 2; m0 < M; m0 += (int)gridDim.x * 2) {
        const int m = m0 + half;
        __syncthreads();                       // previous round's readers are done (also covers the weight fill)
        if (m < M) {
            const float *e1 = equi_s + (size_t)s_mids[m] * 32 * 140, *e2 = equi_t + (size_t)t_mids[m] * 32 * 140;
            for (int i = ht; i < 3200; i += 256) {
                const int c = i / 100, r = i - c * 100;
                d1[i] = __ldg(e1 + c * 140 + 20 + r);       // elevation rows 1..5
                d2[i] = __ldg(e2 + c * 140 + 20 + r);
            }
        }
        __syncthreads();
        if (m >= M) continue;
        float acc0[8], acc1[8];
        if (ht < 120) {                        // A: cg(4) x k(3) x mm(10): positions (k, mm) and (k, mm + 10)
            const int cg = ht / 30, r = ht - cg * 30, k = r / 10, mm = r - k * 10;
#pragma unroll
            for (int j = 0; j < 8; ++j) acc0[j] = acc1[j] = __ldg(bias + cg * 8 + j);
            int c0[5], c1[5];
#pragma unroll
            for (int e = 0; e < 5; ++e) {
                int x = mm + e - 2;
                c0[e] = x < 0 ? x + 20 : x;                 // mm + e - 2 in [-2, 11]
                x = mm + 10 + e - 2;
                c1[e] = x >= 20 ? x - 20 : x;               // in [8, 21]
            }
            for (int c = 0; c < 32; ++c) {
#pragma unroll
                for (int dk = 0; dk < 3; ++dk) {
                    const float *row = d1 + c * 100 + (k + dk) * 20;
                    const float4 *wp = reinterpret_cast<const float4 *>(swa + ((c * 3 + dk) * 5) * 32 + cg * 8);
#pragma unroll
                    for (int e = 0; e < 5; ++e) {
                        const float x0 = row[c0[e]], x1 = row[c1[e]];
                        const float4 w0 = wp[e * 8], w1 = wp[e * 8 + 1];
                        acc0[0] += x0 * w0.x; acc0[1] += x0 * w0.y; acc0[2] += x0 * w0.z; acc0[3] += x0 * w0.w;
                        acc0[4] += x0 * w1.x; acc0[5] += x0 * w1.y; acc0[6] += x0 * w1.z; acc0[7] += x0 * w1.w;
                        acc1[0] += x1 * w0.x; acc1[1] += x1 * w0.y; acc1[2] += x1 * w0.z; acc1[3] += x1 * w0.w;
                        acc1[4] += x1 * w1.x; acc1[5] += x1 * w1.y; acc1[6] += x1 * w1.z; acc1[7] += x1 * w1.w;
                    }
                }
            }
            float4 *o = reinterpret_cast<float4 *>(A) + ((size_t)m * 8 + cg * 2) * 60 + k * 20 + mm;
            o[0] = make_float4(acc0[0], acc0[1], acc0[2], acc0[3]);
            o[60] = make_float4(acc0[4], acc0[5], acc0[6], acc0[7]);
            o[10] = make_float4(acc1[0], acc1[1], acc1[2], acc1[3]);
            o[70] = make_float4(acc1[4], acc1[5], acc1[6], acc1[7]);
        } else if (ht < 120 + 108) {           // B: cg(4) x k(3) x l(9): positions (k, l) and (k, l + 9)
            const int it2 = ht - 120;
            const int cg = it2 / 27, r = it2 - cg * 27, k = r / 9, l = r - k * 9;
#pragma unroll
            for (int j = 0; j < 8; ++j) acc0[j] = acc1[j] = 0.0f;
            for (int c = 0; c < 32; ++c) {
#pragma unroll
                for (int dk = 0; dk < 3; ++dk) {
                    const float *row = d2 + c * 100 + (k + dk) * 20 + l;
                    const float4 *wp = reinterpret_cast<const float4 *>(swb + ((c * 3 + dk) * 3) * 32 + cg * 8);
#pragma unroll
                    for (int dl = 0; dl < 3; ++dl) {
                        const float x0 = row[dl], x1 = row[dl + 9];
                        const float4 w0 = wp[dl * 8], w1 = wp[dl * 8 + 1];
                        acc0[0] += x0 * w0.x; acc0[1] += x0 * w0.y; acc0[2] += x0 * w0.z; acc0[3] += x0 * w0.w;
                        acc0[4] += x0 * w1.x; acc0[5] += x0 * w1.y; acc0[6] += x0 * w1.z; acc0[7] += x0 * w1.w;
                        acc1[0] += x1 * w0.x; acc1[1] += x1 * w0.y; acc1[2] += x1 * w0.z; acc1[3] += x1 * w0.w;
                        acc1[4] += x1 * w1.x; acc1[5] += x1 * w1.y; acc1[6] += x1 * w1.z; acc1[7] += x1 * w1.w;
                    }
                }
            }
            float4 *o = reinterpret_cast<float4 *>(B) + ((size_t)m * 8 + cg * 2) * 54 + k * 18 + l;
            o[0] = make_float4(acc0[0], acc0[1], acc0[2], acc0[3]);
            o[54] = make_float4(acc0[4], acc0[5], acc0[6], acc0[7]);
            o[9] = make_float4(acc1[0], acc1[1], acc1[2], acc1[3]);
            o[63] = make_float4(acc1[4], acc1[5], acc1[6], acc1[7]);
        }
    }
}

}  // namespace

BX_API int bx_pool_desc(const float *x, int K, int C, int S, int channels_last, const float *w1, const float *b1,
                        const float *w2, const float *b2, float *desc, float *equi, void *stream) {
    return bx_pool_desc_n(x, K, C, S, channels_last, w1, b1, w2, b2, desc, equi, nullptr, stream);
}

BX_API int bx_pool_desc_n(const float *x, int K, int C, int S, int channels_last, const float *w1, const float *b1,
                          const float *w2, const float *b2, float *desc, float *equi, const int32_t *d_K, void *stream) {
    BX_REQUIRE(x && w1 && b1 && w2 && b2 && desc && equi, "bx_pool_desc: null pointer");
    BX_REQUIRE(C == 32 && S >= 1 && S <= POOL_T && K >= 0, "bx_pool_desc: expects C=32, S<=%d", POOL_T);
    if (K == 0) return BX_OK;
    BX_REQUIRE(!channels_last || (reinterpret_cast<uintptr_t>(x) & 15) == 0, "bx_pool_desc: x must be 16-byte aligned");
    pool_desc_kernel<<<K, POOL_T, 0, bx_stream(stream)>>>(x, K, C, S, channels_last ? 1 : 0, w1, b1, w2, b2, desc, equi, d_K);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_costvol_ab(const float *equi_s, const float *equi_t, const int32_t *s_mids, const int32_t *t_mids,
                         const int32_t *d_M, int maxM, const float *wa, const float *wb, const float *bias, float *A,
                         float *B, void *stream) {
    BX_REQUIRE(equi_s && equi_t && s_mids && t_mids && d_M && wa && wb && bias && A && B, "bx_costvol_ab: null pointer");
    BX_REQUIRE(maxM >= 0, "bx_costvol_ab: bad maxM");
    BX_REQUIRE(((reinterpret_cast<uintptr_t>(wa) | reinterpret_cast<uintptr_t>(wb)) & 15) == 0, "bx_costvol_ab: weights must be 16-byte aligned");
    if (maxM == 0) return BX_OK;
    BX_REQUIRE(((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 15) == 0, "bx_costvol_ab: A and B must be 16-byte aligned");
    static BxPerDevice attr_done = {};
    if (bx_needs_attr(attr_done))
        BX_CUDA(cudaFuncSetAttribute(costvol_ab_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_SMEM));
    int sms = bx_device_sm_count();
    if (sms <= 0) sms = 132;
    const int grid = (maxM + 1) / 2 < sms ? (maxM + 1) / 2 : sms;
    costvol_ab_kernel<<<grid, AB_T, AB_SMEM, bx_stream(stream)>>>(equi_s, equi_t, s_mids, t_mids, d_M, wa, wb, bias, A, B);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
