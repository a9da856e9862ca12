// bx_train.cu -- the per-pair stages of the training-stage validation forward (cfg.stage "Desc" / "Pose", eval mode):
// ground-truth correspondences, SO(2) augmentation of the patches, the EquiMatch score and the SO(2) label.
// Compiled with -fmad=false, every product and sum evaluated in the order written here: the correspondence search is an
// index decision that is bit-identical to the oracle (oracle/train_stages.py: matching_indices), and the augmentation
// follows the same order as oracle/train_stages.py: so2_augment.  EquiMatch and the SO(2) label match the oracle's torch
// formulae to fp32 rounding (the integer label can differ only where angle * azi_n / 2 pi is next to a half-integer).
#include <math.h>

#include "bx_common.cuh"

namespace {

constexpr int GT_THREADS = 128;
constexpr int GT_TILE = 2048;           // target points per shared-memory tile (24 KB)
constexpr float BX_TWO_PI_F = 6.283185307179586f;   // fp32(2*pi): the scalar torch applies to an fp32 tensor

// --------------------------------------------------------------------------------------------------------------
// ground-truth correspondences: nearest target point of every transformed source point (first minimum in target
// order wins ties, like knn_cuda), kept when the distance is below the voxel size
__global__ void __launch_bounds__(GT_THREADS) gt_nn_kernel(const float *__restrict__ src, int N, const float *__restrict__ tgt,
                                                           int M, const float *__restrict__ T, float voxel,
                                                           int *__restrict__ nn) {
    __shared__ float sx[GT_TILE], sy[GT_TILE], sz[GT_TILE];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float qx = 0.f, qy = 0.f, qz = 0.f;
    if (i < N) {
        // utils/SE3.transform: R @ p + t, each row summed left to right
        const float x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
        qx = (((T[0] * x) + (T[1] * y)) + (T[2] * z)) + T[3];
        qy = (((T[4] * x) + (T[5] * y)) + (T[6] * z)) + T[7];
        qz = (((T[8] * x) + (T[9] * y)) + (T[10] * z)) + T[11];
    }
    float best = INFINITY;
    int bj = 0;
    for (int base = 0; base < M; base += GT_TILE) {
        const int n = min(GT_TILE, M - base);
        __syncthreads();
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            sx[j] = tgt[3 * (base + j)];
            sy[j] = tgt[3 * (base + j) + 1];
            sz[j] = tgt[3 * (base + j) + 2];
        }
        __syncthreads();
        if (i < N) {
            for (int j = 0; j < n; ++j) {
                const float d2 = bx_d2(qx - sx[j], qy - sy[j], qz - sz[j]);
                if (d2 < best) {
                    best = d2;
                    bj = base + j;
                }
            }
        }
    }
    if (i < N) nn[i] = (M > 0 && sqrtf(best) < voxel) ? bj : -1;
}

// one CTA: [i, nn(i)] for every kept source point, in source order; *d_count = number kept
__global__ void __launch_bounds__(1024) gt_compact_kernel(const int *__restrict__ nn, int N, int *__restrict__ pairs,
                                                          int *__restrict__ d_count) {
    __shared__ int sh[33];
    int off = 0;
    for (int base = 0; base < N; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const int j = i < N ? nn[i] : -1;
        int total = 0;
        const int ex = bx_block_exscan(j >= 0 ? 1 : 0, sh, &total);
        if (j >= 0) {
            pairs[2 * (off + ex)] = i;
            pairs[2 * (off + ex) + 1] = j;
        }
        off += total;
    }
    if (threadIdx.x == 0) *d_count = off;
}

// --------------------------------------------------------------------------------------------------------------
// kornia axis_angle_to_rotation_matrix for the axis-angle (0, 0, a) -- the form of oracle.azimuth_rotation
__device__ __forceinline__ void azimuth_rotation(float a, float R[9]) {
    const float th2 = a * a;
    if (th2 > 1e-6f) {
        const float th = sqrtf(th2);
        const float wz = a / (th + 1e-6f);
        const float c = cosf(th), s = sinf(th);
        R[0] = c;      R[1] = -(wz * s); R[2] = 0.f;
        R[3] = wz * s; R[4] = c;         R[5] = 0.f;
        R[6] = 0.f;    R[7] = 0.f;       R[8] = c + (wz * wz) * (1.0f - c);
    } else {
        R[0] = 1.f; R[1] = -a;  R[2] = 0.f;
        R[3] = a;   R[4] = 1.f; R[5] = 0.f;
        R[6] = 0.f; R[7] = 0.f; R[8] = 1.f;
    }
}

// v <- v @ R^T, i.e. v'_j = (v0*R[j][0] + v1*R[j][1]) + v2*R[j][2]
__device__ __forceinline__ void rotate_row(float *v, const float R[9]) {
    const float x = v[0], y = v[1], z = v[2];
    v[0] = ((x * R[0]) + (y * R[1])) + (z * R[2]);
    v[1] = ((x * R[3]) + (y * R[4])) + (z * R[5]);
    v[2] = ((x * R[6]) + (y * R[7])) + (z * R[8]);
}

// one CTA per patch
__global__ void so2_augment_kernel(float *__restrict__ delta, int P, float *__restrict__ rand_axis,
                                   const float *__restrict__ angles, float *__restrict__ aug_R) {
    const int k = blockIdx.x;
    float R[9];
    azimuth_rotation(angles[k], R);
    float *d = delta + (size_t)k * P * 3;
    for (int p = threadIdx.x; p < P; p += blockDim.x) rotate_row(d + 3 * p, R);
    if (threadIdx.x == 0) {
        rotate_row(rand_axis + 3 * k, R);
        if (aug_R)
            for (int e = 0; e < 9; ++e) aug_R[9 * k + e] = R[e];
    }
}

// --------------------------------------------------------------------------------------------------------------
// EquiMatch: cor[b,a] = sum_{c,k,l} D1[b,c,k,(l-a) mod L] * D2[b,c,k,l].  One CTA per patch, one warp per shift a;
// lane c sums its channels over (k, l) in order, then a fixed xor-tree sums the 32 lanes.
__global__ void equi_match_kernel(const float *__restrict__ D1, const float *__restrict__ D2, int C, int K, int L,
                                  float *__restrict__ cor) {
    extern __shared__ float sm[];
    const int b = blockIdx.x, n = C * K * L;
    float *s1 = sm, *s2 = sm + n;
    const float *g1 = D1 + (size_t)b * n, *g2 = D2 + (size_t)b * n;
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
        s1[e] = g1[e];
        s2[e] = g2[e];
    }
    __syncthreads();
    const int a = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (a >= L) return;
    float acc = 0.f;
    for (int c = lane; c < C; c += 32) {
        for (int kk = 0; kk < K; ++kk) {
            const float *r1 = s1 + (c * K + kk) * L, *r2 = s2 + (c * K + kk) * L;
            int src = L - a;                        // (l - a) mod L for l = 0
            if (src == L) src = 0;
            for (int l = 0; l < L; ++l) {
                acc = acc + r1[src] * r2[l];
                if (++src == L) src = 0;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(BX_FULL, acc, o);
    if (lane == 0) cor[(size_t)b * L + a] = acc;
}

// --------------------------------------------------------------------------------------------------------------
// SO(2) label of BufferX.cal_so2_gt, one thread per patch
__global__ void so2_gt_kernel(const float *__restrict__ s_ra, const float *__restrict__ s_R, const float *__restrict__ t_R,
                              const float *__restrict__ T, const float *__restrict__ aug_R, int Pn, int azi_n,
                              long long *__restrict__ lab_i, float *__restrict__ lab_f) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Pn) return;
    const float s0 = s_ra[3 * i], s1 = s_ra[3 * i + 1], s2 = s_ra[3 * i + 2];
    // t = s @ gtR^T
    float t[3];
    for (int j = 0; j < 3; ++j) t[j] = ((s0 * T[4 * j]) + (s1 * T[4 * j + 1])) + (s2 * T[4 * j + 2]);
    // s' = s @ s_R, t' = t @ t_R
    const float *A = s_R + 9 * (size_t)i, *B = t_R + 9 * (size_t)i;
    float u[3], v[3];
    for (int j = 0; j < 3; ++j) {
        u[j] = ((s0 * A[j]) + (s1 * A[3 + j])) + (s2 * A[6 + j]);
        v[j] = ((t[0] * B[j]) + (t[1] * B[3 + j])) + (t[2] * B[6 + j]);
    }
    if (aug_R) rotate_row(v, aug_R + 9 * (size_t)i);
    // projection onto the xy plane (t - (t.z) z = (t0, t1, 0)), F.normalize (eps 1e-12)
    const float pn = sqrtf(((v[0] * v[0]) + (v[1] * v[1])) + 0.0f);
    const float pd = fmaxf(pn, 1e-12f);
    const float p0 = v[0] / pd, p1 = v[1] / pd, p2 = 0.0f;
    // F.cosine_similarity: each side divided by max(norm, 1e-8), then the dot product
    const float un = fmaxf(sqrtf(((u[0] * u[0]) + (u[1] * u[1])) + (u[2] * u[2])), 1e-8f);
    const float qn = fmaxf(sqrtf(((p0 * p0) + (p1 * p1)) + (p2 * p2)), 1e-8f);
    const float cs = (((u[0] / un) * (p0 / qn)) + ((u[1] / un) * (p1 / qn))) + ((u[2] / un) * (p2 / qn));
    float ang = acosf(fminf(fmaxf(cs, -1.0f), 1.0f));
    // sign from the z component of s x p
    const float cz = (u[0] * p1) - (u[1] * p0);
    if (cz < 0.0f) ang = BX_TWO_PI_F - ang;
    float lab = (ang * (float)azi_n) / BX_TWO_PI_F;
    if (lab_i) {
        float r = rintf(lab);                       // torch.round: half to even
        if (r == (float)azi_n) r = 0.0f;
        lab_i[i] = (long long)r;
    } else {
        if (lab == (float)azi_n) lab = 0.0f;
        lab_f[i] = lab;
    }
}

}  // namespace

BX_API int bx_gt_matches(const float *src, int N, const float *tgt, int M, const float *T, float voxel, int32_t *nn_ws,
                         int32_t *pairs, int32_t *d_count, void *stream) {
    BX_REQUIRE(src && (tgt || M == 0) && T && nn_ws && pairs && d_count, "bx_gt_matches: null pointer");
    BX_REQUIRE(N >= 0 && M >= 0, "bx_gt_matches: negative size");
    cudaStream_t st = bx_stream(stream);
    if (N == 0) {
        BX_CUDA(cudaMemsetAsync(d_count, 0, sizeof(int), st));
        return BX_OK;
    }
    gt_nn_kernel<<<(N + GT_THREADS - 1) / GT_THREADS, GT_THREADS, 0, st>>>(src, N, tgt, M, T, voxel, nn_ws);
    BX_LAUNCH_CHECK();
    gt_compact_kernel<<<1, 1024, 0, st>>>(nn_ws, N, pairs, d_count);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_so2_augment(float *delta, int K, int P, float *rand_axis, const float *angles, float *aug_R, void *stream) {
    BX_REQUIRE(delta && rand_axis && angles, "bx_so2_augment: null pointer");
    BX_REQUIRE(K >= 0 && P >= 1, "bx_so2_augment: bad sizes");
    if (K == 0) return BX_OK;
    so2_augment_kernel<<<K, 256, 0, bx_stream(stream)>>>(delta, P, rand_axis, angles, aug_R);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_equi_match(const float *D1, const float *D2, int B, int C, int K, int L, float *cor, void *stream) {
    BX_REQUIRE(D1 && D2 && cor, "bx_equi_match: null pointer");
    BX_REQUIRE(B >= 0 && C >= 1 && K >= 1 && L >= 1 && L <= 32, "bx_equi_match: bad sizes (1 <= L <= 32)");
    const size_t smem = 2 * (size_t)C * K * L * sizeof(float);
    BX_REQUIRE(smem <= 48 * 1024, "bx_equi_match: maps of %d x %d x %d do not fit in shared memory", C, K, L);
    if (B == 0) return BX_OK;
    equi_match_kernel<<<B, 32 * L, smem, bx_stream(stream)>>>(D1, D2, C, K, L, cor);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_so2_gt(const float *s_rand_axis, const float *s_R, const float *t_R, const float *T, const float *aug_R, int P,
                     int azi_n, long long *label_int, float *label_float, void *stream) {
    BX_REQUIRE(s_rand_axis && s_R && t_R && T, "bx_so2_gt: null pointer");
    BX_REQUIRE((label_int != nullptr) != (label_float != nullptr), "bx_so2_gt: exactly one of label_int / label_float");
    BX_REQUIRE(P >= 0 && azi_n >= 1, "bx_so2_gt: bad sizes");
    if (P == 0) return BX_OK;
    so2_gt_kernel<<<(P + 127) / 128, 128, 0, bx_stream(stream)>>>(s_rand_axis, s_R, t_R, T, aug_R, P, azi_n, label_int,
                                                                  label_float);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
