// bx_match.cu -- a10 mutual nearest-neighbour matching, a11-tail/a12 pose hypotheses, a13 consensus.
//
// a10 replaces BufferX.mutual_matching (/root/reference/models/BUFFERX.py:469-496): two knn_cuda
// KNN(k=1) calls (two full distance matrices + per-query insertion sort).  Here ONE tiled pass over
// the Ka x Kb pairs computes each squared L2 once and feeds both the row and the column arg-min
// through 64-bit atomicMin on (distance bits << 32 | index) keys -- the packed compare reproduces the
// "first minimum wins" tie rule.  Distances are accumulated over the feature dimension in order
// without FMA, bit-identical to oracle bxo_mutual_nn.
// a12 replaces the softmax expectation (BUFFERX.py:66-69) and the hypothesis build (:382-389).
// a13 replaces the [Mc,Mc,3] broadcast of BUFFERX.py:404-417 (243 MB at Mc=4500) with a
// warp-per-hypothesis inlier counter over shared-memory-resident correspondences.
// Compiled with -fmad=false (bit contracts of bxo_mutual_nn / bxo_consensus).
#include "bx_common.cuh"

namespace {

// ---- a10 --------------------------------------------------------------------------------------------
constexpr int NN_TI = 64;   // rows of a per CTA
constexpr int NN_TJ = 64;   // cols of b per CTA
constexpr int NN_C = 32;    // descriptor length (fixed by the network)

// rows present this launch: min(*d_n, n), or n without a device count
__device__ __forceinline__ int nn_count(const int *d_n, int n) { return d_n ? min(max(*d_n, 0), n) : n; }

// one step of the squared distance, summed over the feature dimension in order from +0 (the arithmetic of bxo_mutual_nn)
__device__ __forceinline__ float nn_acc(float acc, float x, float y) {
    const float t = x - y;
    return acc + (t * t);
}

__global__ void nn_init_kernel(unsigned long long *keys, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) keys[i] = ~0ull;
}

// grid (ceil(Ka/64), ceil(Kb/64)), 256 threads: thread (ti = tid/4 .. handles 1 row, 16 cols)
__global__ void __launch_bounds__(256)
nn_tile_kernel(const float *__restrict__ a, int Ka, const float *__restrict__ b, int Kb,
               unsigned long long *__restrict__ row_keys, unsigned long long *__restrict__ col_keys, const int *__restrict__ d_Ka,
               const int *__restrict__ d_Kb) {
    __shared__ float sa[NN_TI][NN_C + 1];
    __shared__ float sb[NN_TJ][NN_C + 1];
    __shared__ unsigned long long scol[NN_TJ];
    const int i0 = blockIdx.x * NN_TI, j0 = blockIdx.y * NN_TJ;
    Ka = nn_count(d_Ka, Ka);
    Kb = nn_count(d_Kb, Kb);
    if (i0 >= Ka || j0 >= Kb) return;             // the whole CTA: before any barrier
    const int tid = threadIdx.x;
    for (int e = tid; e < NN_TI * NN_C; e += 256) {
        const int r = e / NN_C, c = e % NN_C;
        sa[r][c] = (i0 + r < Ka) ? a[(size_t)(i0 + r) * NN_C + c] : 0.0f;
        sb[r][c] = (j0 + r < Kb) ? b[(size_t)(j0 + r) * NN_C + c] : 0.0f;
    }
    if (tid < NN_TJ) scol[tid] = ~0ull;
    __syncthreads();
    const int ti = tid >> 2;        // 0..63 row inside the tile
    const int tj = tid & 3;         // columns tj, tj+4, ...
    const int gi = i0 + ti;
    unsigned long long rbest = ~0ull;
    if (gi < Ka) {
        for (int jj = tj; jj < NN_TJ; jj += 4) {
            const int gj = j0 + jj;
            if (gj >= Kb) break;
            float acc = 0.0f;
#pragma unroll
            for (int c = 0; c < NN_C; ++c) acc = nn_acc(acc, sa[ti][c], sb[jj][c]);
            const unsigned long long kd = (unsigned long long)__float_as_uint(acc) << 32;
            const unsigned long long rk = kd | (unsigned)gj;
            if (rk < rbest) rbest = rk;
            atomicMin(&scol[jj], kd | (unsigned)gi);
        }
    }
    // combine the 4 threads of a row
    unsigned long long o = __shfl_xor_sync(BX_FULL, rbest, 1);
    if (o < rbest) rbest = o;
    o = __shfl_xor_sync(BX_FULL, rbest, 2);
    if (o < rbest) rbest = o;
    if (tj == 0 && gi < Ka) atomicMin(&row_keys[gi], rbest);
    __syncthreads();
    if (tid < NN_TJ && j0 + tid < Kb) atomicMin(&col_keys[j0 + tid], scol[tid]);
}

// single CTA: mutual mask + ordered compaction
__global__ void __launch_bounds__(1024)
nn_select_kernel(const unsigned long long *__restrict__ row_keys, const unsigned long long *__restrict__ col_keys,
                 int Ka, int Kb, int *__restrict__ s_mids, int *__restrict__ t_mids, int *__restrict__ d_M,
                 int *__restrict__ snn, int *__restrict__ tnn, const int *__restrict__ d_Ka, const int *__restrict__ d_Kb) {
    __shared__ int sh[33];
    Ka = nn_count(d_Ka, Ka);
    Kb = nn_count(d_Kb, Kb);
    if (Ka == 0 || Kb == 0) {                     // a side without key-points: no match, nothing else written
        if (threadIdx.x == 0) *d_M = 0;
        return;
    }
    int run = 0;
    for (int base = 0; base < Ka; base += 1024) {
        const int i = base + threadIdx.x;
        int flag = 0, sj = 0;
        if (i < Ka) {
            sj = (int)(row_keys[i] & 0xffffffffull);
            if (Kb > 0) {
                const int ti = (int)(col_keys[sj] & 0xffffffffull);
                flag = (ti == i) ? 1 : 0;
            }
            if (snn) snn[i] = sj;
        }
        int total;
        const int ex = bx_block_exscan(flag, sh, &total);
        if (flag) {
            s_mids[run + ex] = i;
            t_mids[run + ex] = sj;
        }
        run += total;
    }
    if (tnn)
        for (int j = threadIdx.x; j < Kb; j += 1024) tnn[j] = (int)(col_keys[j] & 0xffffffffull);
    if (threadIdx.x == 0) *d_M = run;
}

// k = 1 nearest neighbour of every query row among the ref rows, any feature length D, B independent problems
// (knn_cuda.KNN(k=1, transpose_mode=True)).  The tile and key scheme of nn_tile_kernel, rows only: grid (ceil(Nq/64),
// ceil(Nr/64), B), 256 threads, thread (row tid/4, columns tid%4 + 4u); the features are staged NN_C at a time and each
// thread carries its 16 partial sums across the stages, so every distance is summed over D in order.
constexpr int KNN_COLS = NN_TJ / 4;

__global__ void __launch_bounds__(256)
knn1_tile_kernel(const float *__restrict__ ref, int Nr, const float *__restrict__ qry, int Nq, int D,
                 unsigned long long *__restrict__ keys) {
    __shared__ float sq[NN_TI][NN_C + 1];
    __shared__ float sr[NN_TJ][NN_C + 1];
    const size_t b = blockIdx.z;
    const int i0 = blockIdx.x * NN_TI, j0 = blockIdx.y * NN_TJ;
    ref += b * Nr * D;
    qry += b * Nq * D;
    const int tid = threadIdx.x, ti = tid >> 2, tj = tid & 3;
    float acc[KNN_COLS];
#pragma unroll
    for (int u = 0; u < KNN_COLS; ++u) acc[u] = 0.0f;
    for (int c0 = 0; c0 < D; c0 += NN_C) {
        const int dc = min(NN_C, D - c0);
        for (int e = tid; e < NN_TI * NN_C; e += 256) {
            const int r = e / NN_C, c = e % NN_C;
            sq[r][c] = (i0 + r < Nq && c < dc) ? qry[(size_t)(i0 + r) * D + c0 + c] : 0.0f;
            sr[r][c] = (j0 + r < Nr && c < dc) ? ref[(size_t)(j0 + r) * D + c0 + c] : 0.0f;
        }
        __syncthreads();
        for (int c = 0; c < dc; ++c) {
            const float x = sq[ti][c];
#pragma unroll
            for (int u = 0; u < KNN_COLS; ++u) acc[u] = nn_acc(acc[u], x, sr[tj + 4 * u][c]);
        }
        __syncthreads();
    }
    unsigned long long best = ~0ull;
#pragma unroll
    for (int u = 0; u < KNN_COLS; ++u) {
        const int gj = j0 + tj + 4 * u;
        const unsigned long long k = ((unsigned long long)__float_as_uint(acc[u]) << 32) | (unsigned)gj;
        if (gj < Nr && k < best) best = k;
    }
    unsigned long long o = __shfl_xor_sync(BX_FULL, best, 1);
    if (o < best) best = o;
    o = __shfl_xor_sync(BX_FULL, best, 2);
    if (o < best) best = o;
    if (tj == 0 && i0 + ti < Nq) atomicMin(&keys[b * Nq + i0 + ti], best);
}

__global__ void knn1_finish_kernel(const unsigned long long *__restrict__ keys, size_t n, float *__restrict__ dist,
                                   long long *__restrict__ idx) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long k = keys[i];
    dist[i] = sqrtf(__uint_as_float((unsigned)(k >> 32)));
    idx[i] = (long long)(k & 0xffffffffull);
}

// ---- a11 tail + a12 ---------------------------------------------------------------------------------
__global__ void hypotheses_kernel(const float *__restrict__ logits, int azi_n, const float *__restrict__ kpts_s,
                                  const float *__restrict__ kpts_t, const float *__restrict__ Rt_s,
                                  const float *__restrict__ Rt_t, const int *__restrict__ s_mids,
                                  const int *__restrict__ t_mids, const int *__restrict__ d_M,
                                  const int *__restrict__ d_off, int *__restrict__ d_off_out,
                                  float *__restrict__ ind_out, float *__restrict__ R_acc, float *__restrict__ t_acc,
                                  float *__restrict__ ss_acc, float *__restrict__ tt_acc) {
    const int M = *d_M, off = *d_off;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) *d_off_out = off + M;
    if (i >= M) return;
    // softmax expectation over the azimuth bins
    const float *lg = logits + (size_t)i * azi_n;
    float mx = lg[0];
    for (int k = 1; k < azi_n; ++k) mx = fmaxf(mx, lg[k]);
    float den = 0.0f, num = 0.0f;
    for (int k = 0; k < azi_n; ++k) {
        const float e = expf(lg[k] - mx);
        den += e;
        num += e * (float)k;
    }
    const float ind = num / den;
    if (ind_out) ind_out[i] = ind;
    // angle = ind*2*pi/azi_n + 1e-6 ; kornia axis_angle_to_rotation_matrix for (0,0,angle)
    const float angle = ((ind * 2.0f) * 3.14159265358979323846f) / (float)azi_n + 1e-6f;
    const float th2 = angle * angle;
    float A[3][3];
    if (th2 > 1e-6f) {
        const float th = sqrtf(th2);
        const float wz = angle / (th + 1e-6f);
        const float c = cosf(th), s = sinf(th);
        A[0][0] = c;       A[0][1] = -wz * s; A[0][2] = 0.f;
        A[1][0] = wz * s;  A[1][1] = c;       A[1][2] = 0.f;
        A[2][0] = 0.f;     A[2][1] = 0.f;     A[2][2] = c + wz * wz * (1.0f - c);
    } else {
        A[0][0] = 1.f;   A[0][1] = -angle; A[0][2] = 0.f;
        A[1][0] = angle; A[1][1] = 1.f;    A[1][2] = 0.f;
        A[2][0] = 0.f;   A[2][1] = 0.f;    A[2][2] = 1.f;
    }
    const int si = s_mids[i], ti = t_mids[i];
    const float *Rs = Rt_s + (size_t)si * 9, *Rtt = Rt_t + (size_t)ti * 9;
    // R = tt_R @ A @ ss_R^T
    float B[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) B[r][c] = Rtt[3 * r] * A[0][c] + Rtt[3 * r + 1] * A[1][c] + Rtt[3 * r + 2] * A[2][c];
    float R[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) R[r][c] = B[r][0] * Rs[3 * c] + B[r][1] * Rs[3 * c + 1] + B[r][2] * Rs[3 * c + 2];
    const float sx = kpts_s[3 * (size_t)si], sy = kpts_s[3 * (size_t)si + 1], sz = kpts_s[3 * (size_t)si + 2];
    const float tx = kpts_t[3 * (size_t)ti], tyy = kpts_t[3 * (size_t)ti + 1], tz = kpts_t[3 * (size_t)ti + 2];
    const size_t o = (size_t)(off + i);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) R_acc[o * 9 + 3 * r + c] = R[r][c];
    t_acc[o * 3] = tx - (R[0][0] * sx + R[0][1] * sy + R[0][2] * sz);
    t_acc[o * 3 + 1] = tyy - (R[1][0] * sx + R[1][1] * sy + R[1][2] * sz);
    t_acc[o * 3 + 2] = tz - (R[2][0] * sx + R[2][1] * sy + R[2][2] * sz);
    ss_acc[o * 3] = sx; ss_acc[o * 3 + 1] = sy; ss_acc[o * 3 + 2] = sz;
    tt_acc[o * 3] = tx; tt_acc[o * 3 + 1] = tyy; tt_acc[o * 3 + 2] = tz;
}

// ---- a13 --------------------------------------------------------------------------------------------
__device__ __forceinline__ bool consensus_inlier(const float *Rj, const float *tj, float x, float y, float z, float gx,
                                                 float gy, float gz, float thr) {
    const float qx = (((Rj[0] * x) + (Rj[1] * y)) + (Rj[2] * z)) + tj[0];
    const float qy = (((Rj[3] * x) + (Rj[4] * y)) + (Rj[5] * z)) + tj[1];
    const float qz = (((Rj[6] * x) + (Rj[7] * y)) + (Rj[8] * z)) + tj[2];
    const float d = sqrtf(bx_d2(qx - gx, qy - gy, qz - gz));
    return d < thr;
}

// one warp per hypothesis j; the correspondences are read through L1 (Mc <= a few thousand).
__global__ void __launch_bounds__(256)
consensus_count_kernel(const float *__restrict__ ss, const float *__restrict__ tt, const float *__restrict__ R,
                       const float *__restrict__ t, const int *__restrict__ d_Mc, int azi_n, float inlier_th,
                       int *__restrict__ counts) {
    const int Mc = *d_Mc;
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (j >= Mc) return;
    float Rj[9], tj[3];
#pragma unroll
    for (int e = 0; e < 9; ++e) Rj[e] = R[(size_t)j * 9 + e];
#pragma unroll
    for (int e = 0; e < 3; ++e) tj[e] = t[(size_t)j * 3 + e];
    const float pi_f = 3.14159265358979323846f;
    int c = 0;
    for (int i = lane; i < Mc; i += 32) {
        const float x = ss[3 * (size_t)i], y = ss[3 * (size_t)i + 1], z = ss[3 * (size_t)i + 2];
        const float nrm = sqrtf(((x * x) + (y * y)) + (z * z));
        const float thr = ((nrm * pi_f) / (float)azi_n) * inlier_th;
        c += consensus_inlier(Rj, tj, x, y, z, tt[3 * (size_t)i], tt[3 * (size_t)i + 1], tt[3 * (size_t)i + 2], thr) ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) c += __shfl_xor_sync(BX_FULL, c, o);
    if (lane == 0) counts[j] = c;
}

// single CTA: first arg-max of counts, then the ordered inlier list of the winner
__global__ void __launch_bounds__(1024)
consensus_select_kernel(const float *__restrict__ ss, const float *__restrict__ tt, const float *__restrict__ R,
                        const float *__restrict__ t, const int *__restrict__ d_Mc, int azi_n, float inlier_th,
                        const int *__restrict__ counts, int *__restrict__ inlier_ind, int *__restrict__ d_I,
                        int *__restrict__ d_best) {
    __shared__ int sh[33];
    __shared__ unsigned long long sbest[32];
    __shared__ int s_best;
    const int Mc = *d_Mc;
    if (Mc <= 0) {
        if (threadIdx.x == 0) { *d_I = 0; *d_best = 0; }
        return;
    }
    // key = (count << 32) | ~j  -> max picks the largest count, lowest j on ties
    unsigned long long key = 0ull;
    for (int j = threadIdx.x; j < Mc; j += 1024) {
        const unsigned long long k = ((unsigned long long)(unsigned)counts[j] << 32) | (unsigned)(~(unsigned)j);
        if (k > key) key = k;
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(BX_FULL, key, o);
        if (other > key) key = other;
    }
    if ((threadIdx.x & 31) == 0) sbest[threadIdx.x >> 5] = key;
    __syncthreads();
    if (threadIdx.x < 32) {
        unsigned long long k = sbest[threadIdx.x];
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(BX_FULL, k, o);
            if (other > k) k = other;
        }
        if (threadIdx.x == 0) s_best = (int)(~(unsigned)(k & 0xffffffffull));
    }
    __syncthreads();
    const int b = s_best;
    float Rj[9], tj[3];
#pragma unroll
    for (int e = 0; e < 9; ++e) Rj[e] = R[(size_t)b * 9 + e];
#pragma unroll
    for (int e = 0; e < 3; ++e) tj[e] = t[(size_t)b * 3 + e];
    const float pi_f = 3.14159265358979323846f;
    int run = 0;
    for (int base = 0; base < Mc; base += 1024) {
        const int i = base + threadIdx.x;
        int flag = 0;
        if (i < Mc) {
            const float x = ss[3 * (size_t)i], y = ss[3 * (size_t)i + 1], z = ss[3 * (size_t)i + 2];
            const float nrm = sqrtf(((x * x) + (y * y)) + (z * z));
            const float thr = ((nrm * pi_f) / (float)azi_n) * inlier_th;
            flag = consensus_inlier(Rj, tj, x, y, z, tt[3 * (size_t)i], tt[3 * (size_t)i + 1], tt[3 * (size_t)i + 2], thr) ? 1 : 0;
        }
        int total;
        const int ex = bx_block_exscan(flag, sh, &total);
        if (flag) inlier_ind[run + ex] = i;
        run += total;
    }
    if (threadIdx.x == 0) { *d_I = run; *d_best = b; }
}

}  // namespace

BX_API int bx_mutual_nn(const float *a, int Ka, const float *b, int Kb, int C, unsigned long long *keys, int32_t *s_mids,
                        int32_t *t_mids, int32_t *d_M, int32_t *snn, int32_t *tnn, void *stream) {
    return bx_mutual_nn_n(a, Ka, b, Kb, C, nullptr, nullptr, keys, s_mids, t_mids, d_M, snn, tnn, stream);
}

BX_API int bx_mutual_nn_n(const float *a, int Ka, const float *b, int Kb, int C, const int32_t *d_Ka, const int32_t *d_Kb,
                          unsigned long long *keys, int32_t *s_mids, int32_t *t_mids, int32_t *d_M, int32_t *snn, int32_t *tnn,
                          void *stream) {
    BX_REQUIRE(a && b && keys && s_mids && t_mids && d_M, "bx_mutual_nn: null pointer");
    BX_REQUIRE(C == NN_C, "bx_mutual_nn: descriptor length must be %d", NN_C);
    BX_REQUIRE(Ka >= 0 && Kb >= 0, "bx_mutual_nn: negative size");
    cudaStream_t st = bx_stream(stream);
    if (Ka == 0 || Kb == 0) {
        BX_CUDA(cudaMemsetAsync(d_M, 0, sizeof(int), st));
        return BX_OK;
    }
    nn_init_kernel<<<(Ka + Kb + 255) / 256, 256, 0, st>>>(keys, Ka + Kb);
    BX_LAUNCH_CHECK();
    dim3 grid((Ka + NN_TI - 1) / NN_TI, (Kb + NN_TJ - 1) / NN_TJ);
    nn_tile_kernel<<<grid, 256, 0, st>>>(a, Ka, b, Kb, keys, keys + Ka, d_Ka, d_Kb);
    BX_LAUNCH_CHECK();
    nn_select_kernel<<<1, 1024, 0, st>>>(keys, keys + Ka, Ka, Kb, s_mids, t_mids, d_M, snn, tnn, d_Ka, d_Kb);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_knn1(const float *ref, int Nr, const float *qry, int Nq, int D, int B, unsigned long long *keys, float *dist,
                   int64_t *idx, void *stream) {
    BX_REQUIRE(ref && qry && keys && dist && idx, "bx_knn1: null pointer");
    BX_REQUIRE(B >= 1 && B <= 65535 && Nr >= 1 && Nq >= 0 && D >= 1,
               "bx_knn1: bad sizes (B=%d in [1,65535], Nr=%d >= 1, Nq=%d >= 0, D=%d >= 1)", B, Nr, Nq, D);
    BX_REQUIRE((long long)B * Nq < (1ll << 31), "bx_knn1: B*Nq=%lld query rows exceed 2^31", (long long)B * Nq);
    BX_REQUIRE(Nr <= 65535 * NN_TJ, "bx_knn1: Nr=%d exceeds %d ref rows", Nr, 65535 * NN_TJ);
    if (Nq == 0) return BX_OK;
    cudaStream_t st = bx_stream(stream);
    const int n = B * Nq;
    nn_init_kernel<<<(n + 255) / 256, 256, 0, st>>>(keys, n);
    BX_LAUNCH_CHECK();
    knn1_tile_kernel<<<dim3((unsigned)((Nq + NN_TI - 1) / NN_TI), (unsigned)((Nr + NN_TJ - 1) / NN_TJ), (unsigned)B), 256, 0, st>>>(
        ref, Nr, qry, Nq, D, keys);
    BX_LAUNCH_CHECK();
    knn1_finish_kernel<<<(n + 255) / 256, 256, 0, st>>>(keys, (size_t)n, dist, reinterpret_cast<long long *>(idx));
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_hypotheses(const float *logits, int azi_n, const float *kpts_s, const float *kpts_t, const float *Rt_s,
                         const float *Rt_t, const int32_t *s_mids, const int32_t *t_mids, const int32_t *d_M, int maxM,
                         const int32_t *d_off, int32_t *d_off_out, float *ind_out, float *R_acc, float *t_acc,
                         float *ss_acc, float *tt_acc, void *stream) {
    BX_REQUIRE(logits && kpts_s && kpts_t && Rt_s && Rt_t && s_mids && t_mids && d_M && d_off && d_off_out && R_acc &&
                   t_acc && ss_acc && tt_acc,
               "bx_hypotheses: null pointer");
    BX_REQUIRE(azi_n >= 1 && maxM >= 0, "bx_hypotheses: bad sizes");
    BX_REQUIRE(d_off != d_off_out, "bx_hypotheses: d_off and d_off_out must differ");
    const int blocks = maxM > 0 ? (maxM + 127) / 128 : 1;
    hypotheses_kernel<<<blocks, 128, 0, bx_stream(stream)>>>(logits, azi_n, kpts_s, kpts_t, Rt_s, Rt_t, s_mids, t_mids, d_M,
                                                            d_off, d_off_out, ind_out, R_acc, t_acc, ss_acc, tt_acc);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

namespace {
struct ConcatOffsets { int s_off[8], t_off[8]; };

// one CTA per scale: the scale's match list is appended at the prefix sum of the earlier scales' device-side counts
__global__ void concat_matches_kernel(const int *__restrict__ s_lists, const int *__restrict__ t_lists,
                                      const int *__restrict__ d_counts, int S, int stride, ConcatOffsets ro,
                                      int *__restrict__ s_all, int *__restrict__ t_all, int *__restrict__ d_offs) {
    const int i = blockIdx.x;
    int off = 0;
    for (int j = 0; j < i; ++j) off += d_counts[j];
    const int M = d_counts[i];
    if (threadIdx.x == 0) {
        d_offs[i] = off;
        if (i == S - 1) d_offs[S] = off + M;
    }
    for (int m = threadIdx.x; m < M; m += blockDim.x) {
        s_all[off + m] = s_lists[(size_t)i * stride + m] + ro.s_off[i];
        t_all[off + m] = t_lists[(size_t)i * stride + m] + ro.t_off[i];
    }
}
}  // namespace

BX_API int bx_concat_matches(const int32_t *s_lists, const int32_t *t_lists, const int32_t *d_counts, int S, int stride,
                             const int32_t *h_s_off, const int32_t *h_t_off, int32_t *s_all, int32_t *t_all,
                             int32_t *d_offs, void *stream) {
    BX_REQUIRE(s_lists && t_lists && d_counts && h_s_off && h_t_off && s_all && t_all && d_offs, "bx_concat_matches: null pointer");
    BX_REQUIRE(S >= 1 && S <= 8 && stride >= 0, "bx_concat_matches: 1 <= S <= 8");
    ConcatOffsets ro = {};
    for (int i = 0; i < S; ++i) { ro.s_off[i] = h_s_off[i]; ro.t_off[i] = h_t_off[i]; }
    concat_matches_kernel<<<S, 256, 0, bx_stream(stream)>>>(s_lists, t_lists, d_counts, S, stride, ro, s_all, t_all, d_offs);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_consensus(const float *ss, const float *tt, const float *R, const float *t, const int32_t *d_Mc, int maxMc,
                        int azi_n, float inlier_th, int32_t *counts, int32_t *inlier_ind, int32_t *d_I, int32_t *d_best,
                        void *stream) {
    BX_REQUIRE(ss && tt && R && t && d_Mc && counts && inlier_ind && d_I && d_best, "bx_consensus: null pointer");
    BX_REQUIRE(maxMc >= 0 && azi_n >= 1, "bx_consensus: bad sizes");
    cudaStream_t st = bx_stream(stream);
    if (maxMc > 0) {
        consensus_count_kernel<<<(maxMc + 7) / 8, 256, 0, st>>>(ss, tt, R, t, d_Mc, azi_n, inlier_th, counts);
        BX_LAUNCH_CHECK();
    }
    consensus_select_kernel<<<1, 1024, 0, st>>>(ss, tt, R, t, d_Mc, azi_n, inlier_th, counts, inlier_ind, d_I, d_best);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
