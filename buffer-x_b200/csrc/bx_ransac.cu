// bx_ransac.cu -- a14 RANSAC hypothesise-and-verify, a15 post refinement (fp64 geometry).
//
// a14 replaces PoseEstimator._estimate_ransac (/root/reference/models/pose_estimator.py:84-117), i.e.
// Open3D 0.18 RegistrationRANSACBasedOnCorrespondence running on host cores with a D2H/H2D round trip
// (pose_estimator.py:36-38).  Device pipeline per chunk of iterations (no host involvement):
//   1. hypothesise: one thread per iteration -- Philox4x32-10(seed, itr) draws 3 correspondences,
//      EdgeLength checker, Horn quaternion fit (4x4 cyclic Jacobi), Distance checker; survivors are
//      compacted into a pass list (warp-aggregated atomic).
//   2. verify: one thread per surviving hypothesis walks the correspondence list in order (all lanes
//      read the same correspondence -> broadcast loads) accumulating the inlier count and squared error
//      in the ORACLE's order, so (good, rmse) are bit-identical to oracle bxo_ransac.
//   3. scan: one warp replays Open3D's sequential bookkeeping over the chunk (better := more inliers,
//      ties by rmse; confidence-driven est_k; stop when itr >= est_k).
// Later chunks see est_k in device memory and turn into no-ops once itr >= est_k.
// a15 replaces post_refinement + rigid_transform_3d (/root/reference/models/BUFFERX.py:522-603; builds
// an I x I diag matrix for a 3x3 result): one CTA, <= 20 rounds, weighted Horn fit from 16 block sums.
// Compiled with -fmad=false (bit contract with the oracle's fp64 arithmetic).
#include "bx_common.cuh"

namespace {

struct RansacState {      // lives at the head of the workspace
    double T[16];
    double best_rmse;
    int best_good;
    int best_itr;
    int est_k;
    int iters_run;
    int pass_count;
    int pad;
};

struct RansacResult {     // 144 bytes, mirrored in the header comment
    double T[16];
    int num_inliers, best_itr, iters_run, reserved;
};

constexpr int CHUNK = 8192;

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                              uint32_t k1, uint32_t (&out)[4]) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
        const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = h1 ^ c1 ^ k0, n1 = l1, n2 = h0 ^ c3 ^ k1, n3 = l0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// symmetric 4x4 stored as the 10 upper-triangle scalars + 16 eigenvector scalars, all in registers
struct Sym4 {
    double a00, a01, a02, a03, a11, a12, a13, a22, a23, a33;
};

#define BX_ROT(App, Aqq, Apq, Arp, Arq, Asp, Asq, V0p, V0q, V1p, V1q, V2p, V2q, V3p, V3q)      \
    do {                                                                                         \
        const double apq = (Apq);                                                                \
        if (apq != 0.0) {                                                                        \
            const double theta = ((Aqq) - (App)) / (2.0 * apq);                                  \
            const double at = fabs(theta);                                                       \
            double tt_ = 1.0 / (at + sqrt((theta * theta) + 1.0));                               \
            if (theta < 0.0) tt_ = -tt_;                                                         \
            const double c_ = 1.0 / sqrt((tt_ * tt_) + 1.0);                                     \
            const double s_ = tt_ * c_;                                                          \
            (App) = (App) - (tt_ * apq);                                                         \
            (Aqq) = (Aqq) + (tt_ * apq);                                                         \
            (Apq) = 0.0;                                                                         \
            double x_, y_;                                                                       \
            x_ = (Arp); y_ = (Arq); (Arp) = (c_ * x_) - (s_ * y_); (Arq) = (s_ * x_) + (c_ * y_); \
            x_ = (Asp); y_ = (Asq); (Asp) = (c_ * x_) - (s_ * y_); (Asq) = (s_ * x_) + (c_ * y_); \
            x_ = (V0p); y_ = (V0q); (V0p) = (c_ * x_) - (s_ * y_); (V0q) = (s_ * x_) + (c_ * y_); \
            x_ = (V1p); y_ = (V1q); (V1p) = (c_ * x_) - (s_ * y_); (V1q) = (s_ * x_) + (c_ * y_); \
            x_ = (V2p); y_ = (V2q); (V2p) = (c_ * x_) - (s_ * y_); (V2q) = (s_ * x_) + (c_ * y_); \
            x_ = (V3p); y_ = (V3q); (V3p) = (c_ * x_) - (s_ * y_); (V3q) = (s_ * x_) + (c_ * y_); \
        }                                                                                        \
    } while (0)

// Horn's closed form from the cross-covariance S (row-major 3x3), centroids ca, cb -> T (row-major 4x4).
// Same operation order as oracle horn_fit / jacobi4_max_eigvec.
__device__ void horn_from_S(const double (&S)[3][3], const double (&ca)[3], const double (&cb)[3], double (&T)[16]) {
    double a00 = (S[0][0] + S[1][1]) + S[2][2];
    double a01 = S[1][2] - S[2][1];
    double a02 = S[2][0] - S[0][2];
    double a03 = S[0][1] - S[1][0];
    double a11 = (S[0][0] - S[1][1]) - S[2][2];
    double a12 = S[0][1] + S[1][0];
    double a13 = S[2][0] + S[0][2];
    double a22 = ((-S[0][0]) + S[1][1]) - S[2][2];
    double a23 = S[1][2] + S[2][1];
    double a33 = ((-S[0][0]) - S[1][1]) + S[2][2];
    double v00 = 1, v01 = 0, v02 = 0, v03 = 0, v10 = 0, v11 = 1, v12 = 0, v13 = 0;
    double v20 = 0, v21 = 0, v22 = 1, v23 = 0, v30 = 0, v31 = 0, v32 = 0, v33 = 1;
    for (int sweep = 0; sweep < 10; ++sweep) {
        // (p,q) in the oracle's order; "r,s" are the two remaining indices in increasing order
        BX_ROT(a00, a11, a01, a02, a12, a03, a13, v00, v01, v10, v11, v20, v21, v30, v31);  // (0,1): r=2,s=3
        BX_ROT(a00, a22, a02, a01, a12, a03, a23, v00, v02, v10, v12, v20, v22, v30, v32);  // (0,2): r=1,s=3
        BX_ROT(a00, a33, a03, a01, a13, a02, a23, v00, v03, v10, v13, v20, v23, v30, v33);  // (0,3): r=1,s=2
        BX_ROT(a11, a22, a12, a01, a02, a13, a23, v01, v02, v11, v12, v21, v22, v31, v32);  // (1,2): r=0,s=3
        BX_ROT(a11, a33, a13, a01, a03, a12, a23, v01, v03, v11, v13, v21, v23, v31, v33);  // (1,3): r=0,s=2
        BX_ROT(a22, a33, a23, a02, a03, a12, a13, v02, v03, v12, v13, v22, v23, v32, v33);  // (2,3): r=0,s=1
    }
    double em = a00, q0 = v00, q1 = v10, q2 = v20, q3 = v30;
    if (a11 > em) { em = a11; q0 = v01; q1 = v11; q2 = v21; q3 = v31; }
    if (a22 > em) { em = a22; q0 = v02; q1 = v12; q2 = v22; q3 = v32; }
    if (a33 > em) { em = a33; q0 = v03; q1 = v13; q2 = v23; q3 = v33; }
    const double qn = sqrt((((q0 * q0) + (q1 * q1)) + (q2 * q2)) + (q3 * q3));
    const double w = q0 / qn, x = q1 / qn, y = q2 / qn, z = q3 / qn;
    double R[3][3];
    R[0][0] = 1.0 - (2.0 * ((y * y) + (z * z)));
    R[0][1] = 2.0 * ((x * y) - (w * z));
    R[0][2] = 2.0 * ((x * z) + (w * y));
    R[1][0] = 2.0 * ((x * y) + (w * z));
    R[1][1] = 1.0 - (2.0 * ((x * x) + (z * z)));
    R[1][2] = 2.0 * ((y * z) - (w * x));
    R[2][0] = 2.0 * ((x * z) - (w * y));
    R[2][1] = 2.0 * ((y * z) + (w * x));
    R[2][2] = 1.0 - (2.0 * ((x * x) + (y * y)));
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) T[4 * r + c] = R[r][c];
        T[4 * r + 3] = cb[r] - (((R[r][0] * ca[0]) + (R[r][1] * ca[1])) + (R[r][2] * ca[2]));
    }
    T[12] = 0.0; T[13] = 0.0; T[14] = 0.0; T[15] = 1.0;
}

__global__ void ransac_init_kernel(RansacState *st, int max_iter) {
    if (threadIdx.x == 0) {
        for (int i = 0; i < 16; ++i) st->T[i] = (i % 5 == 0) ? 1.0 : 0.0;
        st->best_rmse = 0.0;
        st->best_good = 0;
        st->best_itr = -1;
        st->est_k = max_iter;
        st->iters_run = 0;
        st->pass_count = 0;
    }
}

// 1. hypothesise
__global__ void __launch_bounds__(128)
ransac_hyp_kernel(const float *__restrict__ ss, const float *__restrict__ tt, const int *__restrict__ inlier_ind,
                  const int *__restrict__ d_I, double dist_th, double similar_th, int itr0, int itr1, uint32_t k0,
                  uint32_t k1, RansacState *__restrict__ st, int *__restrict__ pass_itr, double *__restrict__ pass_T,
                  int *__restrict__ rec_good) {
    const int I = *d_I;
    const int itr = itr0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (I < 3 || itr0 >= st->est_k) return;
    bool ok = itr < itr1;
    double T[16];
    if (ok) {
        rec_good[itr - itr0] = -1;
        uint32_t rnd[4];
        philox4x32_10((uint32_t)itr, 0u, 0u, 0u, k0, k1, rnd);
        double a[3][3], b[3][3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int sel = (int)__umulhi(rnd[j], (uint32_t)I);
            const int c = inlier_ind[sel];
#pragma unroll
            for (int e = 0; e < 3; ++e) {
                a[j][e] = (double)ss[3 * (size_t)c + e];
                b[j][e] = (double)tt[3 * (size_t)c + e];
            }
        }
        // EdgeLength checker
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = i + 1; j < 3; ++j) {
                double ds = 0.0, dt = 0.0;
#pragma unroll
                for (int e = 0; e < 3; ++e) {
                    const double u = a[i][e] - a[j][e], v = b[i][e] - b[j][e];
                    ds = ds + (u * u);
                    dt = dt + (v * v);
                }
                ds = sqrt(ds);
                dt = sqrt(dt);
                if (ds < dt * similar_th || dt < ds * similar_th) ok = false;
            }
        if (ok) {
            // unit-weight Horn fit: centroids, cross-covariance (sequential over the 3 samples)
            double ca[3] = {0, 0, 0}, cb[3] = {0, 0, 0}, sw = 0.0;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                sw = sw + 1.0;
#pragma unroll
                for (int e = 0; e < 3; ++e) {
                    ca[e] = ca[e] + (1.0 * a[j][e]);
                    cb[e] = cb[e] + (1.0 * b[j][e]);
                }
            }
#pragma unroll
            for (int e = 0; e < 3; ++e) { ca[e] = ca[e] / sw; cb[e] = cb[e] / sw; }
            double S[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                double da[3], db[3];
#pragma unroll
                for (int e = 0; e < 3; ++e) { da[e] = a[j][e] - ca[e]; db[e] = b[j][e] - cb[e]; }
#pragma unroll
                for (int r = 0; r < 3; ++r)
#pragma unroll
                    for (int c = 0; c < 3; ++c) S[r][c] = S[r][c] + ((1.0 * da[r]) * db[c]);
            }
            horn_from_S(S, ca, cb, T);
            // Distance checker
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                double e2 = 0.0;
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    const double o = (((T[4 * r] * a[j][0]) + (T[4 * r + 1] * a[j][1])) + (T[4 * r + 2] * a[j][2])) + T[4 * r + 3];
                    const double u = b[j][r] - o;
                    e2 = e2 + (u * u);
                }
                if (sqrt(e2) > dist_th) ok = false;
            }
        }
    }
    // warp-aggregated append to the pass list
    const unsigned m = __ballot_sync(BX_FULL, ok);
    if (m) {
        const int lane = threadIdx.x & 31;
        int base = 0;
        if (lane == (__ffs(m) - 1)) base = atomicAdd(&st->pass_count, __popc(m));
        base = __shfl_sync(BX_FULL, base, __ffs(m) - 1);
        if (ok) {
            const int slot = base + __popc(m & ((1u << lane) - 1u));
            pass_itr[slot] = itr;
#pragma unroll
            for (int e = 0; e < 12; ++e) pass_T[(size_t)slot * 12 + e] = T[e];
        }
    }
}

// 2. verify: one thread per surviving hypothesis
__global__ void __launch_bounds__(128)
ransac_verify_kernel(const float *__restrict__ ss, const float *__restrict__ tt, const int *__restrict__ inlier_ind,
                     const int *__restrict__ d_I, double dist_th, int itr0, const RansacState *__restrict__ st,
                     const int *__restrict__ pass_itr, const double *__restrict__ pass_T, int *__restrict__ rec_good,
                     double *__restrict__ rec_rmse) {
    const int I = *d_I;
    const int np = st->pass_count;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (I < 3 || itr0 >= st->est_k || s >= np) return;
    double T[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) T[e] = pass_T[(size_t)s * 12 + e];
    const double max_d2 = dist_th * dist_th;
    int good = 0;
    double err2 = 0.0;
    for (int i = 0; i < I; ++i) {
        const int c = inlier_ind[i];
        const double x = (double)ss[3 * (size_t)c], y = (double)ss[3 * (size_t)c + 1], z = (double)ss[3 * (size_t)c + 2];
        double e2 = 0.0;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const double o = (((T[4 * r] * x) + (T[4 * r + 1] * y)) + (T[4 * r + 2] * z)) + T[4 * r + 3];
            const double u = o - (double)tt[3 * (size_t)c + r];
            e2 = e2 + (u * u);
        }
        if (e2 < max_d2) { ++good; err2 += e2; }
    }
    const int itr = pass_itr[s];
    rec_good[itr - itr0] = good;
    rec_rmse[itr - itr0] = good ? sqrt(err2 / (double)good) : 0.0;
}

// 3. sequential bookkeeping of Open3D's loop over this chunk (one warp)
__global__ void __launch_bounds__(32)
ransac_scan_kernel(const int *__restrict__ d_I, double confidence, int itr0, int itr1, int max_iter,
                   RansacState *__restrict__ st, const int *__restrict__ pass_itr, const double *__restrict__ pass_T,
                   const int *__restrict__ rec_good, const double *__restrict__ rec_rmse, RansacResult *__restrict__ res,
                   int last_chunk) {
    const int I = *d_I;
    const int lane = threadIdx.x;
    int est_k = st->est_k, best_good = st->best_good, best_itr = st->best_itr, iters_run = st->iters_run;
    double best_rmse = st->best_rmse;
    const bool active = (I >= 3) && (itr0 < est_k);
    if (active) {
        const int np = st->pass_count;
        int itr = itr0, last = itr0;  // last = first iteration after the most recent improvement
        while (itr < itr1 && itr < est_k) {
            // look at 32 iterations at a time; find the first one that improves on the current best
            const int my = itr + lane;
            bool better = false;
            if (my < itr1 && my < est_k) {
                const int g = rec_good[my - itr0];
                if (g >= 0) {
                    const double r = rec_rmse[my - itr0];
                    better = (g > best_good) || (g == best_good && r < best_rmse);
                }
            }
            const unsigned m = __ballot_sync(BX_FULL, better);
            if (!m) {
                itr += 32;
                continue;
            }
            const int src = __ffs(m) - 1;
            const int bi = itr + src;
            best_good = rec_good[bi - itr0];
            best_rmse = rec_rmse[bi - itr0];
            best_itr = bi;
            const double ratio = (double)best_good / (double)I;
            const double est = log(1.0 - confidence) / log(1.0 - pow(ratio, 3.0));
            if (est < (double)est_k) est_k = (int)ceil(est);
            itr = bi + 1;  // re-examine the iterations after the improvement against the new best
            last = itr;
        }
        // the sequential loop leaves at the first itr >= est_k (never before the iteration after the
        // last improvement), or runs on into the next chunk
        iters_run = min(itr1, max(est_k, last));
        // fetch the transform of the winner if it changed in this chunk
        if (best_itr >= itr0 && best_itr != st->best_itr) {
            for (int s = lane; s < np; s += 32)
                if (pass_itr[s] == best_itr) {
                    for (int e = 0; e < 12; ++e) st->T[e] = pass_T[(size_t)s * 12 + e];
                }
        }
        __syncwarp();
        if (lane == 0) {
            st->est_k = est_k;
            st->best_good = best_good;
            st->best_rmse = best_rmse;
            st->best_itr = best_itr;
            st->iters_run = iters_run;
            st->pass_count = 0;  // next chunk starts a fresh pass list
        }
    }
    __syncwarp();
    if (last_chunk && lane == 0) {
        for (int e = 0; e < 16; ++e) res->T[e] = st->T[e];
        res->num_inliers = st->best_good;
        res->best_itr = st->best_itr;
        res->iters_run = (I >= 3) ? min(st->iters_run, max_iter) : 0;
        res->reserved = 0;
    }
}

// ---- a15 --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
refine_kernel(const float *__restrict__ ss, const float *__restrict__ tt, const int *__restrict__ d_n,
              const double *__restrict__ T_in, float dist_th, float *__restrict__ T_out, int *__restrict__ d_rounds) {
    __shared__ double red[8][16];
    __shared__ int redc[8];
    __shared__ float sT[16];
    __shared__ int s_cnt;
    const int n = *d_n;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 16) sT[tid] = (float)T_in[tid];
    __syncthreads();
    int prev = 0, r = 0;
    for (r = 0; r < 20; ++r) {
        float T[12];
#pragma unroll
        for (int e = 0; e < 12; ++e) T[e] = sT[e];
        // 16 weighted sums: w, w*a(3), w*b(3), w*a*b^T(9)
        double acc[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[e] = 0.0;
        int cnt = 0;
        for (int i = tid; i < n; i += 256) {
            const float x = ss[3 * (size_t)i], y = ss[3 * (size_t)i + 1], z = ss[3 * (size_t)i + 2];
            const float gx = tt[3 * (size_t)i], gy = tt[3 * (size_t)i + 1], gz = tt[3 * (size_t)i + 2];
            const float qx = (((T[0] * x) + (T[1] * y)) + (T[2] * z)) + T[3];
            const float qy = (((T[4] * x) + (T[5] * y)) + (T[6] * z)) + T[7];
            const float qz = (((T[8] * x) + (T[9] * y)) + (T[10] * z)) + T[11];
            const float d = sqrtf(bx_d2(qx - gx, qy - gy, qz - gz));
            if (d < dist_th) {
                ++cnt;
                const float q = d / dist_th;
                const double w = (double)(1.0f / (1.0f + (q * q)));
                const double a[3] = {(double)x, (double)y, (double)z}, b[3] = {(double)gx, (double)gy, (double)gz};
                acc[0] += w;
#pragma unroll
                for (int e = 0; e < 3; ++e) {
                    acc[1 + e] += w * a[e];
                    acc[4 + e] += w * b[e];
#pragma unroll
                    for (int f = 0; f < 3; ++f) acc[7 + 3 * e + f] += (w * a[e]) * b[f];
                }
            }
        }
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            cnt += __shfl_xor_sync(BX_FULL, cnt, o);
#pragma unroll
            for (int e = 0; e < 16; ++e) acc[e] += __shfl_xor_sync(BX_FULL, acc[e], o);
        }
        if (lane == 0) {
            redc[warp] = cnt;
#pragma unroll
            for (int e = 0; e < 16; ++e) red[warp][e] = acc[e];
        }
        __syncthreads();
        if (tid == 0) {
            int c = 0;
            for (int w = 0; w < 8; ++w) c += redc[w];
            s_cnt = c;
        }
        __syncthreads();
        const int total = s_cnt;
        if (total == prev) break;   // uniform: every thread reads the same s_cnt
        prev = total;
        if (total == 0) break;
        if (tid == 0) {
            double sum[16];
            for (int e = 0; e < 16; ++e) {
                double v = 0.0;
                for (int w = 0; w < 8; ++w) v += red[w][e];
                sum[e] = v;
            }
            const double sw = sum[0];
            double ca[3], cb[3], S[3][3];
            for (int e = 0; e < 3; ++e) { ca[e] = sum[1 + e] / sw; cb[e] = sum[4 + e] / sw; }
            // S = sum w (a-ca)(b-cb)^T = sum w a b^T - sw ca cb^T
            for (int e = 0; e < 3; ++e)
                for (int f = 0; f < 3; ++f) S[e][f] = sum[7 + 3 * e + f] - (sw * ca[e]) * cb[f];
            double Td[16];
            horn_from_S(S, ca, cb, Td);
            for (int e = 0; e < 16; ++e) sT[e] = (float)Td[e];
        }
        __syncthreads();
    }
    __syncthreads();
    if (tid < 16) T_out[tid] = sT[tid];
    if (tid == 0 && d_rounds) *d_rounds = r;
}

// early-exit decision of the multi-scale pair (PoseEstimator.compute_confidence_score): the scale-0 RANSAC result decides on
// the device whether the later scales run, so the pair is enqueued (and captured) without a host read
constexpr int GATE_MAXN = 32;
struct GateCaps { int cap[GATE_MAXN]; };
__global__ void early_exit_gate_kernel(const RansacResult *__restrict__ res, int min_inliers, int n, GateCaps caps,
                                       int *__restrict__ counts, int num_scales, double *__restrict__ scales_used) {
    const bool stop = res->num_inliers >= min_inliers;
    const int i = threadIdx.x;
    if (i < n) counts[i] = stop ? 0 : caps.cap[i];
    if (i == 0 && scales_used) *scales_used = stop ? 1.0 : (double)num_scales;
}

}  // namespace

BX_API int bx_early_exit_gate(const void *result, int min_inliers, int n, const int32_t *h_caps, int32_t *d_counts, int num_scales,
                              double *d_scales_used, void *stream) {
    BX_REQUIRE(result && (n == 0 || (h_caps && d_counts)), "bx_early_exit_gate: null pointer");
    BX_REQUIRE(n >= 0 && n <= GATE_MAXN && num_scales >= 1, "bx_early_exit_gate: 0 <= n <= %d counts, num_scales >= 1", GATE_MAXN);
    GateCaps caps = {};
    for (int i = 0; i < n; ++i) caps.cap[i] = h_caps[i];
    early_exit_gate_kernel<<<1, 32, 0, bx_stream(stream)>>>(static_cast<const RansacResult *>(result), min_inliers, n, caps, d_counts,
                                                           num_scales, d_scales_used);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int64_t bx_ransac_workspace_bytes(int max_iter) {
    (void)max_iter;
    // state + per-chunk: pass_itr (int), pass_T (12 double), rec_good (int), rec_rmse (double)
    return 256 + (int64_t)CHUNK * (4 + 96 + 4 + 8) + 64;
}

BX_API int bx_ransac(const float *ss, const float *tt, const int32_t *inlier_ind, const int32_t *d_I, int maxI,
                     double dist_th, double similar_th, double confidence, int max_iter, uint64_t seed, void *workspace,
                     void *result, void *stream) {
    BX_REQUIRE(ss && tt && inlier_ind && d_I && workspace && result, "bx_ransac: null pointer");
    BX_REQUIRE(max_iter >= 0 && dist_th > 0.0 && maxI >= 0, "bx_ransac: bad parameters");
    BX_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15) == 0 && (reinterpret_cast<uintptr_t>(result) & 7) == 0,
               "bx_ransac: workspace/result alignment");
    cudaStream_t st = bx_stream(stream);
    unsigned char *ws = static_cast<unsigned char *>(workspace);
    RansacState *state = reinterpret_cast<RansacState *>(ws);
    double *pass_T = reinterpret_cast<double *>(ws + 256);
    double *rec_rmse = pass_T + (size_t)CHUNK * 12;
    int *pass_itr = reinterpret_cast<int *>(rec_rmse + CHUNK);
    int *rec_good = pass_itr + CHUNK;
    RansacResult *res = static_cast<RansacResult *>(result);
    ransac_init_kernel<<<1, 32, 0, st>>>(state, max_iter);
    BX_LAUNCH_CHECK();
    const uint32_t k0 = (uint32_t)(seed & 0xffffffffu), k1 = (uint32_t)(seed >> 32);
    const int nchunks = max_iter > 0 ? (max_iter + CHUNK - 1) / CHUNK : 1;
    for (int c = 0; c < nchunks; ++c) {
        const int itr0 = c * CHUNK;
        const int itr1 = (itr0 + CHUNK < max_iter) ? itr0 + CHUNK : max_iter;
        if (itr1 > itr0) {
            ransac_hyp_kernel<<<(itr1 - itr0 + 127) / 128, 128, 0, st>>>(ss, tt, inlier_ind, d_I, dist_th, similar_th, itr0,
                                                                         itr1, k0, k1, state, pass_itr, pass_T, rec_good);
            BX_LAUNCH_CHECK();
            ransac_verify_kernel<<<(itr1 - itr0 + 127) / 128, 128, 0, st>>>(ss, tt, inlier_ind, d_I, dist_th, itr0, state,
                                                                            pass_itr, pass_T, rec_good, rec_rmse);
            BX_LAUNCH_CHECK();
        }
        ransac_scan_kernel<<<1, 32, 0, st>>>(d_I, confidence, itr0, itr1, max_iter, state, pass_itr, pass_T, rec_good,
                                             rec_rmse, res, c == nchunks - 1 ? 1 : 0);
        BX_LAUNCH_CHECK();
    }
    return BX_OK;
}

BX_API int bx_refine(const float *ss, const float *tt, const int32_t *d_n, int maxn, const double *T_in, float dist_th,
                     float *T_out, int32_t *d_rounds, void *stream) {
    BX_REQUIRE(ss && tt && d_n && T_in && T_out, "bx_refine: null pointer");
    BX_REQUIRE(maxn >= 0 && dist_th > 0.0f, "bx_refine: bad parameters");
    refine_kernel<<<1, 256, 0, bx_stream(stream)>>>(ss, tt, d_n, T_in, dist_th, T_out, d_rounds);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
