// bx_svd3.cuh -- the fp64 3x3 singular value decomposition of bx_svd3 (bx_svd.cu), shared with the ICP solve (bx_icp.cu).
//
// One-sided (Hestenes) Jacobi rotates the columns of W = A until they are mutually orthogonal, accumulating the rotations
// in V, so that W = A V = U diag(S) with S_i = |w_i|.  The columns are sorted by S descending and U is completed to an
// orthonormal basis where a singular value vanishes (u_1 by Gram-Schmidt against u_0, u_2 = +-(u_0 x u_1) with the sign of
// w_2), so U and V are orthonormal for every input: rank deficient, zero, isotropic or with a negative determinant.  A is
// not assumed symmetric.  Signs of singular vectors are unspecified, as in cuSOLVER.
#pragma once
#include "bx_common.cuh"

namespace {

constexpr int SVD_MAX_SWEEPS = 12;

__device__ __forceinline__ double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// unit vector orthogonal to the unit vector u: e_k (the axis least aligned with u) minus its projection, twice
__device__ __forceinline__ void orth_complement(const double *u, double *out) {
    const double ax = fabs(u[0]), ay = fabs(u[1]), az = fabs(u[2]);
    const int k = (ax <= ay && ax <= az) ? 0 : (ay <= az ? 1 : 2);
    out[0] = k == 0 ? 1.0 : 0.0;
    out[1] = k == 1 ? 1.0 : 0.0;
    out[2] = k == 2 ? 1.0 : 0.0;
    for (int it = 0; it < 2; ++it) {
        const double p = dot3(u, out);
        for (int r = 0; r < 3; ++r) out[r] -= p * u[r];
    }
    const double n = sqrt(dot3(out, out));
    for (int r = 0; r < 3; ++r) out[r] /= n;
}

// On entry w[j][r] = A[r][j] (column j of A).  On exit sv[0] >= sv[1] >= sv[2] >= 0, u[j] / v[j] = column j of U / V and
// A = U diag(sv) V^T; w is overwritten (column j of A V).
__device__ __forceinline__ void bx_svd3_fp64(double (&w)[3][3], double (&u)[3][3], double (&sv)[3], double (&v)[3][3]) {
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int r = 0; r < 3; ++r) v[j][r] = (r == j) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < SVD_MAX_SWEEPS; ++sweep) {
        bool rotated = false;
#pragma unroll
        for (int pq = 0; pq < 3; ++pq) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
            const double alpha = dot3(w[p], w[p]), beta = dot3(w[q], w[q]), gamma = dot3(w[p], w[q]);
            if (gamma == 0.0 || fabs(gamma) <= 1e-15 * sqrt(alpha * beta)) continue;
            rotated = true;
            const double zeta = (beta - alpha) / (2.0 * gamma);
            const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
            const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const double wp = w[p][r], wq = w[q][r];
                w[p][r] = c * wp - s * wq;
                w[q][r] = s * wp + c * wq;
                const double vp = v[p][r], vq = v[q][r];
                v[p][r] = c * vp - s * vq;
                v[q][r] = s * vp + c * vq;
            }
        }
        if (!rotated) break;
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) sv[j] = sqrt(dot3(w[j], w[j]));
    // three-element sort, descending (stable: equal values keep their column order); constant indices keep it in registers
    auto order = [&](int a, int b) {
        if (sv[a] < sv[b]) {
            double x = sv[a]; sv[a] = sv[b]; sv[b] = x;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                x = w[a][r]; w[a][r] = w[b][r]; w[b][r] = x;
                x = v[a][r]; v[a][r] = v[b][r]; v[b][r] = x;
            }
        }
    };
    order(0, 1);
    order(1, 2);
    order(0, 1);
    const double *w1 = w[1], *w2 = w[2];
    if (sv[0] > 0.0) {
        for (int r = 0; r < 3; ++r) u[0][r] = w[0][r] / sv[0];
    } else {
        u[0][0] = 1.0; u[0][1] = 0.0; u[0][2] = 0.0;
    }
    // u_1: w_1 orthogonalised against u_0 (twice), or any unit vector orthogonal to u_0 when nothing is left of w_1
    for (int r = 0; r < 3; ++r) u[1][r] = w1[r];
    for (int it = 0; it < 2; ++it) {
        const double p = dot3(u[0], u[1]);
        for (int r = 0; r < 3; ++r) u[1][r] -= p * u[0][r];
    }
    const double n1 = sqrt(dot3(u[1], u[1]));
    if (n1 > 1e-300) {
        for (int r = 0; r < 3; ++r) u[1][r] /= n1;
    } else {
        orth_complement(u[0], u[1]);
    }
    u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
    u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
    u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
    if (dot3(u[2], w2) < 0.0)
        for (int r = 0; r < 3; ++r) u[2][r] = -u[2][r];
}

}  // namespace
