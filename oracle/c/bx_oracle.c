/*
 * bx_oracle.c -- CPU restatement (ORACLE) of the BUFFER-X per-pair registration hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product (buffer-x_b200/) may import, link or
 * execute this file; it is the checker that tests/, __graft_entry__.smoke() and the
 * cpu_baseline / --impl reference legs of bench.py compare the CUDA path against.
 *
 * PARITY STATUS: "parity unpinned" by the reference's own tests -- the reference ships no
 * tests, fixtures or golden vectors (SURVEY.md section 4), and four of the stages below live
 * in third-party packages whose sources are NOT under /root/reference:
 *     pointnet2_ops (LucasColas/Pointnet2_PyTorch fork of erikwijmans/Pointnet2_PyTorch,
 *                    un-pinned HEAD, /root/reference/scripts/install.sh:211-212)
 *     knn_cuda 0.2  (install.sh:214), torch_batch_svd (HEAD, install.sh:218-219),
 *     open3d==0.18.0 (/root/reference/requirements/base.txt)
 * For those the published algorithm is restated and parity is anchored on the reference's
 * call sites (cited per function).  The stages whose code IS importable from /root/reference
 * (radius estimation, conv stacks, cost volume, refinement, Rodrigues, voxel table, SO(2)
 * de-rotation) are pinned by oracle/ref_check.py, which runs the reference's own Python on
 * CPU in the build container and writes tests/golden/ (see oracle/README.md).
 *
 * Arithmetic contract (mirrored instruction-for-instruction by the CUDA kernels, which are
 * compiled with -fmad=false): every fp32/fp64 expression below is evaluated exactly as
 * parenthesised, with IEEE round-to-nearest +,-,*,/,sqrt and NO fused multiply-add.  Build
 * with: gcc -O2 -ffp-contract=off -fno-fast-math (see oracle/build.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define BX_EXPORT __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * a1. Farthest point sampling.
 * Call sites: /root/reference/models/BUFFERX.py:286-287, 338-339
 *             (pnt2.furthest_point_sample(xyz[None], npoint)).
 * Algorithm (pointnet2_ops sampling_gpu.cu, furthest_point_sampling_kernel; not vendored):
 *   idx[0] = 0; temp[k] = 1e10; each step: for every k with mag = x*x+y*y+z*z > 1e-3 (the
 *   comparison is done in double, the literal is a double): d = dx*dx+dy*dy+dz*dz,
 *   temp[k] = min(d, temp[k]); thread t of a block of `bs` threads keeps the FIRST strict
 *   maximum over k = t, t+bs, ...; every step of the shared-memory tree (stride bs/2 ... 1) keeps
 *   the lower position on ties, so across slots the winner is the one whose BIT-REVERSED slot
 *   index is smallest (the stride-1 step decides on bit 0 last, i.e. with highest priority).
 *   Hence the winner maximises (value, -bitrev(k mod bs), -k).  bs = min(512, 2^floor(log2 N)).
 *   A thread without candidates contributes (-1, index 0).
 * ------------------------------------------------------------------------------------------ */
static int fps_block_size(int n) {
    int p = 1;
    while ((p << 1) <= n) p <<= 1;
    if (p > 512) p = 512;
    if (p < 1) p = 1;
    return p;
}

static int bitrev(int t, int bits) {
    int r = 0;
    for (int b = 0; b < bits; ++b) r |= ((t >> b) & 1) << (bits - 1 - b);
    return r;
}

BX_EXPORT int bxo_fps(const float *xyz, int n, int m, int32_t *idx) {
    if (m <= 0) return 0;
    if (n <= 0) return -1;
    const int bs = fps_block_size(n);
    int bits = 0;
    while ((1 << bits) < bs) ++bits;
    float *temp = (float *)malloc(sizeof(float) * (size_t)n);
    unsigned char *valid = (unsigned char *)malloc((size_t)n);
    if (!temp || !valid) return -2;
    for (int k = 0; k < n; ++k) {
        const float x = xyz[3 * k], y = xyz[3 * k + 1], z = xyz[3 * k + 2];
        const float mag = ((x * x) + (y * y)) + (z * z);
        valid[k] = ((double)mag <= 1e-3) ? 0 : 1;
        temp[k] = 1e10f;
    }
    int old = 0;
    idx[0] = 0;
    for (int j = 1; j < m; ++j) {
        const float x1 = xyz[3 * old], y1 = xyz[3 * old + 1], z1 = xyz[3 * old + 2];
        float best = -1.0f;
        int besti = 0, bestt = 0x7fffffff;
        for (int k = 0; k < n; ++k) {
            if (!valid[k]) continue;
            const float dx = xyz[3 * k] - x1, dy = xyz[3 * k + 1] - y1, dz = xyz[3 * k + 2] - z1;
            const float d = ((dx * dx) + (dy * dy)) + (dz * dz);
            const float d2 = d < temp[k] ? d : temp[k]; /* min(d, temp) */
            temp[k] = d2;
            const int t = bitrev(k % bs, bits);
            /* k ascending: within one thread slot the first strict max wins; across slots the
             * smaller bit-reversed slot wins on ties */
            if (d2 > best || (d2 == best && t < bestt)) {
                best = d2;
                besti = k;
                bestt = t;
            }
        }
        old = besti;
        idx[j] = old;
    }
    free(temp);
    free(valid);
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * a3 / a6. Ordered ball query (pointnet2_ops ball_query_gpu.cu, query_ball_point_kernel).
 * Call sites: /root/reference/models/patch_embedder.py:99 (patches),
 *             /root/reference/utils/common.py:442 (voxel query inside sphere_query).
 *   r2 = radius*radius (fp32); scan supports in index order, keep the first `nsample` with
 *   d2 = (qx-x)^2+(qy-y)^2+(qz-z)^2 < r2 (strict); on the first hit fill every slot with it;
 *   the output is zero-initialised, so a query without hit yields an all-zero row.
 * `cnt` (optional) receives the number of genuine hits (<= nsample).
 * ------------------------------------------------------------------------------------------ */
BX_EXPORT int bxo_ball_query(const float *xyz, int n, const float *qry, int m, float radius, int nsample,
                             int32_t *idx, int32_t *cnt) {
    const float r2 = radius * radius;
#pragma omp parallel for schedule(static)
    for (int j = 0; j < m; ++j) {
        const float qx = qry[3 * j], qy = qry[3 * j + 1], qz = qry[3 * j + 2];
        int32_t *row = idx + (size_t)j * nsample;
        for (int l = 0; l < nsample; ++l) row[l] = 0;
        int c = 0;
        for (int k = 0; k < n && c < nsample; ++k) {
            const float dx = qx - xyz[3 * k], dy = qy - xyz[3 * k + 1], dz = qz - xyz[3 * k + 2];
            const float d2 = ((dx * dx) + (dy * dy)) + (dz * dz);
            if (d2 < r2) {
                if (c == 0)
                    for (int l = 0; l < nsample; ++l) row[l] = k;
                row[c] = k;
                ++c;
            }
        }
        if (cnt) cnt[j] = c;
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * a3. MiniSpinNet.select_patches -- /root/reference/models/patch_embedder.py:92-120.
 *   pts_perm = pts[perm]; idx = ball_query(r, P, pts_perm, kpts); patch = pts_perm[idx];
 *   every slot s>0 whose index equals slot 0's (padding) and ALWAYS slot P-1 is replaced by
 *   the key-point itself (:105-111).
 * Outputs: idx int32 [K,P] (indices into the PERMUTED cloud), patches fp32 [K,P,3].
 * ------------------------------------------------------------------------------------------ */
BX_EXPORT int bxo_select_patches(const float *pts, int n, const int32_t *perm, const float *kpts, int K, float radius,
                                 int P, int32_t *idx, float *patches) {
    float *pp = (float *)malloc(sizeof(float) * 3 * (size_t)n);
    if (!pp) return -2;
    for (int i = 0; i < n; ++i) {
        const int s = perm ? perm[i] : i;
        pp[3 * i] = pts[3 * s];
        pp[3 * i + 1] = pts[3 * s + 1];
        pp[3 * i + 2] = pts[3 * s + 2];
    }
    bxo_ball_query(pp, n, kpts, K, radius, P, idx, NULL);
#pragma omp parallel for schedule(static)
    for (int k = 0; k < K; ++k) {
        const int32_t *row = idx + (size_t)k * P;
        float *out = patches + (size_t)k * P * 3;
        for (int s = 0; s < P; ++s) {
            const int is_center = (s == P - 1) || (s > 0 && row[s] == row[0]);
            const float *src = is_center ? (kpts + 3 * k) : (pp + 3 * (size_t)row[s]);
            out[3 * s] = src[0];
            out[3 * s + 1] = src[1];
            out[3 * s + 2] = src[2];
        }
    }
    free(pp);
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * a4 + a5. Local reference frame + normalisation.
 * /root/reference/models/patch_embedder.py:122-148 (axis_align), :167-170 (normalize),
 * /root/reference/utils/common.py:709-726 (cal_Z_axis), :501-525 (RodsRotatFormula).
 *   delta = patch - patch[P-1]; (not aligned) cov = delta^T delta; z = eigenvector of the
 *   smallest eigenvalue (reference: last left-singular vector from torch_batch_svd, a cuSOLVER
 *   Jacobi solver; here: cyclic Jacobi in fp64, 8 fixed sweeps); flip so that z . centre <= 0;
 *   z /= |z|; R = Rodrigues(z -> e_z); delta <- R delta; rand_axis = normalise(z x e_z);
 *   the matrix handed back by the reference ("R") is the TRANSPOSE of that rotation.
 *   (aligned) R = I, rand_axis = e_x.   Then delta /= des_r.
 * Frozen summation order of cov: 32 lanes; lane l adds its products for s = l, l+32, ...
 * sequentially starting from +0, then a 5-step xor butterfly (16,8,4,2,1).
 * Rodrigues uses the well-conditioned identities cos(t) = z_z/|z|, sin(t) = |z x e_z|/|z|
 * instead of acos/sin/cos (documented deviation: ulp-level except where the reference's
 * acos is itself ill-conditioned, |z_z| -> 1).
 * Outputs: delta [K,P,3] (normalised), Rt [K,3,3] (the reference's "R"), rand_axis [K,3].
 * ------------------------------------------------------------------------------------------ */
static void jacobi3(double A[3][3], double V[3][3]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
    static const int PQ[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    for (int sweep = 0; sweep < 8; ++sweep) {
        for (int e = 0; e < 3; ++e) {
            const int p = PQ[e][0], q = PQ[e][1];
            const double apq = A[p][q];
            if (apq == 0.0) continue;
            const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
            const double at = fabs(theta);
            double t = 1.0 / (at + sqrt((theta * theta) + 1.0));
            if (theta < 0.0) t = -t;
            const double c = 1.0 / sqrt((t * t) + 1.0);
            const double s = t * c;
            /* A <- J^T A J */
            const double app = A[p][p], aqq = A[q][q];
            A[p][p] = app - (t * apq);
            A[q][q] = aqq + (t * apq);
            A[p][q] = 0.0;
            A[q][p] = 0.0;
            const int r = 3 - p - q;
            const double arp = A[r][p], arq = A[r][q];
            A[r][p] = (c * arp) - (s * arq);
            A[p][r] = A[r][p];
            A[r][q] = (s * arp) + (c * arq);
            A[q][r] = A[r][q];
            for (int k = 0; k < 3; ++k) {
                const double vkp = V[k][p], vkq = V[k][q];
                V[k][p] = (c * vkp) - (s * vkq);
                V[k][q] = (s * vkp) + (c * vkq);
            }
        }
    }
}

BX_EXPORT int bxo_lrf(const float *patches, int K, int P, float des_r, int flags, float *delta, float *Rt,
                      float *rand_axis, const float *z_override, float *z_out) {
    /* flags: bit 0 = is_aligned_to_global_z; bit 1 = well-conditioned Rodrigues (cos = z_z/|z|, sin = |z x e_z|/|z|,
     * NOT the reference's formula; kept for the sensitivity report of oracle/ref_check.py).
     * z_override [K,3] (optional): the disambiguated, normalised z axes to use instead of this function's own
     * covariance + Jacobi result -- ref_check.py feeds the reference run's axes through it so that everything
     * downstream of the (BLAS-order dependent) covariance sum can be compared exactly.  z_out [K,3] (optional). */
    const int aligned = flags & 1, stable = flags & 2;
#pragma omp parallel for schedule(static)
    for (int k = 0; k < K; ++k) {
        const float *pt = patches + (size_t)k * P * 3;
        float *dl = delta + (size_t)k * P * 3;
        const float cx = pt[3 * (P - 1)], cy = pt[3 * (P - 1) + 1], cz = pt[3 * (P - 1) + 2];
        for (int s = 0; s < P; ++s) {
            dl[3 * s] = pt[3 * s] - cx;
            dl[3 * s + 1] = pt[3 * s + 1] - cy;
            dl[3 * s + 2] = pt[3 * s + 2] - cz;
        }
        float R[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}; /* rotation applied to delta */
        float ra[3] = {1.0f, 0.0f, 0.0f};
        if (!aligned) {
            float lane[6][32];
            for (int e = 0; e < 6; ++e)
                for (int l = 0; l < 32; ++l) lane[e][l] = 0.0f;
            for (int l = 0; l < 32; ++l)
                for (int s = l; s < P; s += 32) {
                    const float x = dl[3 * s], y = dl[3 * s + 1], z = dl[3 * s + 2];
                    lane[0][l] = lane[0][l] + (x * x);
                    lane[1][l] = lane[1][l] + (x * y);
                    lane[2][l] = lane[2][l] + (x * z);
                    lane[3][l] = lane[3][l] + (y * y);
                    lane[4][l] = lane[4][l] + (y * z);
                    lane[5][l] = lane[5][l] + (z * z);
                }
            for (int e = 0; e < 6; ++e)
                for (int off = 16; off >= 1; off >>= 1) {
                    float nw[32];
                    for (int l = 0; l < 32; ++l) nw[l] = lane[e][l] + lane[e][l ^ off];
                    memcpy(lane[e], nw, sizeof(nw));
                }
            double A[3][3], V[3][3];
            A[0][0] = lane[0][0]; A[0][1] = lane[1][0]; A[0][2] = lane[2][0];
            A[1][0] = lane[1][0]; A[1][1] = lane[3][0]; A[1][2] = lane[4][0];
            A[2][0] = lane[2][0]; A[2][1] = lane[4][0]; A[2][2] = lane[5][0];
            jacobi3(A, V);
            int m = 0; /* column of the smallest eigenvalue; first minimum wins */
            if (A[1][1] < A[m][m]) m = 1;
            if (A[2][2] < A[m][m]) m = 2;
            float z0 = (float)V[0][m], z1 = (float)V[1][m], z2 = (float)V[2][m];
            /* cal_Z_axis: mask = (sum(-Z * ref_point) < 0) -> Z = -Z */
            const float sgn = (((-z0) * cx) + ((-z1) * cy)) + ((-z2) * cz);
            if (sgn < 0.0f) { z0 = -z0; z1 = -z1; z2 = -z2; }
            const float nz = sqrtf(((z0 * z0) + (z1 * z1)) + (z2 * z2));
            z0 = z0 / nz; z1 = z1 / nz; z2 = z2 / nz;
            if (z_override) { z0 = z_override[3 * k]; z1 = z_override[3 * k + 1]; z2 = z_override[3 * k + 2]; }
            if (z_out) { z_out[3 * k] = z0; z_out[3 * k + 1] = z1; z_out[3 * k + 2] = z2; }
            /* Rodrigues z -> e_z */
            const float n = sqrtf(((z0 * z0) + (z1 * z1)) + (z2 * z2));
            const float sn = sqrtf((z0 * z0) + (z1 * z1));
            float ct = z2 / n, st = sn / n;
            if (!stable) {
                /* RodsRotatFormula literally (utils/common.py:506, 522-523): theta = acos(cosine_similarity(z, e_z))
                 * in fp32, then sin(theta), cos(theta) in fp32.  "fp32" = the correctly rounded value (fp64 libm
                 * rounded once), the one definition a CPU and a GPU can both reproduce bit for bit; torch's own
                 * acos/sin/cos (Sleef on CPU, CUDA libm on the GPU) are each within 1 ulp of it. */
                const float theta = (float)acos((double)ct);
                st = (float)sin((double)theta);
                ct = (float)cos((double)theta);
            }
            const float den = sn > 1e-12f ? sn : 1e-12f;
            const float c0 = z1 / den, c1 = (-z0) / den; /* axis = normalise(z x e_z) = (z1,-z0,0)/|.| */
            const float kk = 1.0f - ct;
            R[0][0] = 1.0f - (kk * (c1 * c1)); R[0][1] = kk * (c0 * c1);          R[0][2] = st * c1;
            R[1][0] = kk * (c0 * c1);          R[1][1] = 1.0f - (kk * (c0 * c0)); R[1][2] = -(st * c0);
            R[2][0] = -(st * c1);              R[2][1] = st * c0;                 R[2][2] = 1.0f - (kk * ((c0 * c0) + (c1 * c1)));
            ra[0] = c0; ra[1] = c1; ra[2] = 0.0f;
        }
        for (int s = 0; s < P; ++s) {
            const float x = dl[3 * s], y = dl[3 * s + 1], z = dl[3 * s + 2];
            float o[3];
            for (int j = 0; j < 3; ++j) o[j] = aligned ? (j == 0 ? x : (j == 1 ? y : z)) : (((R[j][0] * x) + (R[j][1] * y)) + (R[j][2] * z));
            dl[3 * s] = o[0] / des_r;
            dl[3 * s + 1] = o[1] / des_r;
            dl[3 * s + 2] = o[2] / des_r;
        }
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) Rt[(size_t)k * 9 + 3 * i + j] = R[j][i]; /* transpose */
        rand_axis[3 * k] = ra[0]; rand_axis[3 * k + 1] = ra[1]; rand_axis[3 * k + 2] = ra[2];
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * a6. Spherical-voxel point transformer.
 * /root/reference/models/patch_embedder.py:150-165 (SPT), /root/reference/utils/common.py:431-469
 * (sphere_query), :472-498 (var_to_invar).
 *   For each patch and each of the V voxel centres: ordered ball query (first `nv` in index
 *   order, radius voxel_r) over the patch's P points; padding slots (index equal to slot 0's,
 *   slot 0 excluded) are zeroed; slot 0 is ALSO zeroed when its index is 0 (common.py:447-449,
 *   fires both for "no hit" and for a genuine first hit at patch index 0); then every point of
 *   azimuth bin a is rotated by Rz(-a*2pi/azi_n): x' = x*c + y*(-s), y' = x*s + y*c, z' = z
 *   with (c,s) the fp32 casts of the fp64 cos/sin (table built on the host like common.py:483-491).
 * voxels: [V,3] fp32 table (layout [rad,ele,azi], azimuth fastest); rot: [azi_n,2] (c,s).
 * Outputs: out [K,V,nv,3] fp32; vidx int32 [K,V,nv] raw ball-query indices (for bit parity).
 * ------------------------------------------------------------------------------------------ */
BX_EXPORT int bxo_spt(const float *delta, int K, int P, const float *voxels, int V, int azi_n, const float *rot,
                      float voxel_r, int nv, float *out, int32_t *vidx) {
    const float r2 = voxel_r * voxel_r;
#pragma omp parallel for schedule(dynamic, 8)
    for (int k = 0; k < K; ++k) {
        const float *dl = delta + (size_t)k * P * 3;
        for (int v = 0; v < V; ++v) {
            int32_t row[64];
            for (int l = 0; l < nv; ++l) row[l] = 0;
            const float qx = voxels[3 * v], qy = voxels[3 * v + 1], qz = voxels[3 * v + 2];
            int c = 0;
            for (int s = 0; s < P && c < nv; ++s) {
                const float dx = qx - dl[3 * s], dy = qy - dl[3 * s + 1], dz = qz - dl[3 * s + 2];
                const float d2 = ((dx * dx) + (dy * dy)) + (dz * dz);
                if (d2 < r2) {
                    if (c == 0)
                        for (int l = 0; l < nv; ++l) row[l] = s;
                    row[c] = s;
                    ++c;
                }
            }
            const int a = v % azi_n;
            const float cs = rot[2 * a], sn = rot[2 * a + 1];
            for (int l = 0; l < nv; ++l) {
                const int zero = (l == 0) ? (row[0] == 0) : (row[l] == row[0]);
                float *o = out + (((size_t)k * V + v) * nv + l) * 3;
                if (vidx) vidx[((size_t)k * V + v) * nv + l] = row[l];
                if (zero) {
                    o[0] = 0.0f; o[1] = 0.0f; o[2] = 0.0f;
                } else {
                    const float x = dl[3 * row[l]], y = dl[3 * row[l] + 1], z = dl[3 * row[l] + 2];
                    o[0] = (x * cs) + (y * (-sn));
                    o[1] = (x * sn) + (y * cs);
                    o[2] = z;
                }
            }
        }
    }
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * a10. Mutual nearest-neighbour matching.
 * /root/reference/models/BUFFERX.py:469-496 (mutual_matching) -> KNN(k=1) of knn_cuda 0.2
 * (brute force, squared L2 accumulated over the feature dimension in order, first minimum wins).
 *   d(i,j) = sum_c (a_ic - b_jc)^2 sequential over c (no FMA); sNN[i] = argmin_j, tNN[j] = argmin_i;
 *   keep i with tNN[sNN[i]] == i; s_mids ascending, t_mids = sNN[s_mids].
 * Returns M; fills s_mids/t_mids (capacity Ka), and optionally sNN [Ka], tNN [Kb].
 * ------------------------------------------------------------------------------------------ */
BX_EXPORT int bxo_mutual_nn(const float *a, int Ka, const float *b, int Kb, int C, int32_t *s_mids, int32_t *t_mids,
                            int32_t *snn_out, int32_t *tnn_out) {
    int32_t *snn = (int32_t *)malloc(sizeof(int32_t) * (size_t)(Ka > 0 ? Ka : 1));
    int32_t *tnn = (int32_t *)malloc(sizeof(int32_t) * (size_t)(Kb > 0 ? Kb : 1));
    if (!snn || !tnn) return -2;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < Ka; ++i) {
        float best = INFINITY;
        int bj = 0;
        for (int j = 0; j < Kb; ++j) {
            float acc = 0.0f;
            for (int c = 0; c < C; ++c) {
                const float t = a[(size_t)i * C + c] - b[(size_t)j * C + c];
                acc = acc + (t * t);
            }
            if (acc < best) { best = acc; bj = j; }
        }
        snn[i] = bj;
    }
#pragma omp parallel for schedule(static)
    for (int j = 0; j < Kb; ++j) {
        float best = INFINITY;
        int bi = 0;
        for (int i = 0; i < Ka; ++i) {
            float acc = 0.0f;
            for (int c = 0; c < C; ++c) {
                const float t = b[(size_t)j * C + c] - a[(size_t)i * C + c];
                acc = acc + (t * t);
            }
            if (acc < best) { best = acc; bi = i; }
        }
        tnn[j] = bi;
    }
    int M = 0;
    for (int i = 0; i < Ka; ++i)
        if (Kb > 0 && tnn[snn[i]] == i) {
            s_mids[M] = i;
            t_mids[M] = snn[i];
            ++M;
        }
    if (snn_out) memcpy(snn_out, snn, sizeof(int32_t) * (size_t)Ka);
    if (tnn_out) memcpy(tnn_out, tnn, sizeof(int32_t) * (size_t)Kb);
    free(snn);
    free(tnn);
    return M;
}

/* ------------------------------------------------------------------------------------------
 * a2. Density-aware radius estimation -- /root/reference/models/BUFFERX.py:610-696.
 *   d2 = (|k|^2 + |p|^2) - 2*(k.p) in fp32 (squared_cdist :621-624; frozen order: norms and dot
 *   as ((x*x)+(y*y))+(z*z), no FMA), keep d2 <= max_r^2 (:672), then for each threshold a
 *   bisection on r in [0, max_r] (:677-692) with pct = float32(count)/float32(N*Kr)*100 (fp32,
 *   as torch evaluates it), count = #{d2 < float32(r*r)}; stop when high-low <= 1e-3 or
 *   |pct - thr| <= tolerance; result round(r, 2) (:694).
 * Because every probed r is max_r*m/8192 (m integer), the counts are served from a cumulative
 * histogram over those 8192 candidate radii -- identical counts to the reference's masks.
 * hist_out (optional, 8193 int64): hist[m] = #{d2 : d2 <= 25 and d2 < float32((5m/8192)^2)}.
 * `num_pts_denominator` is the ORIGINAL cloud size (the reference keeps it when sub-sampling).
 * ------------------------------------------------------------------------------------------ */
BX_EXPORT int bxo_radius_hist(const float *kpts, int Kr, const float *pts, int n, int64_t *cum /*8193*/) {
    const double max_r = 5.0;
    float thr[8193];
    for (int m = 0; m <= 8192; ++m) {
        const double r = max_r * (double)m / 8192.0;
        thr[m] = (float)(r * r);
    }
    const float cap = (float)(max_r * max_r);
    int64_t *hist = (int64_t *)calloc(8194, sizeof(int64_t));
    if (!hist) return -2;
#pragma omp parallel
    {
        int64_t *loc = (int64_t *)calloc(8194, sizeof(int64_t));
#pragma omp for schedule(static)
        for (int i = 0; i < Kr; ++i) {
            const float kx = kpts[3 * i], ky = kpts[3 * i + 1], kz = kpts[3 * i + 2];
            const float k2 = ((kx * kx) + (ky * ky)) + (kz * kz);
            for (int j = 0; j < n; ++j) {
                const float px = pts[3 * j], py = pts[3 * j + 1], pz = pts[3 * j + 2];
                const float p2 = ((px * px) + (py * py)) + (pz * pz);
                const float dot = ((kx * px) + (ky * py)) + (kz * pz);
                const float d2 = (k2 + p2) - (2.0f * dot);
                if (!(d2 <= cap)) continue;
                /* smallest m with d2 < thr[m]; thr is non-decreasing */
                int lo = 0, hi = 8193; /* answer in [0, 8193]; 8193 = not below any threshold */
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (d2 < thr[mid]) hi = mid; else lo = mid + 1;
                }
                loc[lo] += 1;
            }
        }
#pragma omp critical
        for (int m = 0; m < 8194; ++m) hist[m] += loc[m];
        free(loc);
    }
    int64_t run = 0;
    for (int m = 0; m <= 8192; ++m) {
        run += hist[m];
        cum[m] = run; /* #{d2 < thr[m]} */
    }
    free(hist);
    return 0;
}

/* bisection on the cumulative histogram; returns m (r = 5*m/8192) or 0 if the loop never ran */
BX_EXPORT int bxo_radius_bisect(const int64_t *cum, int64_t denom, double threshold, double tolerance) {
    int lo = 0, hi = 8192, m = 0;
    /* high - low > 1e-3  <=>  5*(hi-lo)/8192 > 1e-3 */
    while (5.0 * (double)hi / 8192.0 - 5.0 * (double)lo / 8192.0 > 1e-3) {
        m = (lo + hi) / 2; /* (low+high)/2 is exact: hi-lo is a power of two >= 2 here */
        const float pct = ((float)cum[m] / (float)denom) * 100.0f;
        const double p = (double)pct;
        if (p < threshold - tolerance) lo = m;
        else if (p > threshold + tolerance) hi = m;
        else break;
    }
    return m;
}

/* ------------------------------------------------------------------------------------------
 * a13. Cross-scale consensus -- /root/reference/models/BUFFERX.py:404-417.
 *   hypothesis j transforms every accumulated source key-point i: q = R_j s_i + t_j;
 *   inlier iff |q - t_i| < |s_i| * pi/azi_n * inlier_th (fp32); best = first arg-max of counts.
 * Frozen order: q_c = ((R[c][0]*sx + R[c][1]*sy) + R[c][2]*sz) + t_c; |.| = sqrt((dx^2+dy^2)+dz^2);
 * thr_i = ((|s_i| * pi_f) / azi_n_f) * inlier_th_f.
 * Returns the number of inliers of the best hypothesis; inlier_ind ascending; best index in *best.
 * ------------------------------------------------------------------------------------------ */
BX_EXPORT int bxo_consensus(const float *ss, const float *tt, const float *R, const float *t, int Mc, int azi_n,
                            float inlier_th, int32_t *inlier_ind, int32_t *best, int32_t *counts_out) {
    if (Mc <= 0) { if (best) *best = 0; return 0; }
    float *thr = (float *)malloc(sizeof(float) * (size_t)Mc);
    int32_t *cnt = (int32_t *)malloc(sizeof(int32_t) * (size_t)Mc);
    const float pi_f = (float)3.14159265358979323846;
    for (int i = 0; i < Mc; ++i) {
        const float x = ss[3 * i], y = ss[3 * i + 1], z = ss[3 * i + 2];
        const float nrm = sqrtf(((x * x) + (y * y)) + (z * z));
        thr[i] = ((nrm * pi_f) / (float)azi_n) * inlier_th;
    }
#pragma omp parallel for schedule(static)
    for (int j = 0; j < Mc; ++j) {
        const float *Rj = R + 9 * (size_t)j, *tj = t + 3 * (size_t)j;
        int c = 0;
        for (int i = 0; i < Mc; ++i) {
            const float x = ss[3 * i], y = ss[3 * i + 1], z = ss[3 * i + 2];
            const float qx = (((Rj[0] * x) + (Rj[1] * y)) + (Rj[2] * z)) + tj[0];
            const float qy = (((Rj[3] * x) + (Rj[4] * y)) + (Rj[5] * z)) + tj[1];
            const float qz = (((Rj[6] * x) + (Rj[7] * y)) + (Rj[8] * z)) + tj[2];
            const float dx = qx - tt[3 * i], dy = qy - tt[3 * i + 1], dz = qz - tt[3 * i + 2];
            const float d = sqrtf(((dx * dx) + (dy * dy)) + (dz * dz));
            c += (d < thr[i]) ? 1 : 0;
        }
        cnt[j] = c;
    }
    int b = 0;
    for (int j = 1; j < Mc; ++j)
        if (cnt[j] > cnt[b]) b = j;
    int I = 0;
    {
        const float *Rj = R + 9 * (size_t)b, *tj = t + 3 * (size_t)b;
        for (int i = 0; i < Mc; ++i) {
            const float x = ss[3 * i], y = ss[3 * i + 1], z = ss[3 * i + 2];
            const float qx = (((Rj[0] * x) + (Rj[1] * y)) + (Rj[2] * z)) + tj[0];
            const float qy = (((Rj[3] * x) + (Rj[4] * y)) + (Rj[5] * z)) + tj[1];
            const float qz = (((Rj[6] * x) + (Rj[7] * y)) + (Rj[8] * z)) + tj[2];
            const float dx = qx - tt[3 * i], dy = qy - tt[3 * i + 1], dz = qz - tt[3 * i + 2];
            const float d = sqrtf(((dx * dx) + (dy * dy)) + (dz * dz));
            if (d < thr[i]) inlier_ind[I++] = i;
        }
    }
    if (best) *best = b;
    if (counts_out) memcpy(counts_out, cnt, sizeof(int32_t) * (size_t)Mc);
    free(thr);
    free(cnt);
    return I;
}

/* ------------------------------------------------------------------------------------------
 * a14. RANSAC on pre-filtered correspondences.
 * /root/reference/models/pose_estimator.py:84-117 -> Open3D 0.18.0
 * registration_ransac_based_on_correspondence (not vendored; algorithm of
 * cpp/open3d/pipelines/registration/Registration.cpp, RegistrationRANSACBasedOnCorrespondence):
 *   corr = {(k,k) : k in inlier_ind}; for itr < max_iter while itr < est_k:
 *     draw ransac_n=3 correspondences uniformly WITH replacement; T = least-squares rigid fit
 *     (TransformationEstimationPointToPoint(False) = Umeyama without scale, fp64);
 *     checkers: EdgeLength(similar_th): for every pair, reject if ds < dt*th or dt < ds*th;
 *               Distance(dist_th): reject if any |T s - t| > dist_th;
 *     validation: good = #{|T s_c - t_c|^2 < dist_th^2}, fitness = good/|corr|,
 *                 rmse = sqrt(sum/good) (0 if good == 0);
 *     better := fitness > best.fitness || (== && rmse < best.rmse); on improvement
 *     est_k = min(est_k, ceil(log(1-conf)/log(1-(good/|corr|)^3))).
 *   Result: best T, its inlier count (no final re-fit).  < 3 correspondences: identity, 0.
 * Determinism: Open3D's RNG/OpenMP schedule are not reproducible, so the draw is made an
 * explicit function of (seed, itr): Philox4x32-10 with key (seed_lo, seed_hi) and counter
 * (itr, 0, 0, 0); sample j = mulhi32(out[j], n_corr).  The sequential (single-thread) order
 * of the Open3D loop is the frozen semantics.
 * The rigid fit uses Horn's quaternion method (largest eigenvector of the 4x4 N matrix, cyclic
 * Jacobi, 10 fixed sweeps, fp64) -- the same optimum as Umeyama/Kabsch-with-det-fix whenever
 * that optimum is unique, and well defined for the always rank-deficient 3-point case.
 * ------------------------------------------------------------------------------------------ */
static inline void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                                 uint32_t out[4]) {
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        const uint32_t n1 = (uint32_t)p1;
        const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        const uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

static void jacobi4_max_eigvec(double A[4][4], double q[4]) {
    double V[4][4];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 10; ++sweep) {
        for (int p = 0; p < 3; ++p)
            for (int qq = p + 1; qq < 4; ++qq) {
                const double apq = A[p][qq];
                if (apq == 0.0) continue;
                const double theta = (A[qq][qq] - A[p][p]) / (2.0 * apq);
                const double at = fabs(theta);
                double t = 1.0 / (at + sqrt((theta * theta) + 1.0));
                if (theta < 0.0) t = -t;
                const double c = 1.0 / sqrt((t * t) + 1.0);
                const double s = t * c;
                const double app = A[p][p], aqq = A[qq][qq];
                A[p][p] = app - (t * apq);
                A[qq][qq] = aqq + (t * apq);
                A[p][qq] = 0.0;
                A[qq][p] = 0.0;
                for (int r = 0; r < 4; ++r) {
                    if (r == p || r == qq) continue;
                    const double arp = A[r][p], arq = A[r][qq];
                    A[r][p] = (c * arp) - (s * arq);
                    A[p][r] = A[r][p];
                    A[r][qq] = (s * arp) + (c * arq);
                    A[qq][r] = A[r][qq];
                }
                for (int k = 0; k < 4; ++k) {
                    const double vkp = V[k][p], vkq = V[k][qq];
                    V[k][p] = (c * vkp) - (s * vkq);
                    V[k][qq] = (s * vkp) + (c * vkq);
                }
            }
    }
    int m = 0; /* first maximum wins */
    for (int i = 1; i < 4; ++i)
        if (A[i][i] > A[m][m]) m = i;
    for (int k = 0; k < 4; ++k) q[k] = V[k][m];
}

/* rigid fit of n weighted pairs (fp64); T row-major 4x4.  w == NULL -> unit weights.
 * Frozen order: centroids = (sum_i w_i p_i) / (sum_i w_i + eps); S = sum_i w_i (a_i - ca)(b_i - cb)^T
 * accumulated sequentially in i; t = cb - R ca.  eps = 1e-6 restates rigid_transform_3d (BUFFERX.py:582-587),
 * 0 gives Open3D's unit-weight fit (RANSAC). */
static void horn_fit(const double *a, const double *b, const double *w, int n, double eps, double T[16]) {
    double ca[3] = {0, 0, 0}, cb[3] = {0, 0, 0}, sw = 0.0;
    for (int i = 0; i < n; ++i) {
        const double wi = w ? w[i] : 1.0;
        sw = sw + wi;
        for (int c = 0; c < 3; ++c) {
            ca[c] = ca[c] + (wi * a[3 * i + c]);
            cb[c] = cb[c] + (wi * b[3 * i + c]);
        }
    }
    for (int c = 0; c < 3; ++c) { ca[c] = ca[c] / (sw + eps); cb[c] = cb[c] / (sw + eps); }
    double S[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int i = 0; i < n; ++i) {
        const double wi = w ? w[i] : 1.0;
        double da[3], db[3];
        for (int c = 0; c < 3; ++c) { da[c] = a[3 * i + c] - ca[c]; db[c] = b[3 * i + c] - cb[c]; }
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) S[r][c] = S[r][c] + ((wi * da[r]) * db[c]);
    }
    double N[4][4];
    N[0][0] = (S[0][0] + S[1][1]) + S[2][2];
    N[0][1] = S[1][2] - S[2][1];
    N[0][2] = S[2][0] - S[0][2];
    N[0][3] = S[0][1] - S[1][0];
    N[1][1] = (S[0][0] - S[1][1]) - S[2][2];
    N[1][2] = S[0][1] + S[1][0];
    N[1][3] = S[2][0] + S[0][2];
    N[2][2] = ((-S[0][0]) + S[1][1]) - S[2][2];
    N[2][3] = S[1][2] + S[2][1];
    N[3][3] = ((-S[0][0]) - S[1][1]) + S[2][2];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < i; ++j) N[i][j] = N[j][i];
    double q[4];
    jacobi4_max_eigvec(N, q);
    const double qn = sqrt((((q[0] * q[0]) + (q[1] * q[1])) + (q[2] * q[2])) + (q[3] * q[3]));
    const double w0 = q[0] / qn, x = q[1] / qn, y = q[2] / qn, z = q[3] / qn;
    double R[3][3];
    R[0][0] = 1.0 - (2.0 * ((y * y) + (z * z)));
    R[0][1] = 2.0 * ((x * y) - (w0 * z));
    R[0][2] = 2.0 * ((x * z) + (w0 * y));
    R[1][0] = 2.0 * ((x * y) + (w0 * z));
    R[1][1] = 1.0 - (2.0 * ((x * x) + (z * z)));
    R[1][2] = 2.0 * ((y * z) - (w0 * x));
    R[2][0] = 2.0 * ((x * z) - (w0 * y));
    R[2][1] = 2.0 * ((y * z) + (w0 * x));
    R[2][2] = 1.0 - (2.0 * ((x * x) + (y * y)));
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) T[4 * r + c] = R[r][c];
        T[4 * r + 3] = cb[r] - (((R[r][0] * ca[0]) + (R[r][1] * ca[1])) + (R[r][2] * ca[2]));
    }
    T[12] = 0.0; T[13] = 0.0; T[14] = 0.0; T[15] = 1.0;
}

BX_EXPORT void bxo_horn_fit(const double *a, const double *b, const double *w, int n, double eps, double *T) {
    horn_fit(a, b, w, n, eps, T);
}

static inline void xform(const double T[16], const double p[3], double o[3]) {
    for (int r = 0; r < 3; ++r) o[r] = (((T[4 * r] * p[0]) + (T[4 * r + 1] * p[1])) + (T[4 * r + 2] * p[2])) + T[4 * r + 3];
}

/* per-iteration record, used by the tests to compare the GPU's hypothesis stage 1:1 */
typedef struct {
    int32_t pass;   /* 1 if both checkers passed */
    int32_t good;   /* inlier count (valid when pass) */
    double rmse;
} bxo_ransac_rec;

BX_EXPORT int bxo_ransac(const float *src, const float *tgt, const int32_t *inlier_ind, int n_corr, double dist_th,
                         double similar_th, double confidence, int max_iter, uint64_t seed, double *T_out /*16*/,
                         int32_t *num_inliers, int32_t *best_itr_out, int32_t *iters_run,
                         bxo_ransac_rec *recs /* optional [max_iter] */) {
    for (int i = 0; i < 16; ++i) T_out[i] = (i % 5 == 0) ? 1.0 : 0.0;
    *num_inliers = 0;
    if (best_itr_out) *best_itr_out = -1;
    if (iters_run) *iters_run = 0;
    if (n_corr < 3 || dist_th <= 0.0) return 0;
    double *S = (double *)malloc(sizeof(double) * 3 * (size_t)n_corr);
    double *D = (double *)malloc(sizeof(double) * 3 * (size_t)n_corr);
    for (int i = 0; i < n_corr; ++i)
        for (int c = 0; c < 3; ++c) {
            S[3 * i + c] = (double)src[3 * (size_t)inlier_ind[i] + c];
            D[3 * i + c] = (double)tgt[3 * (size_t)inlier_ind[i] + c];
        }
    const uint32_t k0 = (uint32_t)(seed & 0xffffffffu), k1 = (uint32_t)(seed >> 32);
    const double max_d2 = dist_th * dist_th;
    int best_good = 0, best_itr = -1, est_k = max_iter, itr = 0;
    double best_rmse = 0.0;
    for (itr = 0; itr < max_iter; ++itr) {
        if (itr >= est_k) break;
        uint32_t rnd[4];
        philox4x32_10((uint32_t)itr, 0u, 0u, 0u, k0, k1, rnd);
        int sel[3];
        double a[9], b[9];
        for (int j = 0; j < 3; ++j) {
            sel[j] = (int)(((uint64_t)rnd[j] * (uint64_t)n_corr) >> 32);
            for (int c = 0; c < 3; ++c) { a[3 * j + c] = S[3 * sel[j] + c]; b[3 * j + c] = D[3 * sel[j] + c]; }
        }
        if (recs) { recs[itr].pass = 0; recs[itr].good = 0; recs[itr].rmse = 0.0; }
        /* cheap checker first (order of evaluation does not change the outcome) */
        int ok = 1;
        for (int i = 0; i < 3 && ok; ++i)
            for (int j = i + 1; j < 3; ++j) {
                double ds = 0.0, dt = 0.0;
                for (int c = 0; c < 3; ++c) {
                    const double u = a[3 * i + c] - a[3 * j + c], v = b[3 * i + c] - b[3 * j + c];
                    ds = ds + (u * u);
                    dt = dt + (v * v);
                }
                ds = sqrt(ds);
                dt = sqrt(dt);
                if (ds < dt * similar_th || dt < ds * similar_th) { ok = 0; break; }
            }
        if (!ok) continue;
        double T[16];
        horn_fit(a, b, NULL, 3, 0.0, T);
        for (int j = 0; j < 3 && ok; ++j) {
            double o[3];
            xform(T, a + 3 * j, o);
            double e = 0.0;
            for (int c = 0; c < 3; ++c) { const double u = b[3 * j + c] - o[c]; e = e + (u * u); }
            if (sqrt(e) > dist_th) ok = 0;
        }
        if (!ok) continue;
        int good = 0;
        double err2 = 0.0;
        for (int i = 0; i < n_corr; ++i) {
            double o[3];
            xform(T, S + 3 * i, o);
            double e = 0.0;
            for (int c = 0; c < 3; ++c) { const double u = o[c] - D[3 * i + c]; e = e + (u * u); }
            if (e < max_d2) { ++good; err2 += e; }
        }
        const double rmse = good ? sqrt(err2 / (double)good) : 0.0;
        if (recs) { recs[itr].pass = 1; recs[itr].good = good; recs[itr].rmse = rmse; }
        /* fitness compare == integer compare of good (same denominator) */
        if (good > best_good || (good == best_good && rmse < best_rmse)) {
            best_good = good;
            best_rmse = rmse;
            best_itr = itr;
            memcpy(T_out, T, sizeof(double) * 16);
            const double ratio = (double)good / (double)n_corr;
            const double est = log(1.0 - confidence) / log(1.0 - pow(ratio, 3.0));
            if (est < (double)est_k) est_k = (int)ceil(est);
        }
    }
    *num_inliers = best_good;
    if (best_itr_out) *best_itr_out = best_itr;
    if (iters_run) *iters_run = itr;
    free(S);
    free(D);
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * a15. Post refinement -- /root/reference/models/BUFFERX.py:522-556 (+ rigid_transform_3d
 * :562-603).  Up to 20 rounds over ALL matches: inliers = |T s - t| < dist_th; stop when the
 * inlier count equals the previous round's; weights 1/(1+(d/th)^2); weighted rigid fit.
 * The reference runs this in fp32 with torch.svd; this restatement evaluates distances in fp32
 * (the inlier decision) and the fit in fp64 (Horn), with the reference's centroids over (sum w + 1e-6).
 * ref_check.py pins it against the
 * reference's own function within 1e-4.
 * ------------------------------------------------------------------------------------------ */
BX_EXPORT int bxo_refine(const float *src, const float *tgt, int n, const float *T_in /*16*/, float dist_th,
                         float *T_out /*16*/, int32_t *rounds) {
    float T[16];
    memcpy(T, T_in, sizeof(T));
    double *a = (double *)malloc(sizeof(double) * 3 * (size_t)(n > 0 ? n : 1));
    double *b = (double *)malloc(sizeof(double) * 3 * (size_t)(n > 0 ? n : 1));
    double *w = (double *)malloc(sizeof(double) * (size_t)(n > 0 ? n : 1));
    int prev = 0, r = 0;
    for (r = 0; r < 20; ++r) {
        int cnt = 0;
        for (int i = 0; i < n; ++i) {
            const float x = src[3 * i], y = src[3 * i + 1], z = src[3 * i + 2];
            const float qx = (((T[0] * x) + (T[1] * y)) + (T[2] * z)) + T[3];
            const float qy = (((T[4] * x) + (T[5] * y)) + (T[6] * z)) + T[7];
            const float qz = (((T[8] * x) + (T[9] * y)) + (T[10] * z)) + T[11];
            const float dx = qx - tgt[3 * i], dy = qy - tgt[3 * i + 1], dz = qz - tgt[3 * i + 2];
            const float d = sqrtf(((dx * dx) + (dy * dy)) + (dz * dz));
            if (d < dist_th) {
                for (int c = 0; c < 3; ++c) { a[3 * cnt + c] = (double)src[3 * i + c]; b[3 * cnt + c] = (double)tgt[3 * i + c]; }
                const float q = d / dist_th;
                w[cnt] = (double)(1.0f / (1.0f + (q * q)));
                ++cnt;
            }
        }
        if (cnt == prev) break;
        prev = cnt;
        if (cnt == 0) break;
        double Td[16];
        horn_fit(a, b, w, cnt, 1e-6, Td);
        for (int i = 0; i < 16; ++i) T[i] = (float)Td[i];
    }
    memcpy(T_out, T, sizeof(T));
    if (rounds) *rounds = r;
    free(a);
    free(b);
    free(w);
    return 0;
}

BX_EXPORT int bxo_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

BX_EXPORT void bxo_set_num_threads(int n) {
#ifdef _OPENMP
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* ------------------------------------------------------------------------------------------
 * a17. Batched fixed-radius neighbours, distance-sorted, padded (baseline semantics of the reference's
 * dead CPU module): /root/reference/cpp_wrappers/cpp_neighbors/neighbors/neighbors.cpp:334-480
 * (batch_nanoflanntbb_neighbors, the variant wired at wrapper.cpp:199).
 *   r2 = radius*radius in fp32; query batch b searches support cloud (b % 2) -- only s_batches[0] and
 *   s_batches[1] get a kd-tree (:377-393, :425, :457); distances in fp64 from the fp32 coordinates,
 *   d = ((dx*dx)+(dy*dy))+(dz*dz), kept iff d < r2 (strict, kiss_matcher/kdtree/nanoflann.hpp:250), sorted by
 *   distance (ties: lower index first here; the reference's std::sort leaves them unspecified); the index of a
 *   cloud-1 support is offset by s_batches[0]; rows are padded to the global maximum count with ns_total.
 * Returns max_count; *out is malloc'ed [nq*max_count] (free with bxo_free).
 * ------------------------------------------------------------------------------------------ */
typedef struct { double d; int32_t i; } bxo_nd;
static int bxo_nd_cmp(const void *a, const void *b) {
    const bxo_nd *x = (const bxo_nd *)a, *y = (const bxo_nd *)b;
    if (x->d < y->d) return -1;
    if (x->d > y->d) return 1;
    return (x->i > y->i) - (x->i < y->i);
}

BX_EXPORT int bxo_radius_neighbors(const float *queries, int nq, const float *supports, int ns_total, const int32_t *q_batches,
                                   int nqb, const int32_t *s_batches, int nsb, float radius, int32_t **out) {
    const double r2 = (double)(radius * radius);
    const int s0 = nsb > 0 ? s_batches[0] : 0, s1 = nsb > 1 ? s_batches[1] : 0;
    int32_t *cnt = (int32_t *)calloc((size_t)(nq > 0 ? nq : 1), sizeof(int32_t));
    bxo_nd **rows = (bxo_nd **)calloc((size_t)(nq > 0 ? nq : 1), sizeof(bxo_nd *));
#pragma omp parallel for schedule(dynamic, 16)
    for (int i = 0; i < nq; ++i) {
        int b = 0, acc = 0;
        for (int k = 0; k < nqb; ++k) {
            if (i >= acc && i < acc + q_batches[k]) { b = k; break; }
            acc += q_batches[k];
        }
        const int off = (b % 2 == 0) ? 0 : s0, n = (b % 2 == 0) ? s0 : s1;
        const double qx = queries[3 * i], qy = queries[3 * i + 1], qz = queries[3 * i + 2];
        bxo_nd *row = (bxo_nd *)malloc(sizeof(bxo_nd) * (size_t)(n > 0 ? n : 1));
        int c = 0;
        for (int j = 0; j < n; ++j) {
            const float *s = supports + 3 * (size_t)(off + j);
            const double dx = qx - (double)s[0], dy = qy - (double)s[1], dz = qz - (double)s[2];
            const double d = ((dx * dx) + (dy * dy)) + (dz * dz);
            if (d < r2) { row[c].d = d; row[c].i = off + j; ++c; }
        }
        qsort(row, (size_t)c, sizeof(bxo_nd), bxo_nd_cmp);
        rows[i] = row;
        cnt[i] = c;
    }
    int mc = 0;
    for (int i = 0; i < nq; ++i) mc = cnt[i] > mc ? cnt[i] : mc;
    int32_t *o = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nq * mc > 0 ? nq * mc : 1));
    for (int i = 0; i < nq; ++i) {
        for (int j = 0; j < mc; ++j) o[(size_t)i * mc + j] = j < cnt[i] ? rows[i][j].i : ns_total;
        free(rows[i]);
    }
    free(rows);
    free(cnt);
    *out = o;
    return mc;
}

BX_EXPORT void bxo_free(void *p) { free(p); }

/* ------------------------------------------------------------------------------------------
 * a18. Voxel-grid barycentre sub-sampling (baseline semantics):
 * /root/reference/cpp_wrappers/cpp_subsampling/grid_subsampling/grid_subsampling.cpp:5-106 (points only).
 *   origin = floor(min * (1/dl)) * dl (fp32, :27); NX, NY = floor((max - origin)/dl) + 1 (:30-31; -1 wraps, so 0);
 *   cell = floor((p - origin)/dl) per axis (:53-55; -1 wraps to 2^64-1), key = iX + NX*iY + NX*NY*iZ (:56, modulo 2^64); per cell the points are
 *   summed in INPUT order in fp32 (SampledData::update_points, grid_subsampling.h:93-98) and the barycentre is
 *   sum * float(1.0/count) (:87).  The reference emits cells in unordered_map iteration order; here ascending key.
 * keys_out / xyz_out / cnt_out need capacity n.  Returns the number of occupied cells.
 * ------------------------------------------------------------------------------------------ */
typedef struct { uint64_t key; int32_t idx; } bxo_ki;
static int bxo_ki_cmp(const void *a, const void *b) {
    const bxo_ki *x = (const bxo_ki *)a, *y = (const bxo_ki *)b;
    if (x->key != y->key) return x->key < y->key ? -1 : 1;
    return (x->idx > y->idx) - (x->idx < y->idx);
}

BX_EXPORT int bxo_grid_subsample(const float *pts, int n, float dl, uint64_t *keys_out, float *xyz_out, int32_t *cnt_out) {
    if (n <= 0) return 0;
    float mn[3] = {pts[0], pts[1], pts[2]}, mx[3] = {pts[0], pts[1], pts[2]};
    for (int i = 0; i < n; ++i)
        for (int c = 0; c < 3; ++c) {
            const float v = pts[3 * i + c];
            if (v < mn[c]) mn[c] = v;
            if (v > mx[c]) mx[c] = v;
        }
    const float inv = 1 / dl;
    float org[3];
    for (int c = 0; c < 3; ++c) org[c] = floorf(mn[c] * inv) * dl;
    /* through int64_t like the cell indices: a flat axis below its rounded-up origin gives floor = -1, NX (NY) = 0 */
    const uint64_t NX = (uint64_t)(int64_t)floorf((mx[0] - org[0]) / dl) + 1, NY = (uint64_t)(int64_t)floorf((mx[1] - org[1]) / dl) + 1;
    bxo_ki *ki = (bxo_ki *)malloc(sizeof(bxo_ki) * (size_t)n);
    for (int i = 0; i < n; ++i) {
        /* through int64_t: a cell index of -1 (origin rounded above the minimum) wraps to 2^64-1 like the reference's
         * x86 build, with defined behaviour */
        const uint64_t ix = (uint64_t)(int64_t)floorf((pts[3 * i] - org[0]) / dl), iy = (uint64_t)(int64_t)floorf((pts[3 * i + 1] - org[1]) / dl),
                       iz = (uint64_t)(int64_t)floorf((pts[3 * i + 2] - org[2]) / dl);
        ki[i].key = ix + NX * iy + NX * NY * iz;
        ki[i].idx = i;
    }
    qsort(ki, (size_t)n, sizeof(bxo_ki), bxo_ki_cmp);
    int m = 0;
    for (int i = 0; i < n;) {
        int j = i;
        float sx = 0.0f, sy = 0.0f, sz = 0.0f;
        while (j < n && ki[j].key == ki[i].key) {
            sx += pts[3 * ki[j].idx]; sy += pts[3 * ki[j].idx + 1]; sz += pts[3 * ki[j].idx + 2];
            ++j;
        }
        const int c = j - i;
        const float a = (float)(1.0 / (double)c);
        keys_out[m] = ki[i].key;
        xyz_out[3 * m] = sx * a; xyz_out[3 * m + 1] = sy * a; xyz_out[3 * m + 2] = sz * a;
        if (cnt_out) cnt_out[m] = c;
        ++m;
        i = j;
    }
    free(ki);
    return m;
}
