// bx_bootstrap.cu -- SURVEY 8(f) row 1: loader-side geometric bootstrapping on the GPU.
//
//   bx_pca_analysis      replaces compute_pca_alignment (/root/reference/utils/tools.py:132-149): PCA of a 10 % random
//                        sample (the sample indices are an input: the reference draws them from NumPy's global RNG).
//                        sklearn.decomposition.PCA(n_components=3) on [n,3] data = eigen-decomposition of the sample
//                        covariance (centred, 1/(n-1)); components_ rows sorted by decreasing eigenvalue, sign of a row
//                        fixed so that its entry of largest magnitude is positive (sklearn >= 1.5 svd_flip,
//                        u_based_decision=False).  fp64 throughout, like the reference (Open3D points are doubles).
//   bx_project_range     min / max of (p - mean) . axis over a whole cloud = the z-range of pca.transform(points)
//                        (tools.py:181-182) without materialising the transformed cloud.
//   bx_voxel_down_sample replaces open3d.geometry.PointCloud.voxel_down_sample (Open3D 0.18, PointCloud.cpp
//                        VoxelDownSample; call sites dataset/*.py, utils/tools.py:218-219): voxel_min_bound = min - 0.5 *
//                        voxel, index = floor((p - voxel_min_bound) / voxel) in fp64, output = mean of the points of a
//                        voxel (fp64 sums).  Open3D emits in unordered_map order; here the order is the hash-table slot
//                        order, parity is on the set of (voxel, mean).
// -fmad=false file: the fp64 expressions are evaluated as written (oracle: oracle/oracle.py, NumPy float64).
#include "bx_common.cuh"

namespace {

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(BX_FULL, v, o);
    return v;
}

// acc[0..2] += sum of the sampled points (pass 0) or acc[3..8] += centred products xx, xy, xz, yy, yz, zz (pass 1)
__global__ void pca_accum_kernel(const float *__restrict__ pts, const int *__restrict__ idx, int ns, int pass,
                                 double *__restrict__ acc) {
    double s[6] = {0, 0, 0, 0, 0, 0};
    const double inv = 1.0 / (double)ns;
    const double mx = acc[0] * inv, my = acc[1] * inv, mz = acc[2] * inv;   // valid in pass 1
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) {
        const int j = idx ? idx[i] : i;
        const double x = (double)pts[3 * (size_t)j], y = (double)pts[3 * (size_t)j + 1], z = (double)pts[3 * (size_t)j + 2];
        if (pass == 0) {
            s[0] += x; s[1] += y; s[2] += z;
        } else {
            const double dx = x - mx, dy = y - my, dz = z - mz;
            s[0] += dx * dx; s[1] += dx * dy; s[2] += dx * dz; s[3] += dy * dy; s[4] += dy * dz; s[5] += dz * dz;
        }
    }
    const int nv = pass == 0 ? 3 : 6;
    for (int q = 0; q < nv; ++q) {
        const double w = warp_sum(s[q]);
        if ((threadIdx.x & 31) == 0) atomicAdd(&acc[(pass == 0 ? 0 : 3) + q], w);
    }
}

// out: mean[3], eigenvalues[3] (descending), components[3][3] (rows, unit norm, largest-magnitude entry positive)
__global__ void pca_eig_kernel(const double *__restrict__ acc, int ns, double *__restrict__ out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const double inv = 1.0 / (double)ns, invn1 = 1.0 / (double)(ns - 1);
    out[0] = acc[0] * inv; out[1] = acc[1] * inv; out[2] = acc[2] * inv;
    double A[3][3] = {{acc[3] * invn1, acc[4] * invn1, acc[5] * invn1},
                      {acc[4] * invn1, acc[6] * invn1, acc[7] * invn1},
                      {acc[5] * invn1, acc[7] * invn1, acc[8] * invn1}};
    double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    for (int sweep = 0; sweep < 60; ++sweep) {          // cyclic Jacobi, fp64
        const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
        if (off < 1e-300) break;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                if (fabs(A[p][q]) < 1e-300) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 3; ++k) {
                    const double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq;
                    A[k][q] = s * akp + c * akq;
                }
                for (int k = 0; k < 3; ++k) {
                    const double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk;
                    A[q][k] = s * apk + c * aqk;
                }
                for (int k = 0; k < 3; ++k) {
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - s * vkq;
                    V[k][q] = s * vkp + c * vkq;
                }
            }
    }
    int ord[3] = {0, 1, 2};
    for (int a = 0; a < 2; ++a)
        for (int b = a + 1; b < 3; ++b)
            if (A[ord[b]][ord[b]] > A[ord[a]][ord[a]]) { const int t = ord[a]; ord[a] = ord[b]; ord[b] = t; }
    for (int r = 0; r < 3; ++r) {
        const int j = ord[r];
        out[3 + r] = A[j][j];
        double v[3] = {V[0][j], V[1][j], V[2][j]};
        const double nrm = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        int im = 0;
        for (int k = 1; k < 3; ++k)
            if (fabs(v[k]) > fabs(v[im])) im = k;
        const double sg = (v[im] < 0 ? -1.0 : 1.0) / nrm;
        for (int k = 0; k < 3; ++k) out[6 + 3 * r + k] = v[k] * sg;
    }
}

// order-preserving encoding of a double as an unsigned 64-bit integer (for atomicMin / atomicMax)
__device__ __forceinline__ unsigned long long enc_ordered(double v) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double dec_ordered(unsigned long long e) {
    const unsigned long long u = (e >> 63) ? (e & 0x7fffffffffffffffull) : ~e;
    return __longlong_as_double((long long)u);
}

__global__ void project_range_kernel(const float *__restrict__ pts, int n, const double *__restrict__ mean_axis,
                                     unsigned long long *__restrict__ mm /* [2]: min, max (ordered encoding) */) {
    const double mx = mean_axis[0], my = mean_axis[1], mz = mean_axis[2];
    const double ax = mean_axis[3], ay = mean_axis[4], az = mean_axis[5];
    double lo = INFINITY, hi = -INFINITY;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const double x = (double)pts[3 * (size_t)i] - mx, y = (double)pts[3 * (size_t)i + 1] - my, z = (double)pts[3 * (size_t)i + 2] - mz;
        const double v = (x * ax + y * ay) + z * az;
        lo = fmin(lo, v);
        hi = fmax(hi, v);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        lo = fmin(lo, __shfl_xor_sync(BX_FULL, lo, o));
        hi = fmax(hi, __shfl_xor_sync(BX_FULL, hi, o));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&mm[0], enc_ordered(lo));
        atomicMax(&mm[1], enc_ordered(hi));
    }
}

__global__ void range_decode_kernel(const unsigned long long *__restrict__ mm, double *__restrict__ out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) { out[0] = dec_ordered(mm[0]); out[1] = dec_ordered(mm[1]); }
}

// ---- voxel_down_sample ------------------------------------------------------------------------------------------
__global__ void vds_minmax_kernel(const float *__restrict__ pts, int n, unsigned long long *__restrict__ mm /* [6] */) {
    double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double v = (double)pts[3 * (size_t)i + c];
            mn[c] = fmin(mn[c], v);
            mx[c] = fmax(mx[c], v);
        }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        for (int o = 16; o >= 1; o >>= 1) {
            mn[c] = fmin(mn[c], __shfl_xor_sync(BX_FULL, mn[c], o));
            mx[c] = fmax(mx[c], __shfl_xor_sync(BX_FULL, mx[c], o));
        }
        if ((threadIdx.x & 31) == 0) {
            atomicMin(&mm[c], enc_ordered(mn[c]));
            atomicMax(&mm[3 + c], enc_ordered(mx[c]));
        }
    }
}

__global__ void vds_insert_kernel(const float *__restrict__ pts, int n, double voxel, const unsigned long long *__restrict__ mm,
                                  unsigned long long *__restrict__ tkeys, double *__restrict__ tacc, int tcap) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    long long iv[3];
    double p[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double vmb = dec_ordered(mm[c]) - voxel * 0.5;          // voxel_min_bound
        p[c] = (double)pts[3 * (size_t)i + c];
        iv[c] = (long long)floor((p[c] - vmb) / voxel);
    }
    // 21 bits per axis: distinct keys below 2^21 voxels per axis.  Not checked here; the host reads minmax6 with d_m
    // and refuses a wider cloud (ops.voxel_down_sample).
    const unsigned long long key = ((unsigned long long)iv[0] & 0x1FFFFFull) | (((unsigned long long)iv[1] & 0x1FFFFFull) << 21) |
                                   (((unsigned long long)iv[2] & 0x1FFFFFull) << 42);
    const unsigned long long h = key * 0x9E3779B97F4A7C15ull;
    unsigned slot = (unsigned)(h >> 32) & (unsigned)(tcap - 1);
    const unsigned long long EMPTY = ~0ull;
    while (true) {
        const unsigned long long prev = atomicCAS(&tkeys[slot], EMPTY, key);
        if (prev == EMPTY || prev == key) break;
        slot = (slot + 1) & (unsigned)(tcap - 1);
    }
    atomicAdd(&tacc[4 * (size_t)slot], p[0]);
    atomicAdd(&tacc[4 * (size_t)slot + 1], p[1]);
    atomicAdd(&tacc[4 * (size_t)slot + 2], p[2]);
    atomicAdd(&tacc[4 * (size_t)slot + 3], 1.0);
}

__global__ void vds_emit_kernel(const unsigned long long *__restrict__ tkeys, const double *__restrict__ tacc, int tcap,
                                unsigned long long *__restrict__ keys_out, float *__restrict__ xyz_out, int *__restrict__ cnt_out,
                                int *__restrict__ d_m) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= tcap) return;
    const unsigned long long k = tkeys[s];
    if (k == ~0ull) return;
    const double c = tacc[4 * (size_t)s + 3];
    const int o = atomicAdd(d_m, 1);
    keys_out[o] = k;
    xyz_out[3 * (size_t)o] = (float)(tacc[4 * (size_t)s] / c);
    xyz_out[3 * (size_t)o + 1] = (float)(tacc[4 * (size_t)s + 1] / c);
    xyz_out[3 * (size_t)o + 2] = (float)(tacc[4 * (size_t)s + 2] / c);
    if (cnt_out) cnt_out[o] = (int)c;
}

int grid_blocks(int n) {
    int b = (n + 255) / 256;
    return b > 592 ? 592 : (b < 1 ? 1 : b);
}

}  // namespace

BX_API int bx_pca_analysis(const float *pts, int n, const int32_t *sample_idx, int n_sample, double *acc9, double *out15,
                           void *stream) {
    BX_REQUIRE(pts && acc9 && out15, "bx_pca_analysis: null pointer");
    BX_REQUIRE(n >= 2 && n_sample >= 3 && (sample_idx || n_sample == n),
               "bx_pca_analysis: PCA(n_components=3) needs at least three samples (n=%d, n_sample=%d)", n, n_sample);
    cudaStream_t st = bx_stream(stream);
    BX_CUDA(cudaMemsetAsync(acc9, 0, 9 * sizeof(double), st));
    pca_accum_kernel<<<grid_blocks(n_sample), 256, 0, st>>>(pts, sample_idx, n_sample, 0, acc9);
    BX_LAUNCH_CHECK();
    pca_accum_kernel<<<grid_blocks(n_sample), 256, 0, st>>>(pts, sample_idx, n_sample, 1, acc9);
    BX_LAUNCH_CHECK();
    pca_eig_kernel<<<1, 32, 0, st>>>(acc9, n_sample, out15);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_project_range(const float *pts, int n, const double *mean_axis6, unsigned long long *work2, double *out2, void *stream) {
    BX_REQUIRE(pts && mean_axis6 && work2 && out2 && n >= 1, "bx_project_range: bad arguments");
    cudaStream_t st = bx_stream(stream);
    const unsigned long long init[2] = {~0ull, 0ull};
    BX_CUDA(cudaMemcpyAsync(work2, init, sizeof(init), cudaMemcpyHostToDevice, st));
    project_range_kernel<<<grid_blocks(n), 256, 0, st>>>(pts, n, mean_axis6, work2);
    BX_LAUNCH_CHECK();
    range_decode_kernel<<<1, 32, 0, st>>>(work2, out2);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_voxel_down_sample(const float *pts, int n, double voxel, unsigned long long *table_keys, double *table_acc, int table_cap,
                                unsigned long long *minmax6, unsigned long long *keys_out, float *xyz_out, int32_t *cnt_out,
                                int32_t *d_m, void *stream) {
    BX_REQUIRE(pts && table_keys && table_acc && minmax6 && keys_out && xyz_out && d_m, "bx_voxel_down_sample: null pointer");
    BX_REQUIRE(n >= 1 && voxel > 0.0, "bx_voxel_down_sample: bad arguments");
    BX_REQUIRE(table_cap >= 2 * n && (table_cap & (table_cap - 1)) == 0, "bx_voxel_down_sample: table_cap must be a power of two >= 2n");
    cudaStream_t st = bx_stream(stream);
    BX_CUDA(cudaMemsetAsync(table_keys, 0xFF, sizeof(unsigned long long) * (size_t)table_cap, st));
    BX_CUDA(cudaMemsetAsync(table_acc, 0, sizeof(double) * 4 * (size_t)table_cap, st));
    BX_CUDA(cudaMemsetAsync(d_m, 0, sizeof(int), st));
    const unsigned long long init[6] = {~0ull, ~0ull, ~0ull, 0ull, 0ull, 0ull};
    BX_CUDA(cudaMemcpyAsync(minmax6, init, sizeof(init), cudaMemcpyHostToDevice, st));
    vds_minmax_kernel<<<grid_blocks(n), 256, 0, st>>>(pts, n, minmax6);
    BX_LAUNCH_CHECK();
    vds_insert_kernel<<<(n + 255) / 256, 256, 0, st>>>(pts, n, voxel, minmax6, table_keys, table_acc, table_cap);
    BX_LAUNCH_CHECK();
    vds_emit_kernel<<<(table_cap + 255) / 256, 256, 0, st>>>(table_keys, table_acc, table_cap, keys_out, xyz_out, cnt_out, d_m);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
