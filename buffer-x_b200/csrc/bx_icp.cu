// bx_icp.cu -- point-to-point ICP: Open3D 0.18 open3d.pipelines.registration.registration_icp with
// TransformationEstimationPointToPoint(with_scaling=False), which the reference's KITTI loader runs on the CPU to refine the
// ground-truth pose of every pair without a cached icp/<drive>_<t0>_<t1>.npy (/root/reference/dataset/kitti.py:95-102: the two
// raw scans, max_correspondence_distance = 0.20, init = I, ICPConvergenceCriteria(max_iteration=200)).
//
// The contract restated (oracle/icp_fp64.py restates it literally in NumPy float64):
//   1. max_correspondence_distance r <= 0 is refused.
//   2. pcd = source; if init is not the identity, pcd is transformed by init.  transformation = init.
//   3. Evaluation: every source point takes the nearest target point with float64 d2 < r*r (d2 = ((dx*dx)+(dy*dy))+(dz*dz));
//      fitness = correspondences / N_src, inlier_rmse = sqrt(sum d2 / correspondences), both 0 without a correspondence.
//   4. for i < max_iteration: update = umeyama(pcd[c0], target[c1]) (the identity without a correspondence);
//      transformation = update * transformation; pcd.Transform(update) (incrementally, in float64, never re-transformed from
//      the source by the accumulated transformation); re-evaluate; stop when |d fitness| < relative_fitness and
//      |d rmse| < relative_rmse.
//   5. umeyama (Eigen, with_scaling = false): centroids, Sigma = (1/n) sum (t - t_mean)(s - s_mean)^T, Sigma = U D V^T,
//      S = I with S_33 = -1 when det U * det V < 0, R = U S V^T, t = t_mean - R s_mean.
// Two rules Open3D leaves to FLANN are assumptions here: the radius test is strict (d2 < r*r), and among equidistant targets
// the lowest target index wins.  The correspondence set is reported by source index (Open3D's order depends on its OpenMP
// threads).
//
// Device pipeline (no host round trip between the steps; the result is read once at the end):
//   grid     the target is binned once per call into the spatial hash of bx_hashgrid.cuh (cells of edge >= r, counting sort
//            by hg_count_body / hg_scan_body / hg_scatter_body on an fp32 copy), then the sorted points are gathered back in
//            float64 with their index;
//   evaluate one thread per source point walks the hash buckets of its window (icp_window) and keeps the nearest target on
//            float64 d2 from the float64 point -- no fp32 prefilter; the moments of the correspondences (count, sum d2, sums
//            of s - p and t - p, sum (t - p)(s - p)^T) are taken about a pivot p (the source centroid of the previous
//            evaluation, the first transformed source point before that) and reduced in a fixed order: one partial per
//            block, then one final block.  No floating-point atomics, so a run is bit-reproducible;
//   finalize the final block turns the sums into fitness / rmse, applies the stopping test and solves the next update
//            (Umeyama on the fp64 Jacobi SVD of bx_svd3.cuh), update * transformation;
//   transform pcd = update * pcd.
// All max_iteration steps are enqueued up front; once the device state says the run has stopped, every later kernel returns
// at once (the scheme of bx_ransac's chunks).  No grid-wide barrier.
// Compiled with -fmad=false.
#include "bx_common.cuh"
#include "bx_hashgrid.cuh"
#include "bx_svd3.cuh"

namespace {

constexpr int ICP_THREADS = 256;
constexpr int ICP_SUMS = 17;                     // count, sum d2, sum (s - p)[3], sum (t - p)[3], sum (t - p)(s - p)^T[9]
constexpr float ICP_WINDOW_MAX = 524288.0f;      // 2^19 cells from the origin

struct IcpState {           // lives at the head of the workspace
    double T[16];           // transformation
    double upd[16];         // the update the next transform step applies
    double pivot[3];        // the next evaluation's moments are taken about this point
    double fitness, rmse;   // the latest evaluation
    int ncorr;
    int iterations;         // updates applied
    int done;               // 1: stopped (converged or max_iteration reached) -- every later kernel returns at once
    int converged;
    float rf;               // the binning radius: fl32(r) rounded up
};

struct IcpResult {          // 160 bytes, mirrored in the header comment
    double T[16];
    double fitness, inlier_rmse;
    int num_correspondences, iterations, converged, reserved;
};

struct alignas(32) Pt4d {
    double x, y, z, idx;
};

// Window (u = 2^-24, u53 = 2^-53, -fmad=false).  The target is binned by b = fl(fl32(p_x) * ic), ic = hg_inv_cell(rf),
// rf = fl32(r) rounded up, so r * ic <= 0.999001 (1 + 2u).  A hit has float64 d2 < r*r, so |q_x - p_x| < r (1 + 2^-50), and
// the fp32 coordinates differ by at most that plus u (|q_x| + |p_x|) <= r + u (2 |q_x| + r).  With a = fl(fl32(q_x) * ic),
// |q_x| ic <= |a| (1 + u)^2, and the roundings of a and b (u |a|, u (|a| + 1)):
//     |a - b| <= 0.99901 + 4.0002 u |a|.
// The window takes the cells [floorf(fl(a - w)), floorf(fl(a + w))] with w = fl(0.9993 + 2^-21 |a|) = 0.9993 + 8u|a| (to
// within u w); one more rounding of a -+ w costs u (|a| + w), so fl(a + w) >= b and fl(a - w) <= b with 2.8e-4 + 2.9 u |a|
// to spare, and floorf is monotone: the cell the point was binned in lies in the window.  That is 3 cells per axis while
// |a| < ~1468 (27 buckets) and at most 4 up to |a| < 2^19 (64 buckets); beyond that, and for a NaN point, the query scans
// the whole target.  tests/test_icp_fp64_cpu.py checks the enclosure and the sizes in fp32 with this arithmetic.
__device__ __forceinline__ void icp_window(float a, int &lo, int &n) {
    const float w = 0.9993f + 4.76837158203125e-07f * fabsf(a);        // 0.9993 + 2^-21 |a|
    lo = (int)floorf(a - w);
    n = (int)floorf(a + w) - lo + 1;                                    // 2 to 4
}

__device__ __forceinline__ void xform(const double *T, double x, double y, double z, double &ox, double &oy, double &oz) {
    ox = (((T[0] * x) + (T[1] * y)) + (T[2] * z)) + T[3];
    oy = (((T[4] * x) + (T[5] * y)) + (T[6] * z)) + T[7];
    oz = (((T[8] * x) + (T[9] * y)) + (T[10] * z)) + T[11];
}

__device__ __forceinline__ bool is_identity(const double *T) {
    bool id = true;
#pragma unroll
    for (int e = 0; e < 16; ++e) id = id && (T[e] == ((e % 5 == 0) ? 1.0 : 0.0));
    return id;
}

// fp32 copy of the target for the binning phases; thread 0 also starts the state
__global__ void icp_prep_kernel(const double *__restrict__ tgt, int Nt, const double *__restrict__ init, float rf, float4 *__restrict__ tgt4,
                                IcpState *__restrict__ st) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < Nt) tgt4[i] = make_float4((float)tgt[3 * (size_t)i], (float)tgt[3 * (size_t)i + 1], (float)tgt[3 * (size_t)i + 2], 0.0f);
    if (i == 0) {
        for (int e = 0; e < 16; ++e) { st->T[e] = init[e]; st->upd[e] = (e % 5 == 0) ? 1.0 : 0.0; }
        st->fitness = 0.0;
        st->rmse = 0.0;
        st->ncorr = 0;
        st->iterations = 0;
        st->done = 0;
        st->converged = 0;
        st->rf = rf;
    }
}

__global__ void icp_count_kernel(const float4 *__restrict__ tgt4, int Nt, const IcpState *__restrict__ st, int *__restrict__ cnt) {
    hg_count_body(tgt4, Nt, &st->rf, cnt, blockIdx.x * blockDim.x + threadIdx.x);
}
__global__ void __launch_bounds__(1024) icp_scan_kernel(const int *__restrict__ cnt, int *__restrict__ start, int *__restrict__ cursor) {
    hg_scan_body(cnt, start, cursor);
}
__global__ void icp_scatter_kernel(const float4 *__restrict__ tgt4, int Nt, const IcpState *__restrict__ st, int *__restrict__ cursor,
                                   float4 *__restrict__ sorted) {
    hg_scatter_body(tgt4, Nt, &st->rf, cursor, sorted, blockIdx.x * blockDim.x + threadIdx.x);
}
// the binned order in float64: sorted_d[k] = (target[j], j), j = the index the scatter stored
__global__ void icp_gather_kernel(const float4 *__restrict__ sorted, const double *__restrict__ tgt, int Nt, Pt4d *__restrict__ sorted_d) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= Nt) return;
    const int j = __float_as_int(sorted[k].w);
    sorted_d[k] = Pt4d{tgt[3 * (size_t)j], tgt[3 * (size_t)j + 1], tgt[3 * (size_t)j + 2], (double)j};
}

// pcd = init * source (a copy when init is the identity, as Open3D skips the transform); the first pivot is pcd[0]
__global__ void icp_init_pcd_kernel(const double *__restrict__ src, int Ns, IcpState *__restrict__ st, double *__restrict__ pcd) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Ns) return;
    double T[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) T[e] = st->T[e];
    double x = src[3 * (size_t)i], y = src[3 * (size_t)i + 1], z = src[3 * (size_t)i + 2];
    if (!is_identity(T)) xform(T, x, y, z, x, y, z);
    pcd[3 * (size_t)i] = x;
    pcd[3 * (size_t)i + 1] = y;
    pcd[3 * (size_t)i + 2] = z;
    if (i == 0) { st->pivot[0] = x; st->pivot[1] = y; st->pivot[2] = z; }
}

__global__ void icp_transform_kernel(double *__restrict__ pcd, int Ns, const IcpState *__restrict__ st) {
    if (st->done) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Ns) return;
    double U[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) U[e] = st->upd[e];
    double x = pcd[3 * (size_t)i], y = pcd[3 * (size_t)i + 1], z = pcd[3 * (size_t)i + 2];
    xform(U, x, y, z, x, y, z);
    pcd[3 * (size_t)i] = x;
    pcd[3 * (size_t)i + 1] = y;
    pcd[3 * (size_t)i + 2] = z;
}

// fixed-order block sum of ICP_SUMS doubles per thread: xor butterfly per warp, then the warps in order
__device__ __forceinline__ void block_sums(double (&acc)[ICP_SUMS], double *__restrict__ out) {
    __shared__ double red[ICP_THREADS / 32][ICP_SUMS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1)
#pragma unroll
        for (int e = 0; e < ICP_SUMS; ++e) acc[e] += __shfl_xor_sync(BX_FULL, acc[e], o);
    if (lane == 0)
#pragma unroll
        for (int e = 0; e < ICP_SUMS; ++e) red[warp][e] = acc[e];
    __syncthreads();
    if (threadIdx.x < ICP_SUMS) {
        double v = 0.0;
        for (int w = 0; w < ICP_THREADS / 32; ++w) v += red[w][threadIdx.x];
        out[threadIdx.x] = v;
    }
}

__global__ void __launch_bounds__(ICP_THREADS)
icp_nn_kernel(const double *__restrict__ pcd, int Ns, const Pt4d *__restrict__ sorted_d, const int *__restrict__ start, int Nt, double r2,
              const IcpState *__restrict__ st, int *__restrict__ corr, double *__restrict__ partials) {
    if (st->done) return;                                      // uniform over the grid
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const double px = st->pivot[0], py = st->pivot[1], pz = st->pivot[2];
    double acc[ICP_SUMS];
#pragma unroll
    for (int e = 0; e < ICP_SUMS; ++e) acc[e] = 0.0;
    if (i < Ns) {
        const double qx = pcd[3 * (size_t)i], qy = pcd[3 * (size_t)i + 1], qz = pcd[3 * (size_t)i + 2];
        double best = r2;
        int bj = -1;
        double bx = 0.0, by = 0.0, bz = 0.0;
        auto test = [&](const Pt4d &p) {
            const double dx = qx - p.x, dy = qy - p.y, dz = qz - p.z;
            const double d2 = ((dx * dx) + (dy * dy)) + (dz * dz);
            const int j = (int)p.idx;
            if (d2 < best || (d2 == best && bj >= 0 && j < bj)) { best = d2; bj = j; bx = p.x; by = p.y; bz = p.z; }
        };
        const float ic = hg_inv_cell(st->rf);
        const float ax = (float)qx * ic, ay = (float)qy * ic, az = (float)qz * ic;
        if (fabsf(ax) < ICP_WINDOW_MAX && fabsf(ay) < ICP_WINDOW_MAX && fabsf(az) < ICP_WINDOW_MAX) {
            int lx, nx, ly, ny, lz, nz;
            icp_window(ax, lx, nx);
            icp_window(ay, ly, ny);
            icp_window(az, lz, nz);
            for (int ix = 0; ix < nx; ++ix)
                for (int iy = 0; iy < ny; ++iy)
                    for (int iz = 0; iz < nz; ++iz) {
                        const unsigned h = hg_hash(lx + ix, ly + iy, lz + iz);
                        const int k1 = start[h + 1];
                        for (int k = start[h]; k < k1; ++k) test(sorted_d[k]);
                    }
        } else {
            for (int k = 0; k < Nt; ++k) test(sorted_d[k]);
        }
        corr[i] = bj;
        if (bj >= 0) {
            const double s[3] = {qx - px, qy - py, qz - pz}, t[3] = {bx - px, by - py, bz - pz};
            acc[0] = 1.0;
            acc[1] = best;
#pragma unroll
            for (int e = 0; e < 3; ++e) {
                acc[2 + e] = s[e];
                acc[5 + e] = t[e];
#pragma unroll
                for (int f = 0; f < 3; ++f) acc[8 + 3 * e + f] = t[e] * s[f];
            }
        }
    }
    block_sums(acc, partials + (size_t)blockIdx.x * ICP_SUMS);
}

// one block: the partials in a fixed order, then (thread 0) the evaluation, the stopping test and the next update
__global__ void __launch_bounds__(ICP_THREADS)
icp_finalize_kernel(const double *__restrict__ partials, int nblocks, int Ns, int step, int max_iteration, double relative_fitness,
                    double relative_rmse, IcpState *__restrict__ st, IcpResult *__restrict__ res) {
    if (st->done) return;
    __shared__ double tot[ICP_SUMS];
    double acc[ICP_SUMS];
#pragma unroll
    for (int e = 0; e < ICP_SUMS; ++e) acc[e] = 0.0;
    for (int b = threadIdx.x; b < nblocks; b += ICP_THREADS)
#pragma unroll
        for (int e = 0; e < ICP_SUMS; ++e) acc[e] += partials[(size_t)b * ICP_SUMS + e];
    block_sums(acc, tot);
    __syncthreads();
    if (threadIdx.x != 0) return;
    const double n = tot[0];
    const double fitness = n > 0.0 ? n / (double)Ns : 0.0;
    const double rmse = n > 0.0 ? sqrt(tot[1] / n) : 0.0;
    bool stop = step >= max_iteration;
    if (step > 0 && fabs(st->fitness - fitness) < relative_fitness && fabs(st->rmse - rmse) < relative_rmse) {
        stop = true;
        st->converged = 1;
    }
    st->fitness = fitness;
    st->rmse = rmse;
    st->ncorr = (int)n;
    st->iterations = step;
    if (!stop) {
        double U[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) U[e] = (e % 5 == 0) ? 1.0 : 0.0;
        if (n > 0.0) {
            double ms[3], mt[3], w[3][3], u[3][3], sv[3], v[3][3];
            for (int e = 0; e < 3; ++e) { ms[e] = tot[2 + e] / n; mt[e] = tot[5 + e] / n; }
            // Sigma[r][c] = (1/n) sum (t - p)_r (s - p)_c - mt_r ms_c; w[c] = column c
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) w[c][r] = tot[8 + 3 * r + c] / n - mt[r] * ms[c];
            bx_svd3_fp64(w, u, sv, v);
            auto det = [](const double (&m)[3][3]) {   // columns m[0], m[1], m[2]: m0 . (m1 x m2)
                return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
                       m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
            };
            const double s3 = (det(u) * det(v) < 0.0) ? -1.0 : 1.0;
            double cs[3], ct[3];
            for (int e = 0; e < 3; ++e) { cs[e] = st->pivot[e] + ms[e]; ct[e] = st->pivot[e] + mt[e]; }
            for (int r = 0; r < 3; ++r) {
                for (int c = 0; c < 3; ++c) U[4 * r + c] = ((u[0][r] * v[0][c]) + (u[1][r] * v[1][c])) + ((s3 * u[2][r]) * v[2][c]);
                U[4 * r + 3] = ct[r] - (((U[4 * r] * cs[0]) + (U[4 * r + 1] * cs[1])) + (U[4 * r + 2] * cs[2]));
            }
            for (int e = 0; e < 3; ++e) st->pivot[e] = cs[e];
        }
        double T[16];
        for (int r = 0; r < 4; ++r)
            for (int c = 0; c < 4; ++c)
                T[4 * r + c] = (((U[4 * r] * st->T[c]) + (U[4 * r + 1] * st->T[4 + c])) + (U[4 * r + 2] * st->T[8 + c])) + (U[4 * r + 3] * st->T[12 + c]);
        for (int e = 0; e < 16; ++e) { st->upd[e] = U[e]; st->T[e] = T[e]; }
    } else {
        st->done = 1;
    }
    // when the run stops, st->T is the transformation that the evaluated pcd carries (no update was made here)
    if (stop) {
        for (int e = 0; e < 16; ++e) res->T[e] = st->T[e];
        res->fitness = fitness;
        res->inlier_rmse = rmse;
        res->num_correspondences = (int)n;
        res->iterations = step;
        res->converged = st->converged;
        res->reserved = 0;
    }
}

size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

}  // namespace

BX_API int64_t bx_icp_workspace_bytes(int n_src, int n_tgt) {
    if (n_src < 0 || n_tgt < 0) return -1;
    const size_t nb = ((size_t)n_src + ICP_THREADS - 1) / ICP_THREADS;
    return (int64_t)(align_up(sizeof(IcpState)) + align_up((size_t)n_src * 24) + 2 * align_up((size_t)n_tgt * 16) +
                     align_up((size_t)n_tgt * sizeof(Pt4d)) + align_up((size_t)(3 * HG_CELLS + 8) * 4) + align_up(nb * ICP_SUMS * 8));
}

BX_API int bx_icp(const double *src, int n_src, const double *tgt, int n_tgt, double max_correspondence_distance, const double *init,
                  double relative_fitness, double relative_rmse, int max_iteration, int32_t *corr, void *result, void *workspace,
                  void *stream) {
    BX_REQUIRE(src && tgt && init && corr && result && workspace, "bx_icp: null pointer");
    BX_REQUIRE(n_src >= 1 && n_tgt >= 1, "bx_icp: empty cloud (n_src=%d, n_tgt=%d)", n_src, n_tgt);
    BX_REQUIRE(max_correspondence_distance > 0.0 && max_correspondence_distance <= 3.0e38,
               "bx_icp: max_correspondence_distance=%g must be positive and finite", max_correspondence_distance);
    BX_REQUIRE(max_iteration >= 0, "bx_icp: max_iteration=%d < 0", max_iteration);
    BX_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0 && (reinterpret_cast<uintptr_t>(result) & 7) == 0,
               "bx_icp: workspace must be 256-byte and result 8-byte aligned");
    cudaStream_t stm = bx_stream(stream);
    unsigned char *ws = static_cast<unsigned char *>(workspace);
    IcpState *st = reinterpret_cast<IcpState *>(ws);
    ws += align_up(sizeof(IcpState));
    double *pcd = reinterpret_cast<double *>(ws);
    ws += align_up((size_t)n_src * 24);
    float4 *tgt4 = reinterpret_cast<float4 *>(ws);
    ws += align_up((size_t)n_tgt * 16);
    float4 *sorted = reinterpret_cast<float4 *>(ws);
    ws += align_up((size_t)n_tgt * 16);
    Pt4d *sorted_d = reinterpret_cast<Pt4d *>(ws);
    ws += align_up((size_t)n_tgt * sizeof(Pt4d));
    int *cnt = reinterpret_cast<int *>(ws);
    int *start = cnt + HG_CELLS, *cursor = start + HG_CELLS + 4;      // 16-byte aligned arrays (int4 accesses in the scan)
    ws += align_up((size_t)(3 * HG_CELLS + 8) * 4);
    double *partials = reinterpret_cast<double *>(ws);
    const int nb = (n_src + ICP_THREADS - 1) / ICP_THREADS, tb = (n_tgt + 255) / 256;

    float rf = (float)max_correspondence_distance;                     // the binning radius may not be below r
    if ((double)rf < max_correspondence_distance) rf = nextafterf(rf, 3.5e38f);
    const double r2 = max_correspondence_distance * max_correspondence_distance;

    icp_prep_kernel<<<tb, 256, 0, stm>>>(tgt, n_tgt, init, rf, tgt4, st);
    BX_LAUNCH_CHECK();
    BX_CUDA(cudaMemsetAsync(cnt, 0, (size_t)HG_CELLS * 4, stm));
    icp_count_kernel<<<tb, 256, 0, stm>>>(tgt4, n_tgt, st, cnt);
    BX_LAUNCH_CHECK();
    icp_scan_kernel<<<1, 1024, 0, stm>>>(cnt, start, cursor);
    BX_LAUNCH_CHECK();
    icp_scatter_kernel<<<tb, 256, 0, stm>>>(tgt4, n_tgt, st, cursor, sorted);
    BX_LAUNCH_CHECK();
    icp_gather_kernel<<<tb, 256, 0, stm>>>(sorted, tgt, n_tgt, sorted_d);
    BX_LAUNCH_CHECK();
    icp_init_pcd_kernel<<<nb, ICP_THREADS, 0, stm>>>(src, n_src, st, pcd);
    BX_LAUNCH_CHECK();
    IcpResult *res = static_cast<IcpResult *>(result);
    for (int step = 0; step <= max_iteration; ++step) {
        if (step > 0) {
            icp_transform_kernel<<<nb, ICP_THREADS, 0, stm>>>(pcd, n_src, st);
            BX_LAUNCH_CHECK();
        }
        icp_nn_kernel<<<nb, ICP_THREADS, 0, stm>>>(pcd, n_src, sorted_d, start, n_tgt, r2, st, corr, partials);
        BX_LAUNCH_CHECK();
        icp_finalize_kernel<<<1, ICP_THREADS, 0, stm>>>(partials, nb, n_src, step, max_iteration, relative_fitness, relative_rmse, st, res);
        BX_LAUNCH_CHECK();
    }
    return BX_OK;
}
