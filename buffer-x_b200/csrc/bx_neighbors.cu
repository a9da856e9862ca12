// bx_neighbors.cu -- a17 / a18: GPU counterparts of the reference's (dead) CPU modules cpp_wrappers.
//
// a17 bx_radius_neighbors replaces radius_neighbors.batch_query
//     (/root/reference/cpp_wrappers/cpp_neighbors/wrapper.cpp:58-239 ->
//      neighbors/neighbors.cpp:334-480 batch_nanoflanntbb_neighbors): for every query ALL supports of its cloud
//     with d < r*r (fp64 distance from the fp32 coordinates, strict), sorted by (distance, index), rows padded with
//     the total support count.  The reference sorts with std::sort, which leaves equal distances in no set order:
//     its rows share our distance sequence and the index set of every equal-distance run, not the order inside one.
//     Query batch b searches support cloud (b % 2) exactly like the reference, which only builds kd-trees for
//     s_batches[0] and s_batches[1].  One CTA per query: ballot-free brute scan with a
//     shared-memory append, then an in-CTA bitonic sort of (distance, index) -- two double kd-trees and a TBB
//     reduction in the reference.
// a18 bx_grid_subsample replaces grid_subsampling.subsample
//     (/root/reference/cpp_wrappers/cpp_subsampling/wrapper.cpp:631-859 -> grid_subsampling.cpp:5-106):
//     voxel barycentres through a device hash grid keyed by the reference's cell id
//     iX + NX*iY + NX*NY*iZ (origin = floor(min/dl)*dl), instead of a serial unordered_map.
// Bit contract: oracle bxo_radius_neighbors (exact, ties by index) / bxo_grid_subsample (cell keys and counts exact,
// barycentres to fp32 summation order).  Compiled with -fmad=false.
#include "bx_common.cuh"

namespace {

constexpr int RN_THREADS = 256;
constexpr int RN_CAP = 4096;  // neighbours per query that fit the in-CTA sort

struct Batches {
    int q_acc[9];  // prefix sums of up to 8 query batches
    int nqb;
    int s0, s1, ns_total;
};

__device__ __forceinline__ bool nd_less(double da, int ia, double db, int ib) { return da < db || (da == db && ia < ib); }

__global__ void __launch_bounds__(RN_THREADS)
radius_neighbors_kernel(const float *__restrict__ queries, int nq, const float *__restrict__ supports, const Batches bt,
                        float radius, int *__restrict__ out, int cap, int *__restrict__ d_max_count,
                        double *__restrict__ big_d, int *__restrict__ big_i) {
    extern __shared__ unsigned char rn_smem[];
    double *sd = reinterpret_cast<double *>(rn_smem);          // RN_CAP
    int *si = reinterpret_cast<int *>(sd + RN_CAP);            // RN_CAP
    __shared__ int s_cnt;
    const int i = blockIdx.x;
    if (i >= nq) return;
    int b = 0;
    for (int k = 0; k < bt.nqb; ++k)
        if (i >= bt.q_acc[k] && i < bt.q_acc[k + 1]) { b = k; break; }
    const int off = (b % 2 == 0) ? 0 : bt.s0;
    const int n = (b % 2 == 0) ? bt.s0 : bt.s1;
    const double r2 = (double)(radius * radius);
    const double qx = queries[3 * (size_t)i], qy = queries[3 * (size_t)i + 1], qz = queries[3 * (size_t)i + 2];
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += RN_THREADS) {
        const float *s = supports + 3 * (size_t)(off + j);
        const double dx = qx - (double)s[0], dy = qy - (double)s[1], dz = qz - (double)s[2];
        const double d = ((dx * dx) + (dy * dy)) + (dz * dz);
        if (d < r2) {
            const int slot = atomicAdd(&s_cnt, 1);
            if (slot < RN_CAP) { sd[slot] = d; si[slot] = off + j; }
        }
    }
    __syncthreads();
    const int cnt = s_cnt;
    if (threadIdx.x == 0) atomicMax(d_max_count, cnt);
    if (out == nullptr) return;                      // counting pass
    if (cnt > RN_CAP) {
        // Ball too large for the shared-memory sort (needs the caller's global scratch rows of `cap` entries): collect the
        // (distance, index) pairs again into global memory, then place every entry at its RANK -- the number of entries that
        // precede it in (distance, index) order.  O(cnt^2 / 256) per query, exact, no power-of-two padding.
        int *row = out + (size_t)i * cap;
        if (big_d == nullptr || cnt > cap) {          // caller promised cap <= RN_CAP: truncating silently is not an option
            for (int j = threadIdx.x; j < cap; j += RN_THREADS) row[j] = -1;
            return;
        }
        double *gd = big_d + (size_t)i * cap;
        int *gi = big_i + (size_t)i * cap;
        __syncthreads();
        if (threadIdx.x == 0) s_cnt = 0;
        __syncthreads();
        for (int j = threadIdx.x; j < n; j += RN_THREADS) {
            const float *s = supports + 3 * (size_t)(off + j);
            const double dx = qx - (double)s[0], dy = qy - (double)s[1], dz = qz - (double)s[2];
            const double d = ((dx * dx) + (dy * dy)) + (dz * dz);
            if (d < r2) {
                const int slot = atomicAdd(&s_cnt, 1);
                gd[slot] = d;
                gi[slot] = off + j;
            }
        }
        __syncthreads();
        for (int e = threadIdx.x; e < cnt; e += RN_THREADS) {
            const double de = gd[e];
            const int ie = gi[e];
            int rank = 0;
            for (int j = 0; j < cnt; ++j) rank += nd_less(gd[j], gi[j], de, ie) ? 1 : 0;
            row[rank] = ie;
        }
        for (int j = cnt + threadIdx.x; j < cap; j += RN_THREADS) row[j] = bt.ns_total;
        return;
    }
    const int m = min(cnt, RN_CAP);
    int p2 = 1;
    while (p2 < m) p2 <<= 1;
    for (int j = m + threadIdx.x; j < p2; j += RN_THREADS) { sd[j] = 1e300; si[j] = 0x7fffffff; }
    __syncthreads();
    for (int k = 2; k <= p2; k <<= 1)
        for (int jj = k >> 1; jj > 0; jj >>= 1) {
            for (int t = threadIdx.x; t < p2; t += RN_THREADS) {
                const int l = t ^ jj;
                if (l > t) {
                    const bool up = (t & k) == 0;
                    const double da = sd[t], db = sd[l];
                    const int ia = si[t], ib = si[l];
                    const bool sw = up ? nd_less(db, ib, da, ia) : nd_less(da, ia, db, ib);
                    if (sw) { sd[t] = db; sd[l] = da; si[t] = ib; si[l] = ia; }
                }
            }
            __syncthreads();
        }
    int *row = out + (size_t)i * cap;
    for (int j = threadIdx.x; j < cap; j += RN_THREADS) row[j] = (j < m) ? si[j] : bt.ns_total;
}

// ---- a18 --------------------------------------------------------------------------------------------------
// Empty-slot marker of the cell table.  Keys wrap modulo 2^64 (a cell index of -1 gives keys just below 2^64, 2^64-1
// itself included), so ~0 cannot mark an empty slot; 0x8080... (a memset byte) is reached only by a grid of more
// than 9e18 cells.
constexpr unsigned long long GRID_EMPTY = 0x8080808080808080ull;

struct GridGeom {
    float org[3];
    float dl;
    unsigned long long NX, NY;
};

__global__ void minmax_kernel(const float *__restrict__ pts, int n, float *__restrict__ mm /* 6: min xyz, max xyz as ordered ints */) {
    __shared__ float smn[3][32], smx[3][32];
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v = pts[3 * (size_t)i + c];
            mn[c] = fminf(mn[c], v);
            mx[c] = fmaxf(mx[c], v);
        }
#pragma unroll
    for (int c = 0; c < 3; ++c)
        for (int o = 16; o >= 1; o >>= 1) {
            mn[c] = fminf(mn[c], __shfl_xor_sync(BX_FULL, mn[c], o));
            mx[c] = fmaxf(mx[c], __shfl_xor_sync(BX_FULL, mx[c], o));
        }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0)
        for (int c = 0; c < 3; ++c) { smn[c][w] = mn[c]; smx[c][w] = mx[c]; }
    __syncthreads();
    if (w == 0) {
        const int nw = blockDim.x >> 5;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float a = lane < nw ? smn[c][lane] : INFINITY, b2 = lane < nw ? smx[c][lane] : -INFINITY;
            for (int o = 16; o >= 1; o >>= 1) {
                a = fminf(a, __shfl_xor_sync(BX_FULL, a, o));
                b2 = fmaxf(b2, __shfl_xor_sync(BX_FULL, b2, o));
            }
            if (lane == 0) {
                // order-preserving int encoding so that atomicMin / atomicMax on ints work for floats
                const int ia = __float_as_int(a), ib = __float_as_int(b2);
                atomicMin(reinterpret_cast<int *>(mm) + c, ia >= 0 ? ia : ia ^ 0x7fffffff);
                atomicMax(reinterpret_cast<int *>(mm) + 3 + c, ib >= 0 ? ib : ib ^ 0x7fffffff);
            }
        }
    }
}

__device__ __forceinline__ float decode_ordered(int v) { return __int_as_float(v >= 0 ? v : v ^ 0x7fffffff); }

__global__ void grid_insert_kernel(const float *__restrict__ pts, int n, float dl, const float *__restrict__ mm,
                                   unsigned long long *__restrict__ tkeys, float *__restrict__ tacc, int tcap) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int *mi = reinterpret_cast<const int *>(mm);
    const float inv = 1.0f / dl;
    float org[3], mx[2];
#pragma unroll
    for (int c = 0; c < 3; ++c) org[c] = floorf(decode_ordered(mi[c]) * inv) * dl;
    mx[0] = decode_ordered(mi[3]);
    mx[1] = decode_ordered(mi[4]);
    // The grid dimensions wrap the same way: a flat axis whose origin rounded above it gives floor = -1, hence NX = 0
    // (or NY = 0) in the reference, and every point of the cloud shares its aliased keys.
    const unsigned long long NX = (unsigned long long)(long long)floorf((mx[0] - org[0]) / dl) + 1ull;
    const unsigned long long NY = (unsigned long long)(long long)floorf((mx[1] - org[1]) / dl) + 1ull;
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    // The fp32 origin can round above the minimum (dl = 0.025, min 40.6f: origin 40.600002), giving a cell index of -1.
    // The reference's (size_t)floor(-1.f) is 2^64-1 on x86 (cvttss2si), so its key aliases cell (NX-1, iY-1, iZ); a
    // direct float -> u64 cvt clamps to 0 instead.  Going through long long wraps like the reference.
    const unsigned long long ix = (unsigned long long)(long long)floorf((x - org[0]) / dl),
                             iy = (unsigned long long)(long long)floorf((y - org[1]) / dl),
                             iz = (unsigned long long)(long long)floorf((z - org[2]) / dl);
    const unsigned long long key = ix + NX * iy + NX * NY * iz;
    unsigned long long h = key * 0x9E3779B97F4A7C15ull;
    unsigned slot = (unsigned)(h >> 32) & (unsigned)(tcap - 1);
    while (true) {
        const unsigned long long prev = atomicCAS(&tkeys[slot], GRID_EMPTY, key);
        if (prev == GRID_EMPTY || prev == key) break;
        slot = (slot + 1) & (unsigned)(tcap - 1);
    }
    atomicAdd(&tacc[4 * (size_t)slot], x);
    atomicAdd(&tacc[4 * (size_t)slot + 1], y);
    atomicAdd(&tacc[4 * (size_t)slot + 2], z);
    atomicAdd(reinterpret_cast<int *>(&tacc[4 * (size_t)slot + 3]), 1);
}

__global__ void grid_emit_kernel(const unsigned long long *__restrict__ tkeys, const float *__restrict__ tacc, int tcap,
                                 unsigned long long *__restrict__ keys_out, float *__restrict__ xyz_out, int *__restrict__ cnt_out,
                                 int *__restrict__ d_m) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= tcap) return;
    const unsigned long long k = tkeys[s];
    if (k == GRID_EMPTY) return;
    const int c = *reinterpret_cast<const int *>(&tacc[4 * (size_t)s + 3]);
    const int o = atomicAdd(d_m, 1);
    const float a = (float)(1.0 / (double)c);
    keys_out[o] = k;
    xyz_out[3 * (size_t)o] = tacc[4 * (size_t)s] * a;
    xyz_out[3 * (size_t)o + 1] = tacc[4 * (size_t)s + 1] * a;
    xyz_out[3 * (size_t)o + 2] = tacc[4 * (size_t)s + 2] * a;
    if (cnt_out) cnt_out[o] = c;
}

}  // namespace

BX_API int bx_radius_neighbors(const float *queries, int nq, const float *supports, int ns, const int32_t *h_q_batches, int nqb,
                               const int32_t *h_s_batches, int nsb, float radius, int32_t *out, int cap, int32_t *d_max_count,
                               double *scratch_d, int32_t *scratch_i, void *stream) {
    BX_REQUIRE(queries && supports && h_q_batches && h_s_batches && d_max_count, "bx_radius_neighbors: null pointer");
    BX_REQUIRE(nq >= 0 && ns >= 0 && nqb >= 1 && nqb <= 8 && nsb >= 1 && nsb <= 2, "bx_radius_neighbors: 1..8 query batches, 1..2 support clouds");
    BX_REQUIRE(out == nullptr || cap >= 1, "bx_radius_neighbors: capacity must be >= 1");
    BX_REQUIRE(out == nullptr || cap <= RN_CAP || (scratch_d && scratch_i), "bx_radius_neighbors: more than %d neighbours per ball need the global scratch rows", RN_CAP);
    Batches bt = {};
    bt.nqb = nqb;
    int acc = 0;
    for (int k = 0; k < nqb; ++k) { bt.q_acc[k] = acc; acc += h_q_batches[k]; }
    bt.q_acc[nqb] = acc;
    BX_REQUIRE(acc == nq, "bx_radius_neighbors: query batches sum to %d, nq = %d", acc, nq);
    bt.s0 = h_s_batches[0];
    bt.s1 = nsb > 1 ? h_s_batches[1] : 0;
    bt.ns_total = ns;
    BX_REQUIRE(bt.s0 + bt.s1 <= ns, "bx_radius_neighbors: support batches exceed ns");
    cudaStream_t st = bx_stream(stream);
    BX_CUDA(cudaMemsetAsync(d_max_count, 0, sizeof(int), st));
    if (nq == 0) return BX_OK;
    const size_t smem = RN_CAP * (sizeof(double) + sizeof(int));
    static BxPerDevice attr_done = {};
    if (bx_needs_attr(attr_done))
        BX_CUDA(cudaFuncSetAttribute(radius_neighbors_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    radius_neighbors_kernel<<<nq, RN_THREADS, smem, st>>>(queries, nq, supports, bt, radius, out, cap, d_max_count, scratch_d, scratch_i);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_grid_subsample(const float *pts, int n, float dl, unsigned long long *table_keys, float *table_acc, int table_cap,
                             float *minmax6, unsigned long long *keys_out, float *xyz_out, int32_t *cnt_out, int32_t *d_m,
                             void *stream) {
    BX_REQUIRE(pts && table_keys && table_acc && minmax6 && keys_out && xyz_out && d_m, "bx_grid_subsample: null pointer");
    BX_REQUIRE(n >= 1 && dl > 0.0f, "bx_grid_subsample: bad arguments");
    BX_REQUIRE(table_cap >= 2 * n && (table_cap & (table_cap - 1)) == 0, "bx_grid_subsample: table_cap must be a power of two >= 2n");
    cudaStream_t st = bx_stream(stream);
    BX_CUDA(cudaMemsetAsync(table_keys, 0x80, sizeof(unsigned long long) * (size_t)table_cap, st));   // GRID_EMPTY
    BX_CUDA(cudaMemsetAsync(table_acc, 0, sizeof(float) * 4 * (size_t)table_cap, st));
    BX_CUDA(cudaMemsetAsync(d_m, 0, sizeof(int), st));
    // min -> +inf (0x7f800000), max -> -inf encoded: ordered-int(-inf) = 0xff800000 ^ 0x7fffffff = 0x807fffff
    const int init[6] = {0x7f800000, 0x7f800000, 0x7f800000, (int)0x807fffff, (int)0x807fffff, (int)0x807fffff};
    BX_CUDA(cudaMemcpyAsync(minmax6, init, sizeof(init), cudaMemcpyHostToDevice, st));
    int blocks = (n + 255) / 256;
    if (blocks > 592) blocks = 592;
    minmax_kernel<<<blocks, 256, 0, st>>>(pts, n, minmax6);
    BX_LAUNCH_CHECK();
    grid_insert_kernel<<<(n + 255) / 256, 256, 0, st>>>(pts, n, dl, minmax6, table_keys, table_acc, table_cap);
    BX_LAUNCH_CHECK();
    grid_emit_kernel<<<(table_cap + 255) / 256, 256, 0, st>>>(table_keys, table_acc, table_cap, keys_out, xyz_out, cnt_out, d_m);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
