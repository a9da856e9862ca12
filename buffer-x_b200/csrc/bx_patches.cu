// bx_patches.cu -- a3 (order-preserving radius-neighbour patch gathering) and a4+a5 (LRF, normalise).
//
// a3 replaces MiniSpinNet.select_patches (/root/reference/models/patch_embedder.py:92-120), i.e.
// pointnet2_ops.ball_query (ONE CTA for the whole cloud when B=1) + grouping_operation + four
// full-size mask temporaries.  Semantics: "the first P points of the permuted cloud, in index order,
// inside the ball" -- not the P nearest.  One WARP per key-point scans the permuted cloud (float4,
// coalesced 512-byte warp loads, L1/L2 resident: the cloud is 320 KB) in chunks of 128 points; a
// ballot + popcount prefix compacts the hits in order, and the scan stops as soon as P slots are
// filled.  Indices and gathered coordinates are written straight from the registers that just
// tested the point.
// a4+a5 replace axis_align / normalize (patch_embedder.py:122-148,167-170), cal_Z_axis
// (utils/common.py:709-726: torch_batch_svd -> cuSOLVER gesvdjBatched on K 3x3 matrices) and
// RodsRotatFormula (:501-525): one warp per patch, covariance by lane-strided sums + xor butterfly,
// fp64 cyclic Jacobi in registers, Rodrigues from cos = z_z/|z|, sin = |z x e_z|/|z|.
//
// Bit contract: oracle/c/bx_oracle.c::bxo_ball_query / bxo_select_patches / bxo_lrf.  -fmad=false.
#include "bx_common.cuh"

namespace {

__global__ void permute_cloud_kernel(const float *__restrict__ pts, const int *__restrict__ perm, int N,
                                     float4 *__restrict__ out, const int *__restrict__ d_N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (d_N ? min(max(*d_N, 0), N) : N)) return;
    const int s = perm ? perm[i] : i;
    out[i] = make_float4(pts[3 * (size_t)s], pts[3 * (size_t)s + 1], pts[3 * (size_t)s + 2], 0.0f);
}

// SP_KP key-points per CTA, SP_SPLIT warps per key-point.  The cloud is streamed through shared memory in chunks of
// SP_CH points; the SP_SPLIT warps of a key-point scan consecutive quarters of a chunk, exchange their hit counts
// through shared memory and write their hits at the ordered offsets -- the serial scan of one warp per key-point was a
// ~100 K-cycle dependent chain with 10 warps per SM; splitting it four ways (and keeping 16 warps per CTA) cuts the
// chain and raises the occupancy.  The scan order, and with it every index and coordinate, is unchanged.
constexpr int SP_KP = 4;
constexpr int SP_SPLIT = 4;
constexpr int SP_WARPS = SP_KP * SP_SPLIT;
constexpr int SP_CH = 2048;
constexpr int SP_SUB = SP_CH / SP_SPLIT;      // points of a chunk scanned by one warp
constexpr int SP_STEPS = SP_SUB / 32;         // ballots per warp and chunk
constexpr int BQ_WARPS = 8;

__device__ __forceinline__ void select_patches_body(const float4 *__restrict__ pts4, int N, const float *__restrict__ kpts, int K, float radius,
                                                    const float *__restrict__ d_radius, int P, int *__restrict__ idx, float *__restrict__ patches,
                                                    int block) {
    __shared__ float4 tile[SP_CH];
    __shared__ int s_cnt[SP_KP][SP_SPLIT], s_first[SP_KP][SP_SPLIT];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int kl = warp / SP_SPLIT, part = warp % SP_SPLIT;      // key-point of the CTA, quarter of the chunk
    const int k = block * SP_KP + kl;
    const bool valid = k < K;
    const int kk = valid ? k : K - 1;
    const float r = d_radius ? *d_radius : radius;
    const float r2 = r * r;
    const float qx = kpts[3 * (size_t)kk], qy = kpts[3 * (size_t)kk + 1], qz = kpts[3 * (size_t)kk + 2];
    int *row = idx ? idx + (size_t)kk * P : nullptr;
    float *out = patches + (size_t)kk * P * 3;
    int cnt = 0, first = 0;                    // hits of the key-point so far / index of its first hit (same in its 4 warps)
    bool done = !valid;
    constexpr int LD = SP_CH / (SP_WARPS * 32);          // float4 loads per thread and chunk
    float4 stage[LD];                                    // the next chunk travels through registers: its L2 latency
#pragma unroll                                           // overlaps the scan of the current one
    for (int q = 0; q < LD; ++q) {
        const int i = q * SP_WARPS * 32 + tid;
        stage[q] = (i < N) ? __ldg(pts4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int base0 = 0; base0 < N; base0 += SP_CH) {
#pragma unroll
        for (int q = 0; q < LD; ++q) tile[q * SP_WARPS * 32 + tid] = stage[q];
        __syncthreads();
#pragma unroll
        for (int q = 0; q < LD; ++q) {
            const int i = base0 + SP_CH + q * SP_WARPS * 32 + tid;
            stage[q] = (i < N) ? __ldg(pts4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        const int lim = min(SP_CH, N - base0);
        unsigned masks[SP_STEPS];
        int c_w = 0, f_w = 0x7fffffff;
        if (!done) {
#pragma unroll
            for (int st = 0; st < SP_STEPS; ++st) {
                const int j = part * SP_SUB + st * 32 + lane;
                const float4 p = tile[j];
                const float d2 = bx_d2(qx - p.x, qy - p.y, qz - p.z);
                const unsigned m = __ballot_sync(BX_FULL, (j < lim) && (d2 < r2));
                masks[st] = m;
                if (m && c_w == 0) f_w = base0 + part * SP_SUB + st * 32 + (__ffs(m) - 1);
                c_w += __popc(m);
            }
            if (lane == 0) { s_cnt[kl][part] = c_w; s_first[kl][part] = f_w; }
        }
        __syncthreads();
        if (!done) {
            int off = cnt, tot = 0;
#pragma unroll
            for (int w = 0; w < SP_SPLIT; ++w) {
                const int c = s_cnt[kl][w];
                if (w < part) off += c;
                if (cnt == 0 && tot == 0 && c > 0) first = s_first[kl][w];
                tot += c;
            }
            if (c_w > 0 && off < P) {
#pragma unroll
                for (int st = 0; st < SP_STEPS; ++st) {
                    const unsigned m = masks[st];
                    if (m) {
                        const int slot = off + __popc(m & ((1u << lane) - 1u));
                        if (((m >> lane) & 1u) && slot < P) {
                            const int j = part * SP_SUB + st * 32 + lane;
                            const float4 p = tile[j];
                            if (row) row[slot] = base0 + j;
                            // slot P-1 always holds the key-point itself (patch_embedder.py:109)
                            const bool centre = (slot == P - 1);
                            out[3 * slot] = centre ? qx : p.x;
                            out[3 * slot + 1] = centre ? qy : p.y;
                            out[3 * slot + 2] = centre ? qz : p.z;
                        }
                        off += __popc(m);
                    }
                }
            }
            cnt += tot;
            if (cnt >= P) done = true;
        }
        if (!__syncthreads_or(!done)) break;    // barrier: tile / counters may be overwritten; all key-points full -> stop
    }
    if (!valid || part != 0) return;
    if (cnt > P) cnt = P;
    // padding: ball_query repeats the first hit; the fix-up replaces those slots by the key-point.
    // No hit at all: index row = 0, slot 0 = point 0 of the permuted cloud, every other slot = key-point.
    for (int s = cnt + lane; s < P; s += 32) {
        if (row) row[s] = first;
        float x = qx, y = qy, z = qz;
        if (cnt == 0 && s == 0 && P > 1) {
            const float4 p0 = pts4[0];
            x = p0.x; y = p0.y; z = p0.z;
        }
        out[3 * s] = x;
        out[3 * s + 1] = y;
        out[3 * s + 2] = z;
    }
}

__global__ void __launch_bounds__(SP_WARPS * 32)
select_patches_kernel(const float4 *__restrict__ pts4, int N, const float *__restrict__ kpts, int K, float radius,
                      const float *__restrict__ d_radius, int P, int *__restrict__ idx, float *__restrict__ patches) {
    select_patches_body(pts4, N, kpts, K, radius, d_radius, P, idx, patches, blockIdx.x);
}

// All (cloud, scale) key-point sets of a pair in ONE launch: job j = (permuted cloud j, key-points j, device radius j); its
// patches are rows [koff_j, koff_j + K_j) of one buffer.  Six launches of 375 CTAs (2.5 per SM) become one of 2250.
constexpr int SP_MAXJOBS = 16;
struct SpJobs {
    const float4 *pts4[SP_MAXJOBS];
    const float *kpts[SP_MAXJOBS];
    const float *d_radius[SP_MAXJOBS];
    const int *d_K[SP_MAXJOBS];           // optional device key-point count of a job (NULL: K)
    const int *d_N[SP_MAXJOBS];           // optional device point count of a job (NULL: N = the capacity)
    int N[SP_MAXJOBS], K[SP_MAXJOBS], boff[SP_MAXJOBS + 1], koff[SP_MAXJOBS];
    int njobs;
};

// key-points of a job present this launch: min(*d_K, K), or K without a device count
__device__ __forceinline__ int sp_count(const int *d_K, int K) { return d_K ? min(max(*d_K, 0), K) : K; }
// points of a job's permuted cloud present this launch: min(*d_N, N) (at least 1), or N without a device count
__device__ __forceinline__ int sp_points(const int *d_N, int N) { return d_N ? min(max(*d_N, 1), N) : N; }

__global__ void __launch_bounds__(SP_WARPS * 32)
select_patches_batched_kernel(const SpJobs jobs, int P, float *__restrict__ patches) {
    int j = 0;
    while (j + 1 < jobs.njobs && (int)blockIdx.x >= jobs.boff[j + 1]) ++j;
    const int b = (int)blockIdx.x - jobs.boff[j], Kj = sp_count(jobs.d_K[j], jobs.K[j]);
    if (b * SP_KP >= Kj) return;                          // the whole CTA: before any barrier
    select_patches_body(jobs.pts4[j], sp_points(jobs.d_N[j], jobs.N[j]), jobs.kpts[j], Kj, 0.0f, jobs.d_radius[j], P, nullptr,
                        patches + (size_t)jobs.koff[j] * P * 3, b);
}

// ---- hash-grid form of select_patches (large clouds: N >= ~50 k points) --------------------------------------------------
// The streaming kernel reads the permuted cloud front to back until a key-point has its P hits: fine when a ball holds a
// few per cent of the cloud (C2: 20 k points), wasteful for a LiDAR-sized cloud (C3: 120 k points, a ball holds < 2 %).
// Here the cloud is binned into a spatial hash of cubic cells of edge >= radius (classic three-prime hash of the integer
// cell coordinates, 2^17 buckets: no bounding box needed, aliases only add candidates), and a key-point looks at the 27
// cells around it only.  The ORDER contract (first P hits in permuted-index order, patch_embedder.py:92-120) does not
// need a sort: hits set bits in a per-key-point bitmap over the point indices (N / 8 bytes of shared memory), and the
// bitmap is read back front to back -- counts per thread range, a block scan, then every thread emits the hits of its
// range at their ordered slots.  Membership is the same exact test d2 < r*r as everywhere, so index rows and patches are
// bit-identical to the streaming kernel (tests/test_gpu_parity.py::test_select_patches_grid_equals_scan).
constexpr int HG_BITS = 17, HG_CELLS = 1 << HG_BITS;
constexpr int HG_THREADS = 128;

__device__ __forceinline__ int hg_coord(float v, float inv_cell) { return (int)floorf(v * inv_cell); }
__device__ __forceinline__ unsigned hg_hash(int ix, int iy, int iz) {
    return ((unsigned)ix * 73856093u ^ (unsigned)iy * 19349663u ^ (unsigned)iz * 83492791u) & (unsigned)(HG_CELLS - 1);
}
// cell edge = radius * (1 + 1e-3): two points closer than the radius then differ by less than one cell in exact arithmetic
// with 1e-3 of slack for the fp32 rounding of v * inv_cell (|v| / cell < 2^13 cells keeps that error below 1e-3)
__device__ __forceinline__ float hg_inv_cell(float r) { return 1.0f / (r * 1.001f); }

__device__ __forceinline__ void hg_count_body(const float4 *__restrict__ pts4, int N, const float *__restrict__ d_radius, int *__restrict__ cnt, int i) {
    if (i >= N) return;
    const float ic = hg_inv_cell(*d_radius);
    const float4 p = pts4[i];
    atomicAdd(cnt + hg_hash(hg_coord(p.x, ic), hg_coord(p.y, ic), hg_coord(p.z, ic)), 1);
}
__global__ void hg_count_kernel(const float4 *__restrict__ pts4, int N, const float *__restrict__ d_radius, int *__restrict__ cnt) {
    hg_count_body(pts4, N, d_radius, cnt, blockIdx.x * blockDim.x + threadIdx.x);
}

// exclusive scan of the HG_CELLS bucket counts (one CTA of 1024 threads, 128 consecutive buckets per thread, 16-byte accesses);
// cursor = start
__device__ __forceinline__ void hg_scan_body(const int *__restrict__ cnt, int *__restrict__ start, int *__restrict__ cursor) {
    __shared__ int sh[33];
    constexpr int PER4 = HG_CELLS / 1024 / 4;
    const int t = threadIdx.x;
    const int4 *c4 = reinterpret_cast<const int4 *>(cnt) + (size_t)t * PER4;
    int local = 0;
#pragma unroll 8
    for (int j = 0; j < PER4; ++j) { const int4 v = c4[j]; local += (v.x + v.y) + (v.z + v.w); }
    int total;
    int run = bx_block_exscan(local, sh, &total);
    int4 *s4 = reinterpret_cast<int4 *>(start) + (size_t)t * PER4, *u4 = reinterpret_cast<int4 *>(cursor) + (size_t)t * PER4;
#pragma unroll 8
    for (int j = 0; j < PER4; ++j) {
        const int4 v = c4[j];
        int4 o;
        o.x = run; o.y = o.x + v.x; o.z = o.y + v.y; o.w = o.z + v.z;
        run = o.w + v.w;
        s4[j] = o;
        u4[j] = o;
    }
    if (t == 1023) start[HG_CELLS] = run;
}
__global__ void __launch_bounds__(1024) hg_scan_kernel(const int *__restrict__ cnt, int *__restrict__ start, int *__restrict__ cursor) { hg_scan_body(cnt, start, cursor); }

__device__ __forceinline__ void hg_scatter_body(const float4 *__restrict__ pts4, int N, const float *__restrict__ d_radius, int *__restrict__ cursor,
                                                float4 *__restrict__ sorted, int i) {
    if (i >= N) return;
    const float ic = hg_inv_cell(*d_radius);
    const float4 p = pts4[i];
    const int pos = atomicAdd(cursor + hg_hash(hg_coord(p.x, ic), hg_coord(p.y, ic), hg_coord(p.z, ic)), 1);
    sorted[pos] = make_float4(p.x, p.y, p.z, __int_as_float(i));        // the order inside a bucket does not matter (bitmap)
}
__global__ void hg_scatter_kernel(const float4 *__restrict__ pts4, int N, const float *__restrict__ d_radius, int *__restrict__ cursor,
                                  float4 *__restrict__ sorted) {
    hg_scatter_body(pts4, N, d_radius, cursor, sorted, blockIdx.x * blockDim.x + threadIdx.x);
}

__device__ __forceinline__ void hg_query_body(const float4 *__restrict__ pts4, int N, const float *__restrict__ kpts, const float *__restrict__ d_radius, int P,
                                              const int *__restrict__ start, const float4 *__restrict__ sorted, int *__restrict__ idx,
                                              float *__restrict__ patches, int k) {
    extern __shared__ unsigned hg_bits[];                 // (N + 31) / 32 words
    __shared__ int sh[33];
    __shared__ int s_first;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int W = (N + 31) >> 5;
    const float r = *d_radius, r2 = r * r, ic = hg_inv_cell(r);
    const float qx = kpts[3 * (size_t)k], qy = kpts[3 * (size_t)k + 1], qz = kpts[3 * (size_t)k + 2];
    for (int w = tid; w < W; w += HG_THREADS) hg_bits[w] = 0u;
    if (tid == 0) s_first = 0x7fffffff;
    __syncthreads();
    const int cx = hg_coord(qx, ic), cy = hg_coord(qy, ic), cz = hg_coord(qz, ic);
    for (int c = warp; c < 27; c += HG_THREADS / 32) {
        const unsigned h = hg_hash(cx + c % 3 - 1, cy + (c / 3) % 3 - 1, cz + c / 9 - 1);
        const int s = start[h], e = start[h + 1];
        for (int j = s + lane; j < e; j += 32) {
            const float4 p = sorted[j];
            if (bx_d2(qx - p.x, qy - p.y, qz - p.z) < r2) {
                const int i = __float_as_int(p.w);
                atomicOr(&hg_bits[i >> 5], 1u << (i & 31));
            }
        }
    }
    __syncthreads();
    // ordered read-back: thread t owns the contiguous word range [w0, w1)
    const int per = (W + HG_THREADS - 1) / HG_THREADS, w0 = min(tid * per, W), w1 = min(w0 + per, W);
    int local = 0;
    for (int w = w0; w < w1; ++w) local += __popc(hg_bits[w]);
    int total;
    int off = bx_block_exscan(local, sh, &total);
    int *row = idx ? idx + (size_t)k * P : nullptr;
    float *out = patches + (size_t)k * P * 3;
    if (local > 0 && off == 0) {                          // the thread that holds the first hit
        for (int w = w0; w < w1; ++w) if (hg_bits[w]) { s_first = (w << 5) + __ffs(hg_bits[w]) - 1; break; }
    }
    for (int w = w0; w < w1 && off < P; ++w) {
        unsigned m = hg_bits[w];
        while (m && off < P) {
            const int b = __ffs(m) - 1;
            m &= m - 1;
            const int i = (w << 5) + b;
            if (row) row[off] = i;
            const bool centre = (off == P - 1);            // slot P-1 always holds the key-point itself (patch_embedder.py:109)
            const float4 p = pts4[i];
            out[3 * off] = centre ? qx : p.x;
            out[3 * off + 1] = centre ? qy : p.y;
            out[3 * off + 2] = centre ? qz : p.z;
            ++off;
        }
    }
    __syncthreads();
    // padding: ball_query repeats the first hit; the fix-up replaces those slots by the key-point.
    // No hit at all: index row = 0, slot 0 = point 0 of the permuted cloud, every other slot = key-point.
    const int cnt = min(total, P);
    const int first = cnt > 0 ? s_first : 0;
    for (int s = cnt + tid; s < P; s += HG_THREADS) {
        if (row) row[s] = first;
        float x = qx, y = qy, z = qz;
        if (cnt == 0 && s == 0 && P > 1) { const float4 p0 = pts4[0]; x = p0.x; y = p0.y; z = p0.z; }
        out[3 * s] = x; out[3 * s + 1] = y; out[3 * s + 2] = z;
    }
}

__global__ void __launch_bounds__(HG_THREADS)
hg_query_kernel(const float4 *__restrict__ pts4, int N, const float *__restrict__ kpts, int K, const float *__restrict__ d_radius, int P,
                const int *__restrict__ start, const float4 *__restrict__ sorted, int *__restrict__ idx, float *__restrict__ patches) {
    hg_query_body(pts4, N, kpts, d_radius, P, start, sorted, idx, patches, blockIdx.x);
}

// all (cloud, scale) jobs of a pair: one launch per phase (blockIdx.y = job for the point-parallel phases)
struct HgJobs {
    const float4 *pts4[SP_MAXJOBS];
    const float *kpts[SP_MAXJOBS];
    const float *d_radius[SP_MAXJOBS];
    float4 *sorted[SP_MAXJOBS];
    int *cnt[SP_MAXJOBS];                 // cnt, start = cnt + HG_CELLS, cursor = start + HG_CELLS + 4
    const int *d_K[SP_MAXJOBS];           // optional device key-point count of a job: 0 skips every phase of the job
    const int *d_N[SP_MAXJOBS];           // optional device point count of a job (NULL: N = the capacity the workspace is laid out for)
    int N[SP_MAXJOBS], koff[SP_MAXJOBS + 1];
    int njobs;
};
__global__ void hg_count_batched_kernel(const HgJobs J) {
    const int j = blockIdx.y;
    if (J.d_K[j] && *J.d_K[j] <= 0) return;
    hg_count_body(J.pts4[j], sp_points(J.d_N[j], J.N[j]), J.d_radius[j], J.cnt[j], blockIdx.x * blockDim.x + threadIdx.x);
}
__global__ void __launch_bounds__(1024) hg_scan_batched_kernel(const HgJobs J) {
    if (J.d_K[blockIdx.x] && *J.d_K[blockIdx.x] <= 0) return;
    int *cnt = J.cnt[blockIdx.x];
    hg_scan_body(cnt, cnt + HG_CELLS, cnt + 2 * HG_CELLS + 4);
}
// The same scan spread over HG_CHUNKS CTAs per job (one CTA per job scanning 131072 buckets is a long latency chain on six
// SMs): chunk totals first, then every chunk scans its 4096 buckets from the sum of the
// totals before it.  Totals live behind the cursor array (workspace ints [3 * HG_CELLS + 8, + HG_CHUNKS)).
constexpr int HG_CHUNK = 4096, HG_CHUNKS = HG_CELLS / HG_CHUNK, HG_SCAN_THREADS = 256;
__global__ void __launch_bounds__(HG_SCAN_THREADS) hg_chunksum_batched_kernel(const HgJobs J) {
    __shared__ int sh[33];
    if (J.d_K[blockIdx.y] && *J.d_K[blockIdx.y] <= 0) return;
    const int *cnt = J.cnt[blockIdx.y] + (size_t)blockIdx.x * HG_CHUNK;
    const int4 *c4 = reinterpret_cast<const int4 *>(cnt) + threadIdx.x * (HG_CHUNK / HG_SCAN_THREADS / 4);
    int local = 0;
#pragma unroll
    for (int j = 0; j < HG_CHUNK / HG_SCAN_THREADS / 4; ++j) { const int4 v = c4[j]; local += (v.x + v.y) + (v.z + v.w); }
    int total;
    bx_block_exscan(local, sh, &total);
    if (threadIdx.x == 0) J.cnt[blockIdx.y][3 * HG_CELLS + 8 + blockIdx.x] = total;
}
__global__ void __launch_bounds__(HG_SCAN_THREADS) hg_chunkscan_batched_kernel(const HgJobs J) {
    __shared__ int sh[33];
    if (J.d_K[blockIdx.y] && *J.d_K[blockIdx.y] <= 0) return;
    int *base = J.cnt[blockIdx.y];
    const int chunk = blockIdx.x;
    // sum of the totals of the chunks before this one (HG_CHUNKS = 32: one warp-wide sum, computed by every warp)
    const int lane = threadIdx.x & 31;
    int before = (lane < chunk) ? base[3 * HG_CELLS + 8 + lane] : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(BX_FULL, before, o);
    constexpr int PER4 = HG_CHUNK / HG_SCAN_THREADS / 4;
    const size_t off4 = ((size_t)chunk * HG_CHUNK) / 4 + (size_t)threadIdx.x * PER4;
    const int4 *c4 = reinterpret_cast<const int4 *>(base) + off4;
    int4 v[PER4];
    int local = 0;
#pragma unroll
    for (int j = 0; j < PER4; ++j) { v[j] = c4[j]; local += (v[j].x + v[j].y) + (v[j].z + v[j].w); }
    int total;
    int run = before + bx_block_exscan(local, sh, &total);
    int4 *s4 = reinterpret_cast<int4 *>(base + HG_CELLS) + off4, *u4 = reinterpret_cast<int4 *>(base + 2 * HG_CELLS + 4) + off4;
#pragma unroll
    for (int j = 0; j < PER4; ++j) {
        int4 o;
        o.x = run; o.y = o.x + v[j].x; o.z = o.y + v[j].y; o.w = o.z + v[j].z;
        run = o.w + v[j].w;
        s4[j] = o;
        u4[j] = o;
    }
    if (chunk == HG_CHUNKS - 1 && threadIdx.x == HG_SCAN_THREADS - 1) base[HG_CELLS + HG_CELLS] = run;      // start[HG_CELLS] = N
}
__global__ void hg_scatter_batched_kernel(const HgJobs J) {
    const int j = blockIdx.y;
    if (J.d_K[j] && *J.d_K[j] <= 0) return;
    hg_scatter_body(J.pts4[j], sp_points(J.d_N[j], J.N[j]), J.d_radius[j], J.cnt[j] + 2 * HG_CELLS + 4, J.sorted[j],
                    blockIdx.x * blockDim.x + threadIdx.x);
}
__global__ void __launch_bounds__(HG_THREADS) hg_query_batched_kernel(const HgJobs J, int P, float *__restrict__ patches) {
    int j = 0;
    while (j + 1 < J.njobs && (int)blockIdx.x >= J.koff[j + 1]) ++j;
    const int k = (int)blockIdx.x - J.koff[j];
    if (J.d_K[j] && k >= *J.d_K[j]) return;               // the whole CTA: before any barrier
    hg_query_body(J.pts4[j], sp_points(J.d_N[j], J.N[j]), J.kpts[j], J.d_radius[j], P, J.cnt[j] + HG_CELLS, J.sorted[j], nullptr,
                  patches + (size_t)J.koff[j] * P * 3, k);
}

// plain ordered ball query over a packed [n,3] cloud (pointnet2_ops.ball_query semantics)
__global__ void __launch_bounds__(BQ_WARPS * 32)
ball_query_kernel(const float *__restrict__ xyz, int n, const float *__restrict__ qry, int m, float radius, int nsample,
                  int *__restrict__ idx) {
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * BQ_WARPS + (threadIdx.x >> 5);
    if (j >= m) return;
    const float r2 = radius * radius;
    const float qx = qry[3 * (size_t)j], qy = qry[3 * (size_t)j + 1], qz = qry[3 * (size_t)j + 2];
    int *row = idx + (size_t)j * nsample;
    int cnt = 0, first = 0;
    for (int base = 0; base < n && cnt < nsample; base += 32) {
        const int i = base + lane;
        bool hit = false;
        if (i < n) {
            const float d2 = bx_d2(qx - xyz[3 * (size_t)i], qy - xyz[3 * (size_t)i + 1], qz - xyz[3 * (size_t)i + 2]);
            hit = d2 < r2;
        }
        const unsigned msk = __ballot_sync(BX_FULL, hit);
        if (msk) {
            if (cnt == 0) first = base + (__ffs(msk) - 1);
            const int slot = cnt + __popc(msk & ((1u << lane) - 1u));
            if (hit && slot < nsample) row[slot] = i;
            cnt += __popc(msk);
        }
    }
    if (cnt > nsample) cnt = nsample;
    for (int s = cnt + lane; s < nsample; s += 32) row[s] = first;
}

// ---- LRF ------------------------------------------------------------------------------------------
__device__ __forceinline__ void jacobi_rot3(double (&A)[3][3], double (&V)[3][3], const int p, const int q) {
    const double apq = A[p][q];
    if (apq == 0.0) return;
    const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
    const double at = fabs(theta);
    double t = 1.0 / (at + sqrt((theta * theta) + 1.0));
    if (theta < 0.0) t = -t;
    const double c = 1.0 / sqrt((t * t) + 1.0);
    const double s = t * c;
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
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double vkp = V[k][p], vkq = V[k][q];
        V[k][p] = (c * vkp) - (s * vkq);
        V[k][q] = (s * vkp) + (c * vkq);
    }
}

constexpr int LRF_WARPS = 4;

__global__ void __launch_bounds__(LRF_WARPS * 32)
lrf_kernel(const float *__restrict__ patches, int K, int P, float des_r_v, const float *__restrict__ d_des_r, int flags,
           float *__restrict__ delta, float *__restrict__ Rt, float *__restrict__ rand_axis, int r_group, const int *__restrict__ d_K) {
    const int aligned = flags & 1, stable = flags & 2;
    const int lane = threadIdx.x & 31;
    const int k = blockIdx.x * LRF_WARPS + (threadIdx.x >> 5);
    if (k >= K) return;
    if (d_K && (r_group > 0 ? k % r_group >= d_K[k / r_group] : k >= *d_K)) return;     // beyond the group's device count
    const float des_r = d_des_r ? d_des_r[r_group > 0 ? k / r_group : 0] : des_r_v;     // batched call: one radius per r_group patches
    const float *pt = patches + (size_t)k * P * 3;
    float *dl = delta + (size_t)k * P * 3;
    const float cx = pt[3 * (P - 1)], cy = pt[3 * (P - 1) + 1], cz = pt[3 * (P - 1) + 2];
    float R[3][3] = {{1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, 0.f, 1.f}};
    float ra0 = 1.0f, ra1 = 0.0f, ra2 = 0.0f;
    if (!aligned) {
        float c00 = 0.f, c01 = 0.f, c02 = 0.f, c11 = 0.f, c12 = 0.f, c22 = 0.f;
        for (int s = lane; s < P; s += 32) {
            const float x = pt[3 * s] - cx, y = pt[3 * s + 1] - cy, z = pt[3 * s + 2] - cz;
            c00 = c00 + (x * x);
            c01 = c01 + (x * y);
            c02 = c02 + (x * z);
            c11 = c11 + (y * y);
            c12 = c12 + (y * z);
            c22 = c22 + (z * z);
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
            c00 = c00 + __shfl_xor_sync(BX_FULL, c00, off);
            c01 = c01 + __shfl_xor_sync(BX_FULL, c01, off);
            c02 = c02 + __shfl_xor_sync(BX_FULL, c02, off);
            c11 = c11 + __shfl_xor_sync(BX_FULL, c11, off);
            c12 = c12 + __shfl_xor_sync(BX_FULL, c12, off);
            c22 = c22 + __shfl_xor_sync(BX_FULL, c22, off);
        }
        double A[3][3], V[3][3];
        A[0][0] = c00; A[0][1] = c01; A[0][2] = c02;
        A[1][0] = c01; A[1][1] = c11; A[1][2] = c12;
        A[2][0] = c02; A[2][1] = c12; A[2][2] = c22;
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
        for (int sweep = 0; sweep < 8; ++sweep) {
            jacobi_rot3(A, V, 0, 1);
            jacobi_rot3(A, V, 0, 2);
            jacobi_rot3(A, V, 1, 2);
        }
        // smallest eigenvalue, first minimum wins (fully unrolled selects: no dynamic register indexing)
        double em = A[0][0];
        double v0 = V[0][0], v1 = V[1][0], v2 = V[2][0];
        if (A[1][1] < em) { em = A[1][1]; v0 = V[0][1]; v1 = V[1][1]; v2 = V[2][1]; }
        if (A[2][2] < em) { em = A[2][2]; v0 = V[0][2]; v1 = V[1][2]; v2 = V[2][2]; }
        float z0 = (float)v0, z1 = (float)v1, z2 = (float)v2;
        const float sgn = (((-z0) * cx) + ((-z1) * cy)) + ((-z2) * cz);
        if (sgn < 0.0f) { z0 = -z0; z1 = -z1; z2 = -z2; }
        const float nz = sqrtf(((z0 * z0) + (z1 * z1)) + (z2 * z2));
        z0 = z0 / nz; z1 = z1 / nz; z2 = z2 / nz;
        const float n = sqrtf(((z0 * z0) + (z1 * z1)) + (z2 * z2));
        const float sn = sqrtf((z0 * z0) + (z1 * z1));
        float ct = z2 / n, st = sn / n;
        if (!stable) {
            // RodsRotatFormula literally (utils/common.py:506, 522): theta = acos(cosine_similarity(z, e_z)), then
            // sin(theta) / cos(theta).  fp32 results are the correctly rounded ones (evaluated in fp64, rounded once),
            // which the CPU oracle reproduces bit for bit; CUDA's acosf/sinf/cosf are 1-2 ulp routines of their own.
            const float theta = (float)acos((double)ct);
            st = (float)sin((double)theta);
            ct = (float)cos((double)theta);
        }
        const float den = sn > 1e-12f ? sn : 1e-12f;
        const float a0 = z1 / den, a1 = (-z0) / den;
        const float kk = 1.0f - ct;
        R[0][0] = 1.0f - (kk * (a1 * a1)); R[0][1] = kk * (a0 * a1);          R[0][2] = st * a1;
        R[1][0] = kk * (a0 * a1);          R[1][1] = 1.0f - (kk * (a0 * a0)); R[1][2] = -(st * a0);
        R[2][0] = -(st * a1);              R[2][1] = st * a0;                 R[2][2] = 1.0f - (kk * ((a0 * a0) + (a1 * a1)));
        ra0 = a0; ra1 = a1; ra2 = 0.0f;
    }
    for (int s = lane; s < P; s += 32) {
        const float x = pt[3 * s] - cx, y = pt[3 * s + 1] - cy, z = pt[3 * s + 2] - cz;
        float ox = x, oy = y, oz = z;
        if (!aligned) {
            ox = ((R[0][0] * x) + (R[0][1] * y)) + (R[0][2] * z);
            oy = ((R[1][0] * x) + (R[1][1] * y)) + (R[1][2] * z);
            oz = ((R[2][0] * x) + (R[2][1] * y)) + (R[2][2] * z);
        }
        dl[3 * s] = ox / des_r;
        dl[3 * s + 1] = oy / des_r;
        dl[3 * s + 2] = oz / des_r;
    }
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) Rt[(size_t)k * 9 + 3 * i + j] = R[j][i];
        rand_axis[3 * (size_t)k] = ra0;
        rand_axis[3 * (size_t)k + 1] = ra1;
        rand_axis[3 * (size_t)k + 2] = ra2;
    }
}

}  // namespace

BX_API int bx_permute_cloud(const float *pts, const int32_t *perm, int N, float *out4, void *stream) {
    return bx_permute_cloud_n(pts, perm, N, nullptr, out4, stream);
}

BX_API int bx_permute_cloud_n(const float *pts, const int32_t *perm, int N, const int32_t *d_N, float *out4, void *stream) {
    BX_REQUIRE(pts && out4 && N >= 1, "bx_permute_cloud: bad arguments");
    BX_REQUIRE((reinterpret_cast<uintptr_t>(out4) & 15) == 0, "bx_permute_cloud: out4 must be 16-byte aligned");
    permute_cloud_kernel<<<(N + 255) / 256, 256, 0, bx_stream(stream)>>>(pts, perm, N, reinterpret_cast<float4 *>(out4), d_N);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_select_patches(const float *pts4, int N, const float *kpts, int K, float radius, const float *d_radius,
                             int P, int32_t *idx, float *patches, void *stream) {
    BX_REQUIRE(pts4 && kpts && patches, "bx_select_patches: null pointer");
    BX_REQUIRE(N >= 1 && K >= 0 && P >= 1, "bx_select_patches: bad sizes N=%d K=%d P=%d", N, K, P);
    BX_REQUIRE((reinterpret_cast<uintptr_t>(pts4) & 15) == 0, "bx_select_patches: pts4 must be 16-byte aligned");
    if (K == 0) return BX_OK;
    select_patches_kernel<<<(K + SP_KP - 1) / SP_KP, SP_WARPS * 32, 0, bx_stream(stream)>>>(
        reinterpret_cast<const float4 *>(pts4), N, kpts, K, radius, d_radius, P, idx, patches);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_select_patches_batched(int njobs, const void *const *pts4, const int32_t *N, const void *const *kpts, const int32_t *K,
                                     const void *const *d_radius, int P, float *patches, void *stream) {
    return bx_select_patches_batched_n(njobs, pts4, N, kpts, K, d_radius, nullptr, P, patches, stream);
}

BX_API int bx_select_patches_batched_n(int njobs, const void *const *pts4, const int32_t *N, const void *const *kpts, const int32_t *K,
                                       const void *const *d_radius, const void *const *d_K, int P, float *patches, void *stream) {
    return bx_select_patches_batched_counts(njobs, pts4, N, nullptr, kpts, K, d_radius, d_K, P, patches, stream);
}

BX_API int bx_select_patches_batched_counts(int njobs, const void *const *pts4, const int32_t *N, const void *const *d_N, const void *const *kpts,
                                            const int32_t *K, const void *const *d_radius, const void *const *d_K, int P, float *patches,
                                            void *stream) {
    BX_REQUIRE(pts4 && N && kpts && K && d_radius && patches, "bx_select_patches_batched: null pointer");
    BX_REQUIRE(njobs >= 1 && njobs <= SP_MAXJOBS && P >= 1, "bx_select_patches_batched: njobs=%d out of range [1,%d]", njobs, SP_MAXJOBS);
    SpJobs jobs = {};
    jobs.njobs = njobs;
    int blocks = 0, koff = 0;
    for (int j = 0; j < njobs; ++j) {
        BX_REQUIRE(pts4[j] && kpts[j] && d_radius[j] && N[j] >= 1 && K[j] >= 0, "bx_select_patches_batched: bad job %d", j);
        BX_REQUIRE((reinterpret_cast<uintptr_t>(pts4[j]) & 15) == 0, "bx_select_patches_batched: pts4 must be 16-byte aligned");
        jobs.pts4[j] = reinterpret_cast<const float4 *>(pts4[j]);
        jobs.kpts[j] = reinterpret_cast<const float *>(kpts[j]);
        jobs.d_radius[j] = reinterpret_cast<const float *>(d_radius[j]);
        jobs.d_K[j] = d_K ? reinterpret_cast<const int *>(d_K[j]) : nullptr;
        jobs.d_N[j] = d_N ? reinterpret_cast<const int *>(d_N[j]) : nullptr;
        jobs.N[j] = N[j]; jobs.K[j] = K[j];
        jobs.boff[j] = blocks; jobs.koff[j] = koff;
        blocks += (K[j] + SP_KP - 1) / SP_KP;
        koff += K[j];
    }
    jobs.boff[njobs] = blocks;
    if (blocks == 0) return BX_OK;
    select_patches_batched_kernel<<<blocks, SP_WARPS * 32, 0, bx_stream(stream)>>>(jobs, P, patches);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API long long bx_select_patches_grid_workspace_bytes(int N) {
    return (long long)(3 * HG_CELLS + 8 + 32) * 4 + (long long)N * 16;      // sorted points, counts, starts, cursors, chunk totals; a multiple of 16
}

// Hash-grid form (see above): same contract as bx_select_patches with a device-side radius.  workspace:
// bx_select_patches_grid_workspace_bytes(N) bytes, 16-byte aligned, contents undefined on entry.
BX_API int bx_select_patches_grid(const float *pts4, int N, const float *kpts, int K, const float *d_radius, int P, int32_t *idx,
                                  float *patches, void *workspace, void *stream) {
    BX_REQUIRE(pts4 && kpts && patches && workspace && d_radius, "bx_select_patches_grid: null pointer");
    BX_REQUIRE(N >= 1 && K >= 0 && P >= 1, "bx_select_patches_grid: bad sizes N=%d K=%d P=%d", N, K, P);
    BX_REQUIRE(((reinterpret_cast<uintptr_t>(pts4) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0, "bx_select_patches_grid: pts4 / workspace must be 16-byte aligned");
    const size_t bitmap = (size_t)((N + 31) / 32) * 4;
    BX_REQUIRE(bitmap <= 200 * 1024, "bx_select_patches_grid: N=%d exceeds the shared-memory bitmap (1.6 M points)", N);
    if (K == 0) return BX_OK;
    cudaStream_t st = bx_stream(stream);
    float4 *sorted = reinterpret_cast<float4 *>(workspace);
    int *cnt = reinterpret_cast<int *>(sorted + N);
    int *start = cnt + HG_CELLS, *cursor = start + HG_CELLS + 4;      // 16-byte aligned arrays (int4 accesses in the scan)
    BX_CUDA(cudaMemsetAsync(cnt, 0, (size_t)HG_CELLS * 4, st));
    const float4 *p4 = reinterpret_cast<const float4 *>(pts4);
    hg_count_kernel<<<(N + 255) / 256, 256, 0, st>>>(p4, N, d_radius, cnt);
    BX_LAUNCH_CHECK();
    hg_scan_kernel<<<1, 1024, 0, st>>>(cnt, start, cursor);
    BX_LAUNCH_CHECK();
    hg_scatter_kernel<<<(N + 255) / 256, 256, 0, st>>>(p4, N, d_radius, cursor, sorted);
    BX_LAUNCH_CHECK();
    static BxPerDevice attr = {};
    if (bx_needs_attr(attr, bitmap))
        BX_CUDA(cudaFuncSetAttribute(hg_query_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)));
    hg_query_kernel<<<K, HG_THREADS, bitmap, st>>>(p4, N, kpts, K, d_radius, P, start, sorted, idx, patches);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

// All (cloud, scale) jobs of a pair through the hash grid: one launch per phase.  workspace: the sum over the jobs of
// bx_select_patches_grid_workspace_bytes(N[j]) bytes (16-byte aligned); patches: job after job like bx_select_patches_batched.
BX_API int bx_select_patches_grid_batched(int njobs, const void *const *pts4, const int32_t *N, const void *const *kpts, const int32_t *K,
                                          const void *const *d_radius, int P, float *patches, void *workspace, void *stream) {
    return bx_select_patches_grid_batched_n(njobs, pts4, N, kpts, K, d_radius, nullptr, P, patches, workspace, stream);
}

BX_API int bx_select_patches_grid_batched_n(int njobs, const void *const *pts4, const int32_t *N, const void *const *kpts, const int32_t *K,
                                            const void *const *d_radius, const void *const *d_K, int P, float *patches, void *workspace,
                                            void *stream) {
    return bx_select_patches_grid_batched_counts(njobs, pts4, N, nullptr, kpts, K, d_radius, d_K, P, patches, workspace, stream);
}

// d_N: the device point counts of the jobs (see bx_select_patches_batched_counts).  The workspace, the bitmap and the grids of the
// point-parallel phases are sized by the capacities N[j]; every phase stops at the count.
BX_API int bx_select_patches_grid_batched_counts(int njobs, const void *const *pts4, const int32_t *N, const void *const *d_N,
                                                 const void *const *kpts, const int32_t *K, const void *const *d_radius,
                                                 const void *const *d_K, int P, float *patches, void *workspace, void *stream) {
    BX_REQUIRE(pts4 && N && kpts && K && d_radius && patches && workspace, "bx_select_patches_grid_batched: null pointer");
    BX_REQUIRE(njobs >= 1 && njobs <= SP_MAXJOBS && P >= 1, "bx_select_patches_grid_batched: njobs=%d out of range [1,%d]", njobs, SP_MAXJOBS);
    BX_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "bx_select_patches_grid_batched: workspace must be 16-byte aligned");
    HgJobs J = {};
    J.njobs = njobs;
    unsigned char *ws = reinterpret_cast<unsigned char *>(workspace);
    int koff = 0, maxN = 0;
    for (int j = 0; j < njobs; ++j) {
        BX_REQUIRE(pts4[j] && kpts[j] && d_radius[j] && N[j] >= 1 && K[j] >= 0, "bx_select_patches_grid_batched: bad job %d", j);
        BX_REQUIRE((reinterpret_cast<uintptr_t>(pts4[j]) & 15) == 0, "bx_select_patches_grid_batched: pts4 must be 16-byte aligned");
        J.pts4[j] = reinterpret_cast<const float4 *>(pts4[j]);
        J.kpts[j] = reinterpret_cast<const float *>(kpts[j]);
        J.d_radius[j] = reinterpret_cast<const float *>(d_radius[j]);
        J.d_K[j] = d_K ? reinterpret_cast<const int *>(d_K[j]) : nullptr;
        J.d_N[j] = d_N ? reinterpret_cast<const int *>(d_N[j]) : nullptr;
        J.N[j] = N[j];
        J.sorted[j] = reinterpret_cast<float4 *>(ws);
        J.cnt[j] = reinterpret_cast<int *>(J.sorted[j] + N[j]);
        ws += bx_select_patches_grid_workspace_bytes(N[j]);
        J.koff[j] = koff;
        koff += K[j];
        if (N[j] > maxN) maxN = N[j];
    }
    J.koff[njobs] = koff;
    const size_t bitmap = (size_t)((maxN + 31) / 32) * 4;
    BX_REQUIRE(bitmap <= 200 * 1024, "bx_select_patches_grid_batched: N=%d exceeds the shared-memory bitmap (1.6 M points)", maxN);
    if (koff == 0) return BX_OK;
    cudaStream_t st = bx_stream(stream);
    for (int j = 0; j < njobs; ++j) BX_CUDA(cudaMemsetAsync(J.cnt[j], 0, (size_t)HG_CELLS * 4, st));
    const dim3 pg((unsigned)((maxN + 255) / 256), (unsigned)njobs);
    hg_count_batched_kernel<<<pg, 256, 0, st>>>(J);
    BX_LAUNCH_CHECK();
    static_assert(HG_CHUNKS == 32, "the chunk scan sums the earlier chunk totals with one warp");
    hg_chunksum_batched_kernel<<<dim3(HG_CHUNKS, (unsigned)njobs), HG_SCAN_THREADS, 0, st>>>(J);
    BX_LAUNCH_CHECK();
    hg_chunkscan_batched_kernel<<<dim3(HG_CHUNKS, (unsigned)njobs), HG_SCAN_THREADS, 0, st>>>(J);
    BX_LAUNCH_CHECK();
    hg_scatter_batched_kernel<<<pg, 256, 0, st>>>(J);
    BX_LAUNCH_CHECK();
    static BxPerDevice attr = {};
    if (bx_needs_attr(attr, bitmap))
        BX_CUDA(cudaFuncSetAttribute(hg_query_batched_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)));
    hg_query_batched_kernel<<<koff, HG_THREADS, bitmap, st>>>(J, P, patches);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_ball_query(const float *xyz, int n, const float *qry, int m, float radius, int nsample, int32_t *idx,
                         void *stream) {
    BX_REQUIRE(xyz && qry && idx && n >= 1 && m >= 0 && nsample >= 1, "bx_ball_query: bad arguments");
    if (m == 0) return BX_OK;
    ball_query_kernel<<<(m + BQ_WARPS - 1) / BQ_WARPS, BQ_WARPS * 32, 0, bx_stream(stream)>>>(xyz, n, qry, m, radius,
                                                                                                nsample, idx);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_lrf(const float *patches, int K, int P, float des_r, const float *d_des_r, int flags, float *delta,
                  float *Rt, float *rand_axis, void *stream) {
    return bx_lrf_batched(patches, K, P, des_r, d_des_r, 0, flags, delta, Rt, rand_axis, stream);
}

BX_API int bx_lrf_batched(const float *patches, int K, int P, float des_r, const float *d_des_r, int r_group, int flags, float *delta,
                          float *Rt, float *rand_axis, void *stream) {
    return bx_lrf_batched_n(patches, K, P, des_r, d_des_r, r_group, nullptr, flags, delta, Rt, rand_axis, stream);
}

BX_API int bx_lrf_batched_n(const float *patches, int K, int P, float des_r, const float *d_des_r, int r_group, const int32_t *d_K, int flags,
                            float *delta, float *Rt, float *rand_axis, void *stream) {
    BX_REQUIRE(K >= 0 && P >= 1 && r_group >= 0, "bx_lrf: bad sizes");
    if (K == 0) return BX_OK;                 // an empty batch: torch hands empty tensors over as null pointers
    BX_REQUIRE(patches && delta && Rt && rand_axis, "bx_lrf: null pointer");
    lrf_kernel<<<(K + LRF_WARPS - 1) / LRF_WARPS, LRF_WARPS * 32, 0, bx_stream(stream)>>>(patches, K, P, des_r, d_des_r,
                                                                                           flags, delta, Rt, rand_axis, r_group, d_K);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
