// bx_hashgrid.cuh -- counting-sort phases of the spatial hash grid, shared by the patch gatherer (bx_patches.cu) and the
// ICP neighbour search (bx_icp.cu).
//
// A cloud of float4 points (x, y, z, -) is binned into HG_CELLS buckets of cubic cells of edge hg_inv_cell(r)^-1 >= r (classic
// three-prime hash of the integer cell coordinates: no bounding box needed, aliases only add candidates) by three phases:
// count (integer atomics), one exclusive scan, scatter into `sorted` (the point's index in .w).  How a query picks its cells
// and why the window encloses every hit is the caller's own argument (hg_window in bx_patches.cu, icp_window in bx_icp.cu).
#pragma once
#include "bx_common.cuh"

namespace {

constexpr int HG_BITS = 17, HG_CELLS = 1 << HG_BITS;

__device__ __forceinline__ int hg_coord(float v, float inv_cell) { return (int)floorf(v * inv_cell); }
__device__ __forceinline__ unsigned hg_hash(int ix, int iy, int iz) {
    return ((unsigned)ix * 73856093u ^ (unsigned)iy * 19349663u ^ (unsigned)iz * 83492791u) & (unsigned)(HG_CELLS - 1);
}
// cell edge = radius * (1 + 1e-3)
__device__ __forceinline__ float hg_inv_cell(float r) { return 1.0f / (r * 1.001f); }

__device__ __forceinline__ void hg_count_body(const float4 *__restrict__ pts4, int N, const float *__restrict__ d_radius, int *__restrict__ cnt, int i) {
    if (i >= N) return;
    const float ic = hg_inv_cell(*d_radius);
    const float4 p = pts4[i];
    atomicAdd(cnt + hg_hash(hg_coord(p.x, ic), hg_coord(p.y, ic), hg_coord(p.z, ic)), 1);
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

__device__ __forceinline__ void hg_scatter_body(const float4 *__restrict__ pts4, int N, const float *__restrict__ d_radius, int *__restrict__ cursor,
                                                float4 *__restrict__ sorted, int i) {
    if (i >= N) return;
    const float ic = hg_inv_cell(*d_radius);
    const float4 p = pts4[i];
    const int pos = atomicAdd(cursor + hg_hash(hg_coord(p.x, ic), hg_coord(p.y, ic), hg_coord(p.z, ic)), 1);
    sorted[pos] = make_float4(p.x, p.y, p.z, __int_as_float(i));        // the order inside a bucket is not deterministic
}

}  // namespace
