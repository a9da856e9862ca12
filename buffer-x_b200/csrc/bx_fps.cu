// bx_fps.cu -- a1: farthest point sampling, one thread-block cluster per cloud.
//
// Replaces pointnet2_ops.furthest_point_sample (+gather_operation) as called at
// /root/reference/models/BUFFERX.py:286-290 and :338-346.  The upstream kernel runs ONE CTA per
// cloud and re-reads the cloud and a global `temp` array every iteration with ~10 barriers per
// step.  Here the cloud (x,y,z and the running min-distance) lives in REGISTERS spread over a
// cluster of up to 16 CTAs; an iteration is: register scan -> warp redux -> one __syncthreads ->
// warp redux -> DSMEM all-to-all of one 20-byte candidate per CTA -> one cluster barrier.
// The candidate carries the winner's coordinates, so no thread touches global memory in the loop.
//
// Result contract (bit-exact with oracle/c/bx_oracle.c::bxo_fps): idx[0] = 0; candidates with
// |p|^2 <= 1e-3 (double compare) never win; ties are broken like the upstream 512-thread block
// reduction (each tree step keeps the lower position, so the smallest BIT-REVERSED slot wins):
// maximise (value, -bitrev(k mod bs), -k) with bs = min(512, 2^floor(log2 N)).
// Compiled with -fmad=false: d = ((dx*dx)+(dy*dy))+(dz*dz) exactly.
#include <cooperative_groups.h>

#include "bx_common.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kMaxClouds = 16;
struct FpsOffsets {
    int v[kMaxClouds + 1];  // passed by value as a kernel argument: no device copy, no sync
};

struct Cand {
    uint32_t hi, lo;  // hi = fp32 bits of the (non-negative) distance, lo = ~rank  (0,0) = "none" -> index 0
    float x, y, z;    // coordinates of the candidate
};

__device__ __forceinline__ Cand warp_best(const Cand c) {
    const uint32_t mh = __reduce_max_sync(BX_FULL, c.hi);
    const bool in = (c.hi == mh);
    const uint32_t ml = __reduce_max_sync(BX_FULL, in ? c.lo : 0u);
    const unsigned b = __ballot_sync(BX_FULL, in && c.lo == ml);
    const int src = __ffs(b) - 1;
    Cand r;
    r.hi = mh;
    r.lo = ml;
    r.x = __shfl_sync(BX_FULL, c.x, src);
    r.y = __shfl_sync(BX_FULL, c.y, src);
    r.z = __shfl_sync(BX_FULL, c.z, src);
    return r;
}

// ---- cluster exchange without cluster.sync: remote stores + remote mbarrier arrive (release.cluster), local wait
//      (acquire.cluster).  A cluster.sync per FPS iteration is a full cluster barrier and flushes L1; this costs one
//      DSMEM round.
__device__ __forceinline__ uint32_t fps_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t fps_mapa(uint32_t saddr, uint32_t cta) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(cta));
    return r;
}
__device__ __forceinline__ void fps_st_cluster_v4(uint32_t a, uint4 v) {
    asm volatile("st.shared::cluster.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void fps_st_cluster_f32(uint32_t a, float v) {
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory");
}
__device__ __forceinline__ void fps_arrive_cluster(uint32_t rbar) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(rbar) : "memory");
}
// One-way exchange: st.async writes 16 bytes into the peer's shared memory AND completes that many transaction bytes on the
// peer's mbarrier when they have landed -- no separate release-arrive that has to wait for the stores (one DSMEM trip
// instead of two per iteration).
__device__ __forceinline__ void fps_st_async_v4(uint32_t raddr, uint4 v, uint32_t rbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(raddr), "r"(v.x),
                 "r"(v.y), "r"(v.z), "r"(v.w), "r"(rbar)
                 : "memory");
}
__device__ __forceinline__ void fps_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fps_wait_cluster(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "FPS_WAIT:\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra FPS_DONE;\n\t"
        "bra FPS_WAIT;\n\t"
        "FPS_DONE:\n\t"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}

template <int THREADS, int PPT>
__global__ void __launch_bounds__(THREADS, 1)
fps_cluster_kernel(const float *__restrict__ xyz_all, const FpsOffsets offsets, int npoint,
                   int *__restrict__ idx_out, float *__restrict__ kpts_out, int sync_mode, const int *__restrict__ d_counts) {
    constexpr int NW = THREADS / 32;
    cg::cluster_group cluster = cg::this_cluster();
    const int CL = (int)cluster.num_blocks();
    const int rank = (int)cluster.block_rank();
    const int cloud = blockIdx.x / CL;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    const int start = offsets.v[cloud];
    const int cap = offsets.v[cloud + 1] - start;
    // device count (size-class slots): the points of the cloud present this launch, clamped to [1, capacity]
    const int N = d_counts ? min(max(d_counts[cloud], 1), cap) : cap;
    const float *xyz = xyz_all + 3 * (size_t)start;
    int *idx = idx_out + (size_t)cloud * npoint;
    float *kp = kpts_out ? kpts_out + 3 * (size_t)cloud * npoint : nullptr;

    // upstream block size and the per-slot stride used for the tie rank
    int log2bs = 0;
    while ((2 << log2bs) <= N && log2bs < 9) ++log2bs;  // bs = min(512, 2^floor(log2 N))
    const int bs = 1 << log2bs;
    const int cpb = (N + bs - 1) >> log2bs;

    __shared__ uint4 w_a[2][32];
    __shared__ float w_z[2][32];
    __shared__ uint4 c_a[2][16];
    __shared__ float c_z[2][16];
    __shared__ uint4 x_a[2][16][2];                      // st.async exchange: two 16-byte halves per (parity, sender)
    __shared__ __align__(8) unsigned long long cbar[2];   // one exchange barrier per parity, CL arrivals each
    __shared__ __align__(8) unsigned long long xbar[2];   // st.async exchange: 1 arrival (own expect_tx) + 32 * CL bytes per phase

    float px[PPT], py[PPT], pz[PPT], tmp[PPT];
    const int stride = CL * THREADS;
    const int base = rank * THREADS + tid;
#pragma unroll
    for (int s = 0; s < PPT; ++s) {
        const int k = s * stride + base;
        if (k < N) {
            px[s] = xyz[3 * (size_t)k];
            py[s] = xyz[3 * (size_t)k + 1];
            pz[s] = xyz[3 * (size_t)k + 2];
            const float mag = ((px[s] * px[s]) + (py[s] * py[s])) + (pz[s] * pz[s]);
            tmp[s] = ((double)mag <= 1e-3) ? -1.0f : 1e10f;
        } else {
            px[s] = py[s] = pz[s] = 0.0f;
            tmp[s] = -1.0f;
        }
    }
    const float p0x = xyz[0], p0y = xyz[1], p0z = xyz[2];
    float ox = p0x, oy = p0y, oz = p0z;
    if (rank == 0 && tid == 0 && npoint > 0) {
        idx[0] = 0;
        if (kp) { kp[0] = p0x; kp[1] = p0y; kp[2] = p0z; }
    }
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(fps_smem_u32(&cbar[0])), "r"(CL) : "memory");
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(fps_smem_u32(&cbar[1])), "r"(CL) : "memory");
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(fps_smem_u32(&xbar[0])), "r"(1) : "memory");
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(fps_smem_u32(&xbar[1])), "r"(1) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    cluster.sync();  // every CTA of the cluster is resident (and its barriers initialised) before any DSMEM access

    for (int j = 1; j < npoint; ++j) {
        const int par = j & 1;
        Cand best;
        best.hi = 0u; best.lo = 0u; best.x = p0x; best.y = p0y; best.z = p0z;
#pragma unroll
        for (int s = 0; s < PPT; ++s) {
            if (tmp[s] >= 0.0f) {
                const float d = bx_d2(px[s] - ox, py[s] - oy, pz[s] - oz);
                const float d2 = fminf(d, tmp[s]);
                tmp[s] = d2;
                const int k = s * stride + base;
                const uint32_t tr = log2bs ? (__brev((uint32_t)(k & (bs - 1))) >> (32 - log2bs)) : 0u;
                const uint32_t rk = tr * (uint32_t)cpb + (uint32_t)(k >> log2bs);
                const uint32_t hi = __float_as_uint(d2), lo = ~rk;
                if (hi > best.hi || (hi == best.hi && lo > best.lo)) {
                    best.hi = hi; best.lo = lo; best.x = px[s]; best.y = py[s]; best.z = pz[s];
                }
            }
        }
        const Cand wb = warp_best(best);
        if (lane == 0) {
            w_a[par][warp] = make_uint4(wb.hi, wb.lo, __float_as_uint(wb.x), __float_as_uint(wb.y));
            w_z[par][warp] = wb.z;
        }
        __syncthreads();
        Cand c;
        c.hi = 0u; c.lo = 0u; c.x = p0x; c.y = p0y; c.z = p0z;
        if (lane < NW) {
            const uint4 a = w_a[par][lane];
            c.hi = a.x; c.lo = a.y; c.x = __uint_as_float(a.z); c.y = __uint_as_float(a.w); c.z = w_z[par][lane];
        }
        Cand cb = warp_best(c);
        if (CL > 1 && sync_mode == 0) {
            // production: every CTA posts its candidate into every peer's slot with st.async (data + transaction bytes in one
            // DSMEM trip); a CTA's barrier phase completes when its own expect_tx arrival and all 32 * CL bytes are in.
            if (warp == 0) {
                if (lane == 0) fps_expect_tx(fps_smem_u32(&xbar[par]), 32u * (uint32_t)CL);
                if (lane < CL) {
                    const uint32_t dst = fps_mapa(fps_smem_u32(&x_a[par][rank][0]), (uint32_t)lane);
                    const uint32_t rb = fps_mapa(fps_smem_u32(&xbar[par]), (uint32_t)lane);
                    fps_st_async_v4(dst, make_uint4(cb.hi, cb.lo, __float_as_uint(cb.x), __float_as_uint(cb.y)), rb);
                    fps_st_async_v4(dst + 16u, make_uint4(__float_as_uint(cb.z), 0u, 0u, 0u), rb);
                }
            }
            fps_wait_cluster(fps_smem_u32(&xbar[par]), (uint32_t)(((j >> 1) - (par ? 0 : 1)) & 1));
            Cand g;
            g.hi = 0u; g.lo = 0u; g.x = p0x; g.y = p0y; g.z = p0z;
            if (lane < CL) {
                const uint4 a = x_a[par][lane][0];
                g.hi = a.x; g.lo = a.y; g.x = __uint_as_float(a.z); g.y = __uint_as_float(a.w);
                g.z = __uint_as_float(x_a[par][lane][1].x);
            }
            cb = warp_best(g);
        } else if (CL > 1) {
            if (warp == 0 && lane < CL) {   // lane = destination CTA: candidate into its slot [rank], then arrive on its barrier
                fps_st_cluster_v4(fps_mapa(fps_smem_u32(&c_a[par][rank]), (uint32_t)lane),
                                  make_uint4(cb.hi, cb.lo, __float_as_uint(cb.x), __float_as_uint(cb.y)));
                fps_st_cluster_f32(fps_mapa(fps_smem_u32(&c_z[par][rank]), (uint32_t)lane), cb.z);
                if (sync_mode != 1) fps_arrive_cluster(fps_mapa(fps_smem_u32(&cbar[par]), (uint32_t)lane));
            }
            // Buffers and barriers are double-buffered by parity: a peer can only be one iteration ahead (its next
            // wait needs our next arrive), so slot [par] is not rewritten before everybody has read it.
            // sync_mode (BX_FPS_SYNC=1, verification only): the same exchange ordered by a plain cluster.sync() -- the form
            // compute-sanitizer's racecheck models; results are bit-identical (tests/test_gpu_parity.py).
            if (sync_mode == 1) cluster.sync();
            else fps_wait_cluster(fps_smem_u32(&cbar[par]), (uint32_t)(((j >> 1) - (par ? 0 : 1)) & 1));
            Cand g;
            g.hi = 0u; g.lo = 0u; g.x = p0x; g.y = p0y; g.z = p0z;
            if (lane < CL) {
                const uint4 a = c_a[par][lane];
                g.hi = a.x; g.lo = a.y; g.x = __uint_as_float(a.z); g.y = __uint_as_float(a.w); g.z = c_z[par][lane];
            }
            cb = warp_best(g);
        }
        ox = cb.x; oy = cb.y; oz = cb.z;
        if (rank == 0 && tid == 0) {
            int k = 0;
            if (cb.hi != 0u || cb.lo != 0u) {
                const uint32_t rk = ~cb.lo;
                const uint32_t tr = rk / (uint32_t)cpb;
                const uint32_t t = log2bs ? (__brev(tr) >> (32 - log2bs)) : 0u;
                k = (int)((rk % (uint32_t)cpb) << log2bs) + (int)t;
            }
            idx[j] = k;
            if (kp) { kp[3 * j] = ox; kp[3 * j + 1] = oy; kp[3 * j + 2] = oz; }
        }
    }
    cluster.sync();  // nobody exits while a peer may still write into its shared memory
}

int g_fps_sync_override = -1;

template <int THREADS, int PPT>
int launch_fps(const float *xyz, const FpsOffsets off, int B, int CL, int npoint, int *idx, float *kpts, const int *d_counts,
               cudaStream_t st) {
    auto kern = fps_cluster_kernel<THREADS, PPT>;
    if (CL > 8) BX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(B * CL));
    cfg.blockDim = dim3(THREADS);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)CL;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    static int sync_mode = -1;     // BX_FPS_SYNC: 0 = st.async exchange (production), 1 = cluster.sync() (racecheck-clean reference form),
    if (sync_mode < 0) { const char *e = getenv("BX_FPS_SYNC"); sync_mode = e ? atoi(e) : 0; }   // 2 = remote stores + mbarrier arrive / acquire wait (round 1)
    if (g_fps_sync_override >= 0) sync_mode = g_fps_sync_override;
    BX_CUDA(cudaLaunchKernelEx(&cfg, kern, xyz, off, npoint, idx, kpts, sync_mode, d_counts));
    ++g_bx_launches;
    return BX_OK;
}


// Launch configuration of a cloud of n points (the largest cloud of the call): register tier = (threads, points per thread,
// CTAs per cloud).  Also returns, in *hi, the largest n that gets the same configuration -- the cloud's size class.
enum FpsTier { T256x2, T256x4, T1024x4c, T1024x6c, T1024x10c, T1024x12c, T1024x1c16, T1024x2c16, T1024x2, T1024x3, T1024x4,
               T1024x8, T1024x8c16, T512x32, T512x64 };

FpsTier fps_tier(int n, int max_cluster, int *hi) {
    if (n <= 4096) { *hi = 4096; return T256x2; }
    if (n <= 8192) { *hi = 8192; return T256x4; }
    // larger clouds: 1024 threads per CTA and few points per thread -- the per-iteration register scan is a dependent
    // chain per thread, so its latency scales with the points per thread, while the reductions / cluster exchange
    // do not depend on the thread count
    if (max_cluster > 0 && n <= 49152) {
        const int cl = max_cluster >= 4 ? 4 : 2;
        const int per_cta = (n + cl - 1) / cl;          // points per CTA of 1024 threads
        if (per_cta <= 4096) { *hi = min(4096 * cl, 49152); return T1024x4c; }
        if (per_cta <= 6144) { *hi = min(6144 * cl, 49152); return T1024x6c; }
        if (per_cta <= 10240) { *hi = min(10240 * cl, 49152); return T1024x10c; }
        if (per_cta <= 12288) { *hi = min(12288 * cl, 49152); return T1024x12c; }
    }
    { static int cl16 = -1; if (cl16 < 0) { const char *e = getenv("BX_FPS_CL16"); cl16 = e ? atoi(e) : 0; }     // experiment: 16-CTA clusters, fewer points per thread
      if (cl16 && n <= 16384) { *hi = 16384; return T1024x1c16; }
      if (cl16 && n <= 32768) { *hi = 32768; return T1024x2c16; } }
    if (n <= 16384) { *hi = 16384; return T1024x2; }
    if (n <= 24576) { *hi = 24576; return T1024x3; }
    if (n <= 32768) { *hi = 32768; return T1024x4; }
    if (n <= 65536) { *hi = 65536; return T1024x8; }
    if (n <= 131072) { *hi = 131072; return T1024x8c16; }
    // beyond 128 K points per cloud (raw LiDAR sweeps before voxel down-sampling): 512-thread CTAs leave 128 registers per
    // thread, enough for 32 / 64 points each -- slower per iteration, same result contract
    if (n <= 262144) { *hi = 262144; return T512x32; }
    *hi = 524288;
    return T512x64;
}

}  // namespace

// Exchange switch: 0 = st.async + transaction-count mbarrier (production), 1 = plain stores ordered by cluster.sync() (the form
// compute-sanitizer racecheck models), 2 = remote stores + remote mbarrier arrive / acquire wait (round 1's production);
// same results in all three.  -1 = follow the BX_FPS_SYNC environment variable.  Returns the previous value.
BX_API int bx_fps_set_sync_mode(int mode) {
    const int old = g_fps_sync_override;
    g_fps_sync_override = mode;
    return old;
}

BX_API int bx_fps(const float *xyz, const int32_t *h_offsets, int B, int npoint, int32_t *idx, float *kpts,
                  void *stream) {
    return bx_fps_n(xyz, h_offsets, B, npoint, idx, kpts, 0, nullptr, stream);
}

// max_cluster > 0: THROUGHPUT form -- at most that many CTAs per cloud (2 or 4), more points per thread.  An iteration is a
// latency chain (reductions + cluster exchange) whatever the cluster size, so the default form spreads a cloud over 8 SMs
// only to shorten the register scan; when several pairs are in flight the 16 SMs of a pair's two clouds are taken from the
// other pairs' convolutions for the whole sampling.  Two CTAs per cloud hold 10 points per thread: a longer chain on a
// quarter of the SMs.  Same indices in every form (the tie rank does not depend on the layout).
BX_API int bx_fps_ex(const float *xyz, const int32_t *h_offsets, int B, int npoint, int32_t *idx, float *kpts, int max_cluster,
                     void *stream) {
    return bx_fps_n(xyz, h_offsets, B, npoint, idx, kpts, max_cluster, nullptr, stream);
}

// d_counts (optional, device, B ints): cloud b holds min(max(d_counts[b], 1), h_offsets[b+1] - h_offsets[b]) points at
// h_offsets[b]; the launch is sized by the capacities, so one captured launch serves every count up to them.
BX_API int bx_fps_n(const float *xyz, const int32_t *h_offsets, int B, int npoint, int32_t *idx, float *kpts, int max_cluster,
                    const int32_t *d_counts, void *stream) {
    BX_REQUIRE(xyz && h_offsets && idx, "bx_fps: null pointer");
    BX_REQUIRE(B >= 1 && B <= kMaxClouds, "bx_fps: B=%d out of range [1,%d]", B, kMaxClouds);
    BX_REQUIRE(npoint >= 0, "bx_fps: npoint < 0");
    if (npoint == 0) return BX_OK;
    int maxN = 0;
    for (int b = 0; b < B; ++b) {
        const int n = h_offsets[b + 1] - h_offsets[b];
        BX_REQUIRE(n >= 1, "bx_fps: cloud %d is empty", b);
        if (n > maxN) maxN = n;
    }
    BX_REQUIRE(maxN <= 524288, "bx_fps: N=%d exceeds the 524288-point register budget of one 16-CTA cluster", maxN);
    cudaStream_t st = bx_stream(stream);
    FpsOffsets d_off;
    for (int b = 0; b <= kMaxClouds; ++b) d_off.v[b] = h_offsets[b <= B ? b : B];
    const int *dc = d_counts;
    int hi;
    switch (fps_tier(maxN, max_cluster, &hi)) {
        case T256x2: return launch_fps<256, 2>(xyz, d_off, B, 8, npoint, idx, kpts, dc, st);
        case T256x4: return launch_fps<256, 4>(xyz, d_off, B, 8, npoint, idx, kpts, dc, st);
        case T1024x4c: return launch_fps<1024, 4>(xyz, d_off, B, max_cluster >= 4 ? 4 : 2, npoint, idx, kpts, dc, st);
        case T1024x6c: return launch_fps<1024, 6>(xyz, d_off, B, max_cluster >= 4 ? 4 : 2, npoint, idx, kpts, dc, st);
        case T1024x10c: return launch_fps<1024, 10>(xyz, d_off, B, max_cluster >= 4 ? 4 : 2, npoint, idx, kpts, dc, st);
        case T1024x12c: return launch_fps<1024, 12>(xyz, d_off, B, max_cluster >= 4 ? 4 : 2, npoint, idx, kpts, dc, st);
        case T1024x1c16: return launch_fps<1024, 1>(xyz, d_off, B, 16, npoint, idx, kpts, dc, st);
        case T1024x2c16: return launch_fps<1024, 2>(xyz, d_off, B, 16, npoint, idx, kpts, dc, st);
        case T1024x2: return launch_fps<1024, 2>(xyz, d_off, B, 8, npoint, idx, kpts, dc, st);
        case T1024x3: return launch_fps<1024, 3>(xyz, d_off, B, 8, npoint, idx, kpts, dc, st);
        case T1024x4: return launch_fps<1024, 4>(xyz, d_off, B, 8, npoint, idx, kpts, dc, st);
        case T1024x8: return launch_fps<1024, 8>(xyz, d_off, B, 8, npoint, idx, kpts, dc, st);
        case T1024x8c16: return launch_fps<1024, 8>(xyz, d_off, B, 16, npoint, idx, kpts, dc, st);
        case T512x32: return launch_fps<512, 32>(xyz, d_off, B, 16, npoint, idx, kpts, dc, st);
        default: return launch_fps<512, 64>(xyz, d_off, B, 16, npoint, idx, kpts, dc, st);
    }
}

// Size class of a cloud of n points: the largest point count whose launch gets the same configuration as n (n <= 0: 0;
// n > 524288: -1, no launch exists).  Capacity buffers of this size keep the kernel on n's register tier.
BX_API int bx_fps_size_class(int n, int max_cluster) {
    if (n <= 0) return 0;
    if (n > 524288) return -1;
    int hi;
    fps_tier(n, max_cluster, &hi);
    return hi;
}
