// bx_fps_large.cu -- a1 for clouds beyond one cluster's registers: farthest point sampling of ONE cloud of up to
// 1638400 points, spread over G = ceil(N / 18432) SMs of a cooperative grid (G <= 89).
//
// Replaces pointnet2_ops.furthest_point_sample (+gather_operation) as the reference calls it at models/BUFFERX.py:286-290
// for the clouds bx_fps cannot hold (N > 524288).  Result contract: the one in the header of bx_fps.cu, unchanged, and
// bit-exact with oracle/c/bx_oracle.c::bxo_fps -- idx[0] = 0; candidates with |p|^2 <= 1e-3 (double compare) never win;
// d = ((dx*dx)+(dy*dy))+(dz*dz) (compiled with -fmad=false); ties go to the maximum of (value, -bitrev(k mod bs), -k) with
// bs = min(512, 2^floor(log2 N)).  So any N gives the indices of bx_fps.
//
// Layout: CTA c of 1024 threads keeps points k = s * (G * 1024) + c * 1024 + tid, s < 18, with their coordinates in shared
// memory (12 bytes a point, 216 KiB) and their running minimum distances in registers.  Because the stride is a multiple of
// 512, k mod bs is the same for every point of a thread, so within a thread the tie rank grows with s and the first strict
// maximum wins; the rank is formed once per iteration, for the thread's best point.
//
// An iteration: register / shared-memory scan -> warp reduction -> __syncthreads -> warp 0 reduces the CTA's 32 warps,
// posts the CTA's candidate (fp32 distance bits, ~rank, xyz) to a global slot indexed by iteration parity and arrives on a
// grid-wide counter (release) -> warp 0 waits for G * j arrivals (acquire) and reduces the G candidates -> __syncthreads
// -> every thread takes the winner.  Every CTA reduces the same candidates under a total order, so all agree on the winner
// without a second exchange.  Slots are double-buffered: a CTA can only be one iteration ahead of the slowest (its next
// wait needs everybody's next arrival, which follows their read of the current slots).
//
// Count form (bx_fps_large_n, size-class slots): the grid is sized for a capacity and the kernel reads the point count
// from the device.  The layout argument above holds for any G, so the indices are still those of bx_fps for every N; the
// points of a CTA whose range lies beyond N start (and stay) skipped, so it posts the "none" candidate each iteration.
//
// The grid waits on itself, so it must be co-resident: the launch is cooperative (cudaLaunchAttributeCooperative), which
// the driver schedules all at once or not at once, whatever other streams have in flight, and which stream capture turns
// into a cooperative graph node.
#include "bx_common.cuh"

namespace {

constexpr int kThreads = 1024;
constexpr int kPpt = 18;                               // points per thread
constexpr int kPerCta = kThreads * kPpt;               // 18432 points per CTA
constexpr int kSmemBytes = 12 * kPerCta;               // x, y, z planes: 221184 bytes
constexpr int kMaxN = 1638400;                         // the patch gatherer's shared-memory bitmap (bx_patches.cu)
constexpr int kMaxCtas = (kMaxN + kPerCta - 1) / kPerCta;
constexpr size_t kSlotsOffset = 128;                   // workspace: arrival counter, then [2][G] 32-byte candidate slots

struct Cand {
    uint32_t hi, lo;  // hi = fp32 bits of the (non-negative) distance, lo = ~rank  (0,0) = "none" -> index 0
    float x, y, z;
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

__device__ __forceinline__ bool better(uint32_t hi, uint32_t lo, const Cand &b) { return hi > b.hi || (hi == b.hi && lo > b.lo); }

__device__ __forceinline__ void arrive_release(unsigned *ctr) {
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
}
__device__ __forceinline__ unsigned load_acquire(const unsigned *ctr) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    return v;
}

// kCount: the grid is sized for a capacity N and the cloud is its first clamp(*d_n, 1, N) points (a size-class slot).
template <bool kCount>
__global__ void __launch_bounds__(kThreads, 1)
fps_grid_kernel(const float *__restrict__ xyz, int N, int npoint, int *__restrict__ idx, float *__restrict__ kp,
                unsigned char *__restrict__ ws, const int *__restrict__ d_n) {
    extern __shared__ float s_xyz[];                    // [3][kPerCta]
    __shared__ uint4 w_a[32];
    __shared__ float w_z[32];
    __shared__ float win[3];

    const int G = (int)gridDim.x, cta = (int)blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    unsigned *ctr = reinterpret_cast<unsigned *>(ws);
    uint4 *slots = reinterpret_cast<uint4 *>(ws + kSlotsOffset);      // [2][G][2]
    if constexpr (kCount) N = min(max(*d_n, 1), N);                   // CTAs whose range is empty post "none"

    int log2bs = 0;
    while ((2 << log2bs) <= N && log2bs < 9) ++log2bs;  // bs = min(512, 2^floor(log2 N))
    const int bs = 1 << log2bs;
    const uint32_t cpb = (uint32_t)((N + bs - 1) >> log2bs);
    const int stride = G * kThreads;
    const int base = cta * kThreads + tid;
    const uint32_t tr = log2bs ? (__brev((uint32_t)(base & (bs - 1))) >> (32 - log2bs)) : 0u;   // k mod bs = base mod bs

    float tmp[kPpt];
#pragma unroll
    for (int s = 0; s < kPpt; ++s) {
        const int k = s * stride + base;
        const int li = s * kThreads + tid;
        if (k < N) {
            const float x = xyz[3 * (size_t)k], y = xyz[3 * (size_t)k + 1], z = xyz[3 * (size_t)k + 2];
            s_xyz[li] = x;
            s_xyz[kPerCta + li] = y;
            s_xyz[2 * kPerCta + li] = z;
            const float mag = ((x * x) + (y * y)) + (z * z);
            tmp[s] = ((double)mag <= 1e-3) ? -1.0f : 1e10f;
        } else {
            tmp[s] = -1.0f;
        }
    }
    const float p0x = xyz[0], p0y = xyz[1], p0z = xyz[2];
    float ox = p0x, oy = p0y, oz = p0z;
    if (cta == 0 && tid == 0 && npoint > 0) {
        idx[0] = 0;
        if (kp) { kp[0] = p0x; kp[1] = p0y; kp[2] = p0z; }
    }

    for (int j = 1; j < npoint; ++j) {
        const int par = j & 1;
        // thread scan: the first strict maximum in s order is the thread's best (its rank grows with s)
        int bhi = -1, bslot = 0;
#pragma unroll
        for (int s = 0; s < kPpt; ++s) {
            if (tmp[s] >= 0.0f) {
                const int li = s * kThreads + tid;
                const float d = bx_d2(s_xyz[li] - ox, s_xyz[kPerCta + li] - oy, s_xyz[2 * kPerCta + li] - oz);
                const float d2 = fminf(d, tmp[s]);
                tmp[s] = d2;
                const int hi = (int)__float_as_uint(d2);
                if (hi > bhi) { bhi = hi; bslot = s; }
            }
        }
        Cand best;
        best.hi = 0u; best.lo = 0u; best.x = p0x; best.y = p0y; best.z = p0z;
        if (bhi >= 0) {
            const int li = bslot * kThreads + tid;
            best.hi = (uint32_t)bhi;
            best.lo = ~(tr * cpb + (uint32_t)((bslot * stride + base) >> log2bs));
            best.x = s_xyz[li]; best.y = s_xyz[kPerCta + li]; best.z = s_xyz[2 * kPerCta + li];
        }
        const Cand wb = warp_best(best);
        if (lane == 0) {
            w_a[warp] = make_uint4(wb.hi, wb.lo, __float_as_uint(wb.x), __float_as_uint(wb.y));
            w_z[warp] = wb.z;
        }
        __syncthreads();
        if (warp == 0) {
            const uint4 a = w_a[lane];
            Cand c;
            c.hi = a.x; c.lo = a.y; c.x = __uint_as_float(a.z); c.y = __uint_as_float(a.w); c.z = w_z[lane];
            const Cand cb = warp_best(c);
            uint4 *mine = slots + 2 * ((size_t)par * G + cta);
            if (lane == 0) {
                __stcg(mine, make_uint4(cb.hi, cb.lo, __float_as_uint(cb.x), __float_as_uint(cb.y)));
                __stcg(mine + 1, make_uint4(__float_as_uint(cb.z), 0u, 0u, 0u));
                arrive_release(ctr);                    // orders the two stores before the arrival
            }
            const unsigned target = (unsigned)G * (unsigned)j;
            while (load_acquire(ctr) < target) {}      // every lane acquires: the slot loads below follow it
            Cand g;
            g.hi = 0u; g.lo = 0u; g.x = p0x; g.y = p0y; g.z = p0z;
            for (int q = lane; q < G; q += 32) {        // L2 loads (.cg): the slots are written by other SMs
                const uint4 *sl = slots + 2 * ((size_t)par * G + q);
                const uint4 v = __ldcg(sl);
                if (better(v.x, v.y, g)) {
                    g.hi = v.x; g.lo = v.y; g.x = __uint_as_float(v.z); g.y = __uint_as_float(v.w);
                    g.z = __uint_as_float(__ldcg(sl + 1).x);
                }
            }
            const Cand w = warp_best(g);
            if (lane == 0) {
                win[0] = w.x; win[1] = w.y; win[2] = w.z;
                if (cta == 0) {
                    int k = 0;
                    if (w.hi != 0u || w.lo != 0u) {
                        const uint32_t rk = ~w.lo;
                        const uint32_t t = rk / cpb;
                        const uint32_t tb = log2bs ? (__brev(t) >> (32 - log2bs)) : 0u;
                        k = (int)((rk % cpb) << log2bs) + (int)tb;
                    }
                    idx[j] = k;
                    if (kp) { kp[3 * j] = w.x; kp[3 * j + 1] = w.y; kp[3 * j + 2] = w.z; }
                }
            }
        }
        __syncthreads();
        ox = win[0]; oy = win[1]; oz = win[2];
    }
}

int grid_ctas(int n) { return (n + kPerCta - 1) / kPerCta; }

// Size classes above 524288 points: CTA counts on a ladder where each capacity is at most 1.25x the smallest cloud of its
// class (the first one at most 1.25x 524289), then the 1638400-point limit.
constexpr int kClassCtas[] = {35, 43, 53, 66, 82};

template <bool kCount>
int launch(const char *name, const float *xyz, int n, const int32_t *d_n, int npoint, int32_t *idx, float *kpts, void *workspace,
           void *stream) {
    BX_REQUIRE(xyz && idx && workspace && (!kCount || d_n), "%s: null pointer", name);
    BX_REQUIRE(n >= 1, "%s: the cloud is empty", name);
    BX_REQUIRE(n <= kMaxN, "%s: N=%d exceeds the %d-point limit (the patch gatherer's shared-memory bitmap)", name, n, kMaxN);
    BX_REQUIRE(npoint >= 0, "%s: npoint < 0", name);
    BX_REQUIRE(((uintptr_t)workspace & 15) == 0, "%s: workspace must be 16-byte aligned", name);
    if (npoint == 0) return BX_OK;
    const int G = grid_ctas(n);
    static_assert(kMaxCtas <= 96, "the candidate reduction takes at most three slots per lane");
    const int sms = bx_device_sm_count();
    BX_REQUIRE(sms > 0, "%s: no CUDA device", name);
    BX_REQUIRE(G <= sms, "%s: N=%d needs %d co-resident CTAs, the device has %d SMs", name, n, G, sms);
    cudaStream_t st = bx_stream(stream);
    static BxPerDevice attr = {};
    if (bx_needs_attr(attr))
        BX_CUDA(cudaFuncSetAttribute(fps_grid_kernel<kCount>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    BX_CUDA(cudaMemsetAsync(workspace, 0, sizeof(unsigned), st));      // the arrival counter
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)G);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = kSmemBytes;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative;
    at[0].val.cooperative = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    BX_CUDA(cudaLaunchKernelEx(&cfg, fps_grid_kernel<kCount>, xyz, n, npoint, (int *)idx, kpts, (unsigned char *)workspace,
                               (const int *)d_n));
    ++g_bx_launches;
    return BX_OK;
}

}  // namespace

BX_API long long bx_fps_large_workspace_bytes(int n) {
    if (n < 1) n = 1;
    return (long long)kSlotsOffset + 2LL * grid_ctas(n < kMaxN ? n : kMaxN) * 32;
}

BX_API int bx_fps_large(const float *xyz, int n, int npoint, int32_t *idx, float *kpts, void *workspace, void *stream) {
    return launch<false>("bx_fps_large", xyz, n, nullptr, npoint, idx, kpts, workspace, stream);
}

BX_API int bx_fps_large_n(const float *xyz, int cap, const int32_t *d_n, int npoint, int32_t *idx, float *kpts, void *workspace,
                          void *stream) {
    return launch<true>("bx_fps_large_n", xyz, cap, d_n, npoint, idx, kpts, workspace, stream);
}

BX_API int bx_fps_large_size_class(int n) {
    if (n <= 524288) return bx_fps_size_class(n);
    if (n > kMaxN) return -1;
    for (const int g : kClassCtas)
        if (n <= g * kPerCta) return g * kPerCta;
    return kMaxN;
}
