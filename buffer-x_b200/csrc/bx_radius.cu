// bx_radius.cu -- a2: density-aware radius estimation without the [Kr,N] distance matrix.
//
// Replaces density_aware_radius_estimation + squared_cdist
// (/root/reference/models/BUFFERX.py:610-696).  The reference materialises the [Kr,N] fp32 matrix
// (160 MB at Kr=2000, N=20000) three times per pair and runs ~13 bisection steps per scale, each
// with a full-matrix compare + a .item() host sync.  Every radius the bisection can probe is
// r_m = 5*m/8192, so ONE pass that histograms each d2 over those 8192 candidates serves every
// threshold of the pair; the bisection itself then runs on the device on the cumulative histogram.
//
// Bit contract (oracle/c/bx_oracle.c::bxo_radius_hist / bxo_radius_bisect):
//   d2 = (|k|^2 + |p|^2) - 2*(k.p), norms and dot as ((x*x)+(y*y))+(z*z), fp32, no FMA
//   keep d2 <= 25;  count(m) = #{d2 < float32(r_m*r_m)};  pct = (float(count)/float(denom))*100 (fp32)
#include "bx_common.cuh"

namespace {

constexpr int NB = BX_RADIUS_BINS;  // 8192
constexpr int HT = 256;             // threads
constexpr int KT = 500;             // key-points per smem tile (float4 each)

constexpr int kSub = BX_RADIUS_SUBSAMPLE;  // 200000

// hist[m] (m in 0..NB+1) = #{d2 : smallest m with d2 < thr[m]}, bin NB+1 = "d2 == 25".
// kSubsampled (pair form only): a chosen cloud of more than kSub points is read through the kSub indices d_sub.
template <bool kSubsampled>
__global__ void __launch_bounds__(HT)
radius_hist_kernel(const float *__restrict__ kpts, int Kr, const float *__restrict__ pts, int N,
                   uint32_t *__restrict__ hist, const float *__restrict__ kpts_t, const float *__restrict__ pts_t, int N_t,
                   const int *__restrict__ d_counts, const int *__restrict__ d_sub) {
    if (d_counts) {     // pair form: the larger cloud by the reference's rule (source iff Ns > Nt), counts clamped to the capacities
        const int ns = min(max(d_counts[0], 0), N), nt = min(max(d_counts[1], 0), N_t);
        if (ns > nt) {
            N = ns;
        } else {
            kpts = kpts_t; pts = pts_t; N = nt;
        }
    }
    [[maybe_unused]] const int n_full = N;  // kSubsampled: the chosen cloud's size (indices are clamped to it), N the sample size
    if constexpr (kSubsampled) {
        if (N > kSub) N = kSub;
        else d_sub = nullptr;
    }
    extern __shared__ unsigned char smem_raw[];
    float *thr = reinterpret_cast<float *>(smem_raw);                 // NB+1
    uint32_t *sh = reinterpret_cast<uint32_t *>(thr + (NB + 1));      // NB+2
    float4 *kq = reinterpret_cast<float4 *>(sh + (NB + 2) + 1);       // KT  (16-byte aligned: (2*NB+4)*4)
    for (int m = threadIdx.x; m <= NB; m += HT) {
        const double r = 5.0 * (double)m / (double)NB;
        thr[m] = (float)(r * r);
    }
    for (int m = threadIdx.x; m < NB + 2; m += HT) sh[m] = 0u;
    __syncthreads();
    const float scale = (float)NB / 5.0f;
    // blockIdx.y owns a chunk of KT key-points (staged once), blockIdx.x grid-strides over the points
    {
        const int k0 = blockIdx.y * KT;
        const int kn = min(KT, Kr - k0);
        for (int i = threadIdx.x; i < kn; i += HT) {
            const float x = kpts[3 * (size_t)(k0 + i)], y = kpts[3 * (size_t)(k0 + i) + 1], z = kpts[3 * (size_t)(k0 + i) + 2];
            kq[i] = make_float4(x, y, z, ((x * x) + (y * y)) + (z * z));
        }
        __syncthreads();
        for (int p = blockIdx.x * HT + threadIdx.x; p < N; p += gridDim.x * HT) {
            int pi = p;
            if constexpr (kSubsampled) {
                if (d_sub) pi = min(max(d_sub[p], 0), n_full - 1);
            }
            const float px = pts[3 * (size_t)pi], py = pts[3 * (size_t)pi + 1], pz = pts[3 * (size_t)pi + 2];
            const float p2 = ((px * px) + (py * py)) + (pz * pz);
            for (int i = 0; i < kn; ++i) {
                const float4 q = kq[i];
                const float dot = ((q.x * px) + (q.y * py)) + (q.z * pz);
                const float d2 = (q.w + p2) - (2.0f * dot);
                if (d2 <= 25.0f) {
                    int m = (int)(sqrtf(fmaxf(d2, 0.0f)) * scale) + 1;  // first guess, then exact fix-up
                    m = min(max(m, 0), NB + 1);
                    while (m > 0 && d2 < thr[m - 1]) --m;
                    while (m <= NB && !(d2 < thr[m])) ++m;
                    atomicAdd(&sh[m], 1u);
                }
            }
        }
    }
    __syncthreads();
    for (int m = threadIdx.x; m < NB + 2; m += HT) {
        const uint32_t v = sh[m];
        if (v) atomicAdd(&hist[m], v);
    }
}

struct Thresholds {
    double v[16];
};

// one CTA: inclusive prefix over hist (in place, uint32: total < 2^32 by contract), then the
// reference's bisection per threshold (one thread each).
__global__ void __launch_bounds__(1024)
radius_bisect_kernel(uint32_t *__restrict__ hist, long long denom, const Thresholds thresholds, int n_thr,
                     double tolerance, const float *__restrict__ round_table, float *__restrict__ out_r,
                     int *__restrict__ out_m, const int *__restrict__ d_counts, int cap_s, int cap_t, int Kr) {
    if (d_counts) {     // pair form: denom = N * Kr of the cloud the histogram was built on
        const int ns = min(max(d_counts[0], 0), cap_s), nt = min(max(d_counts[1], 0), cap_t);
        denom = (long long)(ns > nt ? ns : nt) * (long long)Kr;
    }
    __shared__ uint32_t part[1024];
    const int b0 = threadIdx.x * 9;  // 9 consecutive bins per thread (9*1024 >= NB+1)
    uint32_t loc[9];
    uint32_t sum = 0;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        const int m = b0 + i;
        loc[i] = (m <= NB) ? hist[m] : 0u;
        sum += loc[i];
    }
    part[threadIdx.x] = sum;
    __syncthreads();
    if (threadIdx.x < 32) {  // warp 0: exclusive scan of the 1024 partials, 32 per lane
        uint32_t acc = 0;
        for (int t = 0; t < 32; ++t) acc += part[threadIdx.x * 32 + t];
        uint32_t inc = acc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t n = __shfl_up_sync(BX_FULL, inc, o);
            if ((int)threadIdx.x >= o) inc += n;
        }
        uint32_t run = inc - acc;
        for (int t = 0; t < 32; ++t) {
            const uint32_t v = part[threadIdx.x * 32 + t];
            part[threadIdx.x * 32 + t] = run;
            run += v;
        }
    }
    __syncthreads();
    uint32_t run = part[threadIdx.x];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        const int m = b0 + i;
        run += loc[i];
        if (m <= NB) hist[m] = run;  // #{d2 < thr[m]}
    }
    __threadfence_block();
    __syncthreads();
    if (threadIdx.x < n_thr) {
        const double threshold = thresholds.v[threadIdx.x];
        int lo = 0, hi = NB, m = 0;
        while (5.0 * (double)hi / (double)NB - 5.0 * (double)lo / (double)NB > 1e-3) {
            m = (lo + hi) / 2;
            const float pct = __fmul_rn(__fdiv_rn((float)hist[m], (float)denom), 100.0f);
            const double p = (double)pct;
            if (p < threshold - tolerance) lo = m;
            else if (p > threshold + tolerance) hi = m;
            else break;
        }
        out_r[threadIdx.x] = round_table[m];
        if (out_m) out_m[threadIdx.x] = m;
    }
}

}  // namespace

namespace {

int radius_launch(const float *kpts, int Kr, const float *pts, int N, int64_t denom, const float *kpts_t, const float *pts_t, int N_t,
                  const int32_t *d_counts, const int32_t *d_sub, const double *h_thresholds, int n_thr, double tolerance, const float *round_table,
                  uint32_t *hist, float *out_r, int32_t *out_m, void *stream) {
    cudaStream_t st = bx_stream(stream);
    BX_CUDA(cudaMemsetAsync(hist, 0, sizeof(uint32_t) * (NB + 2), st));
    const size_t smem = sizeof(float) * (NB + 1) + sizeof(uint32_t) * (NB + 3) + sizeof(float4) * KT;
    static BxPerDevice attr_done = {}, attr_sub_done = {};
    if (bx_needs_attr(attr_done))
        BX_CUDA(cudaFuncSetAttribute(radius_hist_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (d_sub && bx_needs_attr(attr_sub_done))
        BX_CUDA(cudaFuncSetAttribute(radius_hist_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int sms = bx_device_sm_count();
    if (sms <= 0) sms = 132;
    const int gy = (Kr + KT - 1) / KT;
    int gx = ((N > N_t ? N : N_t) + HT - 1) / HT;
    const int cap = (4 * sms + gy - 1) / gy;  // ~4 CTAs per SM overall; beyond that grid-stride
    if (gx > cap) gx = cap;
    if (gx < 1) gx = 1;
    if (d_sub)
        radius_hist_kernel<true><<<dim3(gx, gy), HT, smem, st>>>(kpts, Kr, pts, N, hist, kpts_t, pts_t, N_t, d_counts, d_sub);
    else
        radius_hist_kernel<false><<<dim3(gx, gy), HT, smem, st>>>(kpts, Kr, pts, N, hist, kpts_t, pts_t, N_t, d_counts, nullptr);
    BX_LAUNCH_CHECK();
    Thresholds thr;
    for (int i = 0; i < 16; ++i) thr.v[i] = h_thresholds[i < n_thr ? i : 0];
    radius_bisect_kernel<<<1, 1024, 0, st>>>(hist, (long long)denom, thr, n_thr, tolerance, round_table, out_r, out_m, d_counts, N, N_t, Kr);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

}  // namespace

BX_API int bx_radius_estimate(const float *kpts, int Kr, const float *pts, int N, int64_t denom,
                              const double *h_thresholds, int n_thr, double tolerance, const float *round_table,
                              uint32_t *hist, float *out_r, int32_t *out_m, void *stream) {
    BX_REQUIRE(kpts && pts && h_thresholds && round_table && hist && out_r, "bx_radius_estimate: null pointer");
    BX_REQUIRE(Kr >= 1 && N >= 1 && n_thr >= 1 && n_thr <= 16, "bx_radius_estimate: bad sizes Kr=%d N=%d n_thr=%d", Kr, N, n_thr);
    BX_REQUIRE((int64_t)Kr * (int64_t)N < ((int64_t)1 << 32), "bx_radius_estimate: Kr*N must be < 2^32");
    return radius_launch(kpts, Kr, pts, N, denom, nullptr, nullptr, 0, nullptr, nullptr, h_thresholds, n_thr, tolerance, round_table, hist, out_r,
                         out_m, stream);
}

// Pair form with device point counts: the histogram is built on the source cloud iff ns > nt (ns, nt = d_counts clamped to the
// capacities cap_s, cap_t), with denom = N * Kr of that cloud.  The grid is sized by the larger capacity; the counts are
// integer atomics, so the histogram does not depend on how the points are spread over the CTAs.
BX_API int bx_radius_estimate_n(const float *kpts_s, const float *pts_s, int cap_s, const float *kpts_t, const float *pts_t, int cap_t,
                                int Kr, const int32_t *d_counts, const double *h_thresholds, int n_thr, double tolerance,
                                const float *round_table, uint32_t *hist, float *out_r, int32_t *out_m, void *stream) {
    BX_REQUIRE(kpts_s && pts_s && kpts_t && pts_t && d_counts && h_thresholds && round_table && hist && out_r,
               "bx_radius_estimate_n: null pointer");
    BX_REQUIRE(Kr >= 1 && cap_s >= 1 && cap_t >= 1 && n_thr >= 1 && n_thr <= 16, "bx_radius_estimate_n: bad sizes Kr=%d N=%d/%d n_thr=%d",
               Kr, cap_s, cap_t, n_thr);
    BX_REQUIRE((int64_t)Kr * (int64_t)(cap_s > cap_t ? cap_s : cap_t) < ((int64_t)1 << 32), "bx_radius_estimate_n: Kr*N must be < 2^32");
    return radius_launch(kpts_s, Kr, pts_s, cap_s, 0, kpts_t, pts_t, cap_t, d_counts, nullptr, h_thresholds, n_thr, tolerance, round_table,
                         hist, out_r, out_m, stream);
}

// Sub-sampled pair form: as bx_radius_estimate_n, and when the chosen cloud has more than BX_RADIUS_SUBSAMPLE points the
// histogram runs over its points d_sub[0..BX_RADIUS_SUBSAMPLE) (the reference's draw, made by the caller), denom still N * Kr.
// The counts are integer atomics: the same histogram, radii and m as bx_radius_estimate on the gathered cloud.
BX_API int bx_radius_estimate_n_sub(const float *kpts_s, const float *pts_s, int cap_s, const float *kpts_t, const float *pts_t, int cap_t,
                                    int Kr, const int32_t *d_counts, const int32_t *d_sub, const double *h_thresholds, int n_thr,
                                    double tolerance, const float *round_table, uint32_t *hist, float *out_r, int32_t *out_m, void *stream) {
    BX_REQUIRE(kpts_s && pts_s && kpts_t && pts_t && d_counts && d_sub && h_thresholds && round_table && hist && out_r,
               "bx_radius_estimate_n_sub: null pointer");
    BX_REQUIRE(Kr >= 1 && cap_s >= 1 && cap_t >= 1 && n_thr >= 1 && n_thr <= 16,
               "bx_radius_estimate_n_sub: bad sizes Kr=%d N=%d/%d n_thr=%d", Kr, cap_s, cap_t, n_thr);
    const int cap = cap_s > cap_t ? cap_s : cap_t;
    BX_REQUIRE((int64_t)Kr * (int64_t)(cap < kSub ? cap : kSub) < ((int64_t)1 << 32), "bx_radius_estimate_n_sub: Kr*min(N, %d) must be < 2^32", kSub);
    return radius_launch(kpts_s, Kr, pts_s, cap_s, 0, kpts_t, pts_t, cap_t, d_counts, d_sub, h_thresholds, n_thr, tolerance, round_table,
                         hist, out_r, out_m, stream);
}
