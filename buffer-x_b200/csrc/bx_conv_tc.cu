// bx_conv_tc.cu -- a8/a11 convolution stacks on the Hopper tensor cores (wgmma, TF32 operands).
//
// Implicit GEMM: rows = (sample, output position), cols = Cout, K = taps*Cin.  The circular-azimuth / zero-elevation
// padding and the valid-convolution geometry are folded into the per-row, per-tap input offset computed by the loader (no
// padded copies); BatchNorm (eval) is folded into the weights and bias on the host.  The inner product runs as wgmma .tf32
// with fp32 accumulators in registers.
// fp32-grade accuracy (descriptor parity 1e-4 rel) needs two things:
//   1. the 3xTF32 split  x = hi + lo  (hi = x with the 13 low mantissa bits cleared, lo = x - hi, exact):
//          a*b ~= ah*bh + ah*bl + al*bh          (dropped al*bl ~ 2^-20 relative)
//   2. short accumulation chains: the tensor core does not round its internal accumulation to nearest, so the error of a
//      chain grows with its length.  The products of seg_len stages (default 4 = 24 MMAs) go to a fresh accumulator that
//      is then added with round-to-nearest into fp32 running sums (tools/tc_precision.py measures the effect of seg_len).
//
// Warp-specialised CTA (416 threads, 128 GEMM rows = one tile, N = NT columns):
//   loader warps  four warps, thread -> row.  Per stage (16 input channels of one tap; chunk-outer / tap-inner order keeps a
//               chunk's activations in L1 across its taps; tap geometry from a shared table) a thread fetches its row's 16
//               activations with four 16-byte loads (channel-blocked activations [n][C/4][position][4]), splits them and
//               writes hi / lo into the A ring in shared memory, the canonical K-major no-swizzle image
//               [split][kq(4)][row(128)][4 x fp32] (LBO = one kq image = 2 KB, SBO = 128 B).
//   weight thread streams the host-arranged B (weight) images
//                   [kstep][split][kunit][n(NT)][16 B]      K-major no-swizzle, LBO = NT*16 B, SBO = 128 B
//               through a shared-memory ring with cp.async.bulk + mbarrier transaction counts, up to TC_NBS stages ahead.
//   2 MMA warpgroups  warpgroup g owns tile rows 64 g .. 64 g + 63: per stage 6 wgmmas (2 k-steps x {al*bh, ah*bl, ah*bh},
//               small terms first); a stage's slots are released once the NEXT stage's MMAs are in flight (wgmma.wait_group 1),
//               every seg_len stages the accumulators are folded into the running sums; epilogue: bias (+ReLU) ->
//               channel-blocked stores.
#include "bx_common.cuh"
#include "bx_wgmma.cuh"

namespace {

struct ConvTcParams {
    const float *in, *w, *bias;
    float *out;
    int n;
    const int *d_n;
    int Cin, Cout, D, H, W, kd, kh, kw, relu;
    int S_in, S_out, OD, OH, OW, T;
    int seg_len;  // stages per accumulator segment
    const float *equi_s, *equi_t;  // COSTAB: the factor maps A and B of bx_costvol_ab
    // Unused.  Without these 16 bytes ptxas schedules every instantiation differently; they keep the generated code the
    // one whose speed the project has measured.
    const void *reserved[2];
};

constexpr int TC_BM = 128;
constexpr int TC_STAGES = 4;              // A ring (shared memory)
constexpr int TC_NBS = 8;                 // B ring: weights are prefetched independently of the A slots
constexpr int TC_MAX_TAPS = 128;
constexpr int TC_NC = 8, TC_NL = 4;       // MMA warps (two warpgroups), loader warps
constexpr int TC_THREADS = (TC_NC + TC_NL + 1) * 32;
constexpr int TC_AIMG = TC_BM * 64;       // one split of an A stage: [kq(4)][row(128)][4 x fp32] = 8 KB
constexpr int TC_ASTAGE = 2 * TC_AIMG;

template <int NT> constexpr int tc_smem() { return TC_STAGES * TC_ASTAGE + TC_NBS * (2 * 2 * 2 * NT * 16); }

template <int GEOM, int NT>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const ConvTcParams p) {
    constexpr int B_STAGE = 2 * 2 * 2 * NT * 16;  // [kstep][split][kunit][n][16B]
    constexpr int BAR_AEMPTY = TC_STAGES, BAR_BFULL = 2 * TC_STAGES, BAR_BEMPTY = BAR_BFULL + TC_NBS;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) unsigned long long bars[2 * TC_STAGES + 2 * TC_NBS];
    __shared__ int4 tap_tab[TC_MAX_TAPS];

    const int n_samples = p.d_n ? *p.d_n : p.n;
    const long long Mtotal = (long long)n_samples * p.S_out;
    const long long row0 = (long long)blockIdx.x * TC_BM;
    if (row0 >= Mtotal) return;  // uniform per CTA, before any barrier
    const int tid = threadIdx.x;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);       // warp-uniform role index (keeps the wgmma issue convergent)
    const int n_iters = (p.Cin / 16) * p.T;  // stage = (16-channel chunk, tap); chunk outer, tap inner

    if (tid < p.T) {   // tap geometry table: no counter arithmetic in the loader loop
        const int dz = tid / (p.kh * p.kw), r = tid - dz * (p.kh * p.kw), dy = r / p.kw, dx = r - dy * p.kw;
        int base = 0;
        if (GEOM == BX_GEOM_CYL3D || GEOM == BX_GEOM_CYL2D) base = dz * 140 + (dy - 1) * 20;
        else if (GEOM == BX_GEOM_VALID3D) base = (dz * p.H + dy) * p.W + dx;
        tap_tab[tid] = make_int4(dz, dy, dx, base);
    }
    if (tid == 0) {
        for (int s = 0; s < TC_STAGES; ++s) {
            mbar_init(smem_u32(&bars[s]), TC_NL);            // A full: the four loader warps
            mbar_init(smem_u32(&bars[BAR_AEMPTY + s]), TC_NC);
        }
        for (int s = 0; s < TC_NBS; ++s) {
            mbar_init(smem_u32(&bars[BAR_BFULL + s]), 1);    // B full: the producer's expect_tx arrival + the bulk copy's bytes
            mbar_init(smem_u32(&bars[BAR_BEMPTY + s]), TC_NC);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    uint32_t a_base = smem_u32(smem);
    uint32_t b_base = a_base + (uint32_t)(TC_STAGES * TC_ASTAGE);
    uint32_t bar_base = smem_u32(&bars[0]);
    asm volatile("" : "+r"(a_base), "+r"(b_base), "+r"(bar_base));

    if (warp >= TC_NC && warp < TC_NC + TC_NL) {
        // =========================== loaders ===========================================================
        const int row = tid - TC_NC * 32;
        const long long lm = row0 + row;
        const bool lvalid = lm < Mtotal;
        int ln = 0, oz = 0, oy = 0, ox = 0;
        if (lvalid) {
            ln = (int)(lm / p.S_out);
            const int pos = (int)(lm - (long long)ln * p.S_out);
            if (GEOM == BX_GEOM_CYL3D || GEOM == BX_GEOM_CYL2D) {
                oy = pos / 20;
                ox = pos - oy * 20;
            } else {
                oz = pos / (p.OH * p.OW);
                const int rem = pos - oz * (p.OH * p.OW);
                oy = rem / p.OW;
                ox = rem - oy * p.OW;
            }
        }
        const float *pa = p.in, *pb = nullptr;
        if (GEOM == BX_GEOM_COSTAB) {
            pa = p.equi_s + (size_t)ln * 32 * 60;     // A, channel-blocked [8][3*20][4]
            pb = p.equi_t + (size_t)ln * 32 * 54;     // B, channel-blocked [8][3*18][4]
        } else {
            pa = p.in + (size_t)ln * p.S_in * p.Cin;      // activations are channel-blocked: [n][Cin/4][position][4]
        }
        // (chunk, tap) of the stage filled next; the tap geometry comes from the shared table
        int chunk = 0, t = 0;
        const int oy20 = oy * 20;
        const int rowbase = (oz * p.H + oy) * p.W + ox;   // VALID3D
        float a_reg[16];

        auto load_stage = [&]() {                       // the stage the counters point at
            const int4 tp = tap_tab[t];                  // (dz, dy, dx, geometry-specific base offset)
            int offA = 0, offB = 0;
            bool ok = lvalid;
            if (GEOM == BX_GEOM_CYL3D || GEOM == BX_GEOM_CYL2D) {
                const int yy = oy + tp.y - 1;
                int xx = ox + tp.z - 1;
                xx = xx < 0 ? xx + 20 : (xx >= 20 ? xx - 20 : xx);
                ok = lvalid && (unsigned)yy < 7u;
                offA = tp.w + oy20 + xx;
            } else if (GEOM == BX_GEOM_VALID3D) {
                offA = rowbase + tp.w;
            } else {  // COSTAB: value(c, n, k, l) = relu(A[c][k][(l-n) mod 20] - B[c][k][l])
                const int nn = oz + tp.x, kk = oy + tp.y, ll = ox + tp.z;
                int sh = ll - nn;
                sh = sh < 0 ? sh + 20 : sh;
                offA = kk * 20 + sh;
                offB = kk * 18 + ll;
            }
            const int c0 = chunk * 16;
            if (GEOM == BX_GEOM_COSTAB) {   // relu(A - B) from the channel-blocked factors: 2 x four 16-byte loads
                const float4 *sa = reinterpret_cast<const float4 *>(pa) + (chunk * 4) * 60 + offA;
                const float4 *sb4 = reinterpret_cast<const float4 *>(pb) + (chunk * 4) * 54 + offB;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float4 va = make_float4(0.0f, 0.0f, 0.0f, 0.0f), vb = va;
                    if (ok) { va = __ldg(sa + q * 60); vb = __ldg(sb4 + q * 54); }
                    a_reg[4 * q] = fmaxf(va.x - vb.x, 0.0f); a_reg[4 * q + 1] = fmaxf(va.y - vb.y, 0.0f);
                    a_reg[4 * q + 2] = fmaxf(va.z - vb.z, 0.0f); a_reg[4 * q + 3] = fmaxf(va.w - vb.w, 0.0f);
                }
            } else {  // four 16-byte loads, one per group of 4 channels; a warp's 32 rows read 512 contiguous bytes each
                const float4 *src = reinterpret_cast<const float4 *>(pa) + (size_t)(chunk * 4) * p.S_in + offA;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                    if (ok) v = __ldg(src + (size_t)q * p.S_in);
                    a_reg[4 * q] = v.x; a_reg[4 * q + 1] = v.y; a_reg[4 * q + 2] = v.z; a_reg[4 * q + 3] = v.w;
                }
            }
        };
        // registers -> shared memory: hi = x with the low 13 mantissa bits cleared, lo = x - hi (exact)
        auto store_stage = [&](int s) {
            unsigned char *dst = smem + (size_t)s * TC_ASTAGE + (size_t)row * 16;
#pragma unroll
            for (int kq = 0; kq < 4; ++kq) {
                float hi[4], lo[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    hi[j] = __uint_as_float(__float_as_uint(a_reg[kq * 4 + j]) & 0xFFFFE000u);
                    lo[j] = a_reg[kq * 4 + j] - hi[j];
                }
                *reinterpret_cast<float4 *>(dst + (size_t)kq * TC_BM * 16) = make_float4(hi[0], hi[1], hi[2], hi[3]);
                *reinterpret_cast<float4 *>(dst + TC_AIMG + (size_t)kq * TC_BM * 16) = make_float4(lo[0], lo[1], lo[2], lo[3]);
            }
        };
        load_stage();
        for (int it = 0; it < n_iters; ++it) {
            const int s = it % TC_STAGES;
            if (it >= TC_STAGES) mbar_wait(bar_base + 8u * (BAR_AEMPTY + s), (uint32_t)((it / TC_STAGES - 1) & 1));   // the MMAs have read the slot
            store_stage(s);
            if (it + 1 < n_iters) {                       // the next stage's activations go in flight behind the stores
                if (++t == p.T) { t = 0; ++chunk; }
                load_stage();
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy stores -> tensor-core (async proxy) reads
            __syncwarp();
            if ((tid & 31) == 0) mbar_arrive(bar_base + 8u * s);
        }
    } else if (warp < TC_NC) {
        // =========================== MMA warpgroups ======================================================
        const int lane = tid & 31, wg = warp >> 2;
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);         // fragment rows r0 and r0 + 8 of the tile
        const int cq = 2 * (lane & 3);                                   // fragment column within an 8-column group
        constexpr uint32_t DESC_HI = 128u >> 4;                          // SBO = 128 B
        constexpr uint32_t A_LBO = ((uint32_t)(TC_BM * 16) >> 4) << 16, B_LBO = ((uint32_t)(NT * 16) >> 4) << 16;
        constexpr uint32_t B_IMG = (2u * NT * 16) >> 4;                  // one (kstep, split) image of B, in 16-byte units
        const uint32_t a0 = ((a_base + (uint32_t)wg * 64u * 16u) >> 4) | A_LBO;
        const uint32_t b0 = (b_base >> 4) | B_LBO;
        const int G = p.seg_len;
        float run[NT / 2], acc[NT / 2];
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) run[i] = 0.0f;
        int in_seg = 0, pend = -1;                      // pend: the stage whose slots are released after the next wait
        auto release = [&](int it) {
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(bar_base + 8u * (BAR_AEMPTY + it % TC_STAGES));
                mbar_arrive(bar_base + 8u * (BAR_BEMPTY + it % TC_NBS));
            }
        };
        for (int it = 0; it < n_iters; ++it) {
            const int s = it % TC_STAGES, sb = it % TC_NBS;
            mbar_wait(bar_base + 8u * (BAR_BFULL + sb), (uint32_t)((it / TC_NBS) & 1));
            mbar_wait(bar_base + 8u * s, (uint32_t)((it / TC_STAGES) & 1));
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const uint32_t ah = a0 + (uint32_t)(s * TC_ASTAGE + ks * 2 * TC_BM * 16) / 16u, al = ah + (uint32_t)TC_AIMG / 16u;
                const uint32_t bh = b0 + (uint32_t)sb * ((uint32_t)B_STAGE >> 4) + (uint32_t)(ks * 2) * B_IMG, bl = bh + B_IMG;
                wgmma_tf32<NT>(acc, gmma_desc(al, DESC_HI), gmma_desc(bh, DESC_HI), (in_seg == 0 && ks == 0) ? 0u : 1u);
                wgmma_tf32<NT>(acc, gmma_desc(ah, DESC_HI), gmma_desc(bl, DESC_HI), 1u);
                wgmma_tf32<NT>(acc, gmma_desc(ah, DESC_HI), gmma_desc(bh, DESC_HI), 1u);
            }
            wgmma_commit();
            if (++in_seg == G || it == n_iters - 1) {      // segment done: fold it into the running sums
                wgmma_wait<0>();
                wgmma_fence_regs<NT / 2>(acc);
                if (pend >= 0) release(pend);
                release(it);
                pend = -1;
#pragma unroll
                for (int i = 0; i < NT / 2; ++i) run[i] += acc[i];
                in_seg = 0;
            } else {
                wgmma_wait<1>();                            // the previous stage's MMAs are done
                if (pend >= 0) release(pend);
                pend = it;
            }
        }
        // ---- epilogue: running sums + bias (+ReLU) -> channel-blocked [n][Cout/4][position][4] ----------------------
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const long long em = row0 + r0 + 8 * half;
            if (em < Mtotal) {
                const int en = (int)(em / p.S_out);
                const int epos = (int)(em - (long long)en * p.S_out);
                float *eo = p.out + ((size_t)en * (p.Cout >> 2) * p.S_out + epos) * 4;
#pragma unroll
                for (int j = 0; j < NT / 8; ++j) {
                    const int co = 8 * j + cq;
                    if (co < p.Cout) {
                        float2 r = make_float2(run[4 * j + 2 * half] + __ldg(p.bias + co), run[4 * j + 2 * half + 1] + __ldg(p.bias + co + 1));
                        if (p.relu) { r.x = fmaxf(r.x, 0.0f); r.y = fmaxf(r.y, 0.0f); }
                        *reinterpret_cast<float2 *>(eo + (size_t)(co >> 2) * p.S_out * 4 + (co & 3)) = r;
                    }
                }
            }
        }
    } else {
        // =========================== weight producer ====================================================
        // The weight image of stage `it` is one contiguous block; its order is known in advance, so the producer runs
        // up to TC_NBS stages ahead of the tensor core, independent of the activation slots.
        if ((tid & 31) == 0) {
            for (int it = 0; it < n_iters; ++it) {
                const int sb = it % TC_NBS;
                const uint32_t use = (uint32_t)(it / TC_NBS);
                if (use > 0) mbar_wait(bar_base + 8u * (BAR_BEMPTY + sb), (use - 1) & 1);
                mbar_arrive_expect_tx(bar_base + 8u * (BAR_BFULL + sb), (uint32_t)B_STAGE);
                bulk_g2s(b_base + (uint32_t)(sb * B_STAGE), reinterpret_cast<const unsigned char *>(p.w) + (size_t)it * B_STAGE, (uint32_t)B_STAGE,
                         bar_base + 8u * (BAR_BFULL + sb));
            }
        }
        __syncwarp();
    }
}

template <int GEOM, int NT>
int launch_tc(const ConvTcParams &p, int max_n, cudaStream_t st) {
    const long long maxM = (long long)max_n * p.S_out;
    const unsigned gx = (unsigned)((maxM + TC_BM - 1) / TC_BM);
    if (gx == 0) return BX_OK;
    constexpr int smem = tc_smem<NT>();
    static BxPerDevice attr_done = {};
    if (bx_needs_attr(attr_done))
        BX_CUDA(cudaFuncSetAttribute(conv_tc_kernel<GEOM, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    conv_tc_kernel<GEOM, NT><<<gx, TC_THREADS, smem, st>>>(p);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

template <int GEOM>
int dispatch_nt(const ConvTcParams &p, int max_n, cudaStream_t st) {
    if (p.Cout > 64) return launch_tc<GEOM, 128>(p, max_n, st);
    if (p.Cout > 32) return launch_tc<GEOM, 64>(p, max_n, st);
    return launch_tc<GEOM, 32>(p, max_n, st);
}

}  // namespace

BX_API int bx_conv_tc_ntile(int Cout) { return Cout > 64 ? 128 : (Cout > 32 ? 64 : 32); }

// Tuning knob (experiments / tests): maximum number of 16-channel stages accumulated by the tensor core before the
// accumulators are folded into the running sums with a rounded fp32 add.  <= 0 restores the default.
static int g_tc_max_stages = 4;
BX_API int bx_conv_tc_set_segment_stages(int stages) {
    const int old = g_tc_max_stages;
    g_tc_max_stages = stages > 0 ? stages : 4;
    return old;
}

BX_API int bx_conv_layer_tc(int geom, const float *in, const float *w_tc, const float *bias, float *out, int n,
                            const int32_t *d_n, int Cin, int Cout, int D, int H, int W, int kd, int kh, int kw, int relu,
                            const float *equi_s, const float *equi_t, void *stream) {
    BX_REQUIRE(w_tc && bias && out, "bx_conv_layer_tc: null pointer");
    BX_REQUIRE(n >= 0 && Cin >= 16 && Cin % 16 == 0 && Cout >= 4 && Cout % 4 == 0 && Cout <= 128, "bx_conv_layer_tc: bad channels Cin=%d Cout=%d", Cin, Cout);
    BX_REQUIRE((reinterpret_cast<uintptr_t>(w_tc) & 15) == 0, "bx_conv_layer_tc: weights must be 16-byte aligned");
    BX_REQUIRE(((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(bias)) & 15) == 0,
               "bx_conv_layer_tc: activations and bias must be 16-byte aligned");
    BX_REQUIRE(kd >= 1 && kh >= 1 && kw >= 1 && (long long)kd * kh * kw <= TC_MAX_TAPS, "bx_conv_layer_tc: at most %d kernel taps", TC_MAX_TAPS);
    ConvTcParams p = {};
    p.in = in; p.w = w_tc; p.bias = bias; p.out = out; p.n = n; p.d_n = d_n;
    p.Cin = Cin; p.Cout = Cout; p.D = D; p.H = H; p.W = W; p.kd = kd; p.kh = kh; p.kw = kw; p.relu = relu;
    p.equi_s = equi_s; p.equi_t = equi_t;
    p.T = kd * kh * kw;
    p.seg_len = g_tc_max_stages;
    cudaStream_t st = bx_stream(stream);
    switch (geom) {
        case BX_GEOM_CYL3D:
            BX_REQUIRE(in && D == 3 && H == 7 && W == 20 && kd == 3 && kh == 3 && kw == 3, "bx_conv_layer_tc: CYL3D expects [C,3,7,20], k=3x3x3");
            p.S_in = 420; p.S_out = 140; p.OD = 1; p.OH = 7; p.OW = 20;
            return dispatch_nt<BX_GEOM_CYL3D>(p, n, st);
        case BX_GEOM_CYL2D:
            BX_REQUIRE(in && D == 1 && H == 7 && W == 20 && kd == 1 && kh == 3 && kw == 3, "bx_conv_layer_tc: CYL2D expects [C,7,20], k=3x3");
            p.S_in = 140; p.S_out = 140; p.OD = 1; p.OH = 7; p.OW = 20;
            return dispatch_nt<BX_GEOM_CYL2D>(p, n, st);
        case BX_GEOM_VALID3D:
            BX_REQUIRE(in && D >= kd && H >= kh && W >= kw && kd >= 1 && kh >= 1 && kw >= 1, "bx_conv_layer_tc: VALID3D kernel larger than input");
            p.OD = D - kd + 1; p.OH = H - kh + 1; p.OW = W - kw + 1;
            p.S_in = D * H * W; p.S_out = p.OD * p.OH * p.OW;
            return dispatch_nt<BX_GEOM_VALID3D>(p, n, st);
        case BX_GEOM_COSTAB:
            BX_REQUIRE(equi_s && equi_t, "bx_conv_layer_tc: COSTAB needs the A and B factors");
            BX_REQUIRE(Cin == 32 && D == 18 && H == 3 && W == 18 && kd == 3 && kh == 3 && kw == 3, "bx_conv_layer_tc: COSTAB expects the [32,18,3,18] activation, k=3x3x3");
            p.OD = 16; p.OH = 1; p.OW = 16; p.S_in = 972; p.S_out = 256;
            return dispatch_nt<BX_GEOM_COSTAB>(p, n, st);
        default:
            bx_set_error("bx_conv_layer_tc: unknown geometry %d", geom);
            return BX_ERR_INVALID_ARG;
    }
}
