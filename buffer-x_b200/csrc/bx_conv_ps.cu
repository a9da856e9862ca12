// bx_conv_ps.cu -- the cylindrical descriptor convolutions (the eight layers of Cylindrical_Net) as a PER-SAMPLE shifted-
// descriptor implicit GEMM on the Hopper tensor cores (wgmma).  Same operands, products and rounding as conv_sd_kernel
// (bx_conv_sd.cu, which keeps the CostNet layers and every fp32-input layer); what changes is the unit of work.
//
//   rows        a sample is the padded 8 x 22 raster of bx_conv_sd.cu: GEMM row r = 22 y + x of sample s is output (s, y, x)
//               and reads padded row 176 s + r + 22 dy + dx for tap (dy, dx).  Every real output (y <= 6, x <= 19) lies in
//               rows 0 .. 151, and 152 = 19 x 8: a sample is ONE m64n152k16 B operand.  conv_sd_kernel computes all 176 rows
//               of a sample in 128-row tiles; rows 152 .. 175 (y = 7) are always dead, so this kernel does 152 / 176 of its
//               MMAs.  The 12 wrap positions inside 0 .. 151 (x = 20, 21) are computed and dropped as there.
//   operands    channels-as-M: the weight image (ops.conv_sd_weights, unchanged) is the A operand, 64 output channels; the
//               sample's shifted activation view is the B operand, N = 152.  A chunk of a sample is its rows 0 .. 197 (its
//               176 rows and the next sample's zero row, the reach of tap (2, 2)) in the presplit image: four bulk copies of
//               198 x 16 B, one per (split, kcore), into the canonical K-major no-swizzle layout.  Tap (dy, dx) is the
//               chunk's base descriptor advanced by 22 dy + dx rows.  The last sample's halo reads the zero row the
//               producing kernel wrote after it (bx_conv_sd_rows leaves 48 rows past the last whole tile, this needs 22).
//   work        Cout 128: unit = one sample, warpgroup g computes channels 64 g .. 64 g + 63 of it and both read the same B
//               bytes.  Cout 64 / <= 32: unit = two samples, warpgroup g owns sample 2u + g (an odd count's last unit
//               recomputes sample 2u in warpgroup 1 and stores nothing).
//   precision   per 16-channel chunk a fresh accumulator [main | cross], folded as run += fma(cross, 2^-11, main) into fp32
//               running sums that start from the bias.  Per output element the products and their order are those of
//               conv_sd_kernel: main = Wh * ah over the nine taps; cross = Wh * al then Wl * ah for Cout 128 (the order of
//               its rows-as-M form), Wl * ah then Wh * al for Cout <= 64 (its channels-as-M form; Cout <= 32 with the P / Q
//               weight blocks, main and cross in fragment rows r / r + 8 of one accumulator).  The outputs are bit-identical.
//               |x| >= 65504 cannot be represented: the epilogue raises *flag and the host re-runs the stack on the TF32
//               kernel, as with conv_sd_kernel.
//   registers   Cout <= 32: 76 accumulators + 38 running sums, one N = 152 pass per chunk.  Cout >= 64: [main | cross] at
//               N = 152 plus the 76 running sums would be 228 registers, more than the 224 of conv_sd_kernel's split leaves
//               beside the loop's addresses (a 240 / 24 split spills), so a chunk is two N passes, rows 0 .. 79 and 80 .. 151,
//               each with its own wait and fold (80 accumulators + 76 sums).  The weights are then read twice per chunk,
//               2 KB per wgmma; the activation bytes once.
//   epilogue    the next layer's presplit image (ReLU, fp16 hi / lo, the wrap columns, the zero row of sample s + 1 and of
//               sample 0), or fp32 channel-blocked for the last layer -- the bytes conv_sd_kernel writes.  A finished sample
//               goes through a shared-memory staging buffer 32 rows at a time.
//   scheduling  persistent CTAs, one per SM, each taking every gridDim.x-th unit; the device sample count d_n bounds the
//               units.  Weights resident when the whole image fits next to two A chunks per warpgroup
//               stream, else streamed in stages of three taps, as in conv_sd_kernel.
#include <cuda_fp16.h>

#include <type_traits>

#include "bx_common.cuh"
#include "bx_wgmma.cuh"

namespace {

constexpr int PS_N = 152;                        // computed rows of a sample (y = 0 .. 6 of the padded raster)
constexpr int PS_SROWS = 176;                    // padded rows per sample (8 x 22)
constexpr int PS_AROWS = 198;                    // rows of a sample's chunk image: 152 + the reach of tap (2, 2) = 46
constexpr int PS_KBYTES = PS_AROWS * 16;         // one (split, kcore) image of a chunk: [row][8 x fp16]
constexpr int PS_CHUNK = 4 * PS_KBYTES;          // [split(hi,lo)][kcore(2)]
constexpr int PS_NC = 8;                         // MMA warps: two warpgroups
constexpr int PS_WGT_WARP = PS_NC + 3;           // weight thread: last warp of the producer warpgroup
constexpr int PS_MAXNA = 12, PS_MAXNBS = 24;     // A chunk slots; weight stages
constexpr int PS_SR = 32;                        // rows per staging round of a finished sample
constexpr int PS_SMEM = 227 * 1024 - 2048;       // dynamic shared memory of one CTA (the rest: barriers, bias)

struct ConvPsParams {
    const __half *in_sd;       // presplit padded input  [nchunks][split,kcore (4)][rows_in][8 x fp16]
    const __half *w;
    const float *bias;
    float *out;                // fp32 channel-blocked output [n][Cout/4][140][4] (OUT_SD = 0)
    __half *out_sd;            // presplit padded output [Cout/16][4][rows_out][8 x fp16] (OUT_SD = 1)
    int *flag;
    const int *d_n;            // optional device-side sample count (<= n)
    long long rows_in, rows_out;
    int n, Cout, nchunks, relu, NA, nbs, resident;
};

template <int NT> struct PsCfg {
    static constexpr int SPU = NT == 128 ? 1 : 2;                 // samples per unit of work
    static constexpr int CH = NT == 32 ? 32 : 64;                 // output channels of one warpgroup
    // N passes over a chunk: Cout <= 32 one of 152 rows; Cout >= 64 one of rows 0 .. 79 and one of rows 80 .. 151, since
    // [main 76 | cross 76] next to 76 running sums does not fit beside the loop's addresses in 240 registers
    static constexpr int NP = NT == 32 ? 1 : 2;
    static constexpr int NB0 = NP == 1 ? PS_N : 80;               // width of pass 0 (pass 1: PS_N - NB0 = 72)
    static constexpr int NACC = NT == 32 ? PS_N / 2 : NB0;        // accumulator registers: [main 40 | cross 40], or P / Q rows
    static constexpr int NRUN = NT == 32 ? PS_N / 4 : PS_N / 2;   // running sums
    static constexpr int THREADS = (PS_NC + 4) * 32;
    static constexpr int PROD_REGS = 56, MMA_REGS = 224;          // the split of conv_sd_kernel's presplit kernels
    static constexpr int WR = NT < 64 ? 64 : NT;                  // weight rows per (tap, kcore, split)
    static constexpr int B_STAGE = 3 * 64 * WR;                   // three taps of [kcore][split][WR][16 B]
    static constexpr int STAGE_BYTES = 2 * PS_SR * CH * 4;        // [warpgroup][CH / 4][32 rows][4] fp32
};
static_assert(128 * PsCfg<64>::PROD_REGS + 256 * PsCfg<64>::MMA_REGS == 384 * 168, "register split");

template <int R> __device__ __forceinline__ void ps_setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void ps_setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// D[64 x N] (+)= A[64 x 16] * B[16 x N] for the widths of this kernel (N = 152, 80, 72); fragment as in bx_wgmma.cuh: d[4j + e]
// is row 16 (t / 32) + (t % 32) / 4 + 8 (e / 2), column 8 j + 2 (t % 4) + e % 2.
template <int N> __device__ __forceinline__ void wgmma_ps(float *d, uint64_t da, uint64_t db, uint32_t scale_d);

template <> __device__ __forceinline__ void wgmma_ps<152>(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %78, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n152k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75}, %76, %77, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ps<80>(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ps<72>(float *d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %38, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n72k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35}, %36, %37, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35])
        : "l"(da), "l"(db), "r"(scale_d));
}

// Row r (0 .. 151) of sample s, CW consecutive output channels from co0; get8 yields bias + sum of eight of them.  The wrap
// positions x = 20, 21 produce nothing; otherwise the writes of sd_store_rows in bx_conv_sd.cu for the same output.
template <int CW, int OUT_SD, class Get8>
__device__ __forceinline__ void ps_store_row(const ConvPsParams &p, int s, int r, int co0, Get8 get8) {
    const uint32_t y = (uint32_t)r / 22u, x = (uint32_t)r - 22u * y;
    if (x >= 20u) return;
    if constexpr (!OUT_SD) {
        float4 *eo = reinterpret_cast<float4 *>(p.out) + ((size_t)s * (p.Cout >> 2) + (co0 >> 2)) * 140 + (y * 20 + x);
#pragma unroll
        for (int c = 0; c < CW; c += 8) {
            float v[8];
            get8(c, v);
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = p.relu ? fmaxf(v[e], 0.0f) : v[e];
            if (co0 + c < p.Cout) eo[(size_t)(c >> 2) * 140] = make_float4(v[0], v[1], v[2], v[3]);
            if (co0 + c + 4 < p.Cout) eo[(size_t)((c >> 2) + 1) * 140] = make_float4(v[4], v[5], v[6], v[7]);
        }
    } else {
        // value -> padded row R + 23; azimuth 19 / 0 also into the wrap columns x' = 0 / 21 (R + 3 / R + 43)
        const uint32_t R = (uint32_t)s * PS_SROWS + (uint32_t)r;            // host: rows < 2^31
        const size_t rows = (size_t)p.rows_out, pmain = (size_t)R + 23;
        const long long pdup = x == 19u ? (long long)R + 3 : (x == 0u ? (long long)R + 43 : -1);
        uint4 *img = reinterpret_cast<uint4 *>(p.out_sd) + (size_t)((co0 >> 4) * 4 + ((co0 >> 3) & 1)) * rows;
        float omax = 0.0f;
#pragma unroll
        for (int c = 0; c < CW; c += 8) {
            if (co0 + c < p.Cout) {
                float v[8];
                get8(c, v);
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float a = v[2 * e], b = v[2 * e + 1];
                    if (p.relu) { a = fmaxf(a, 0.0f); b = fmaxf(b, 0.0f); }
                    const __half2 hh = __floats2half2_rn(a, b);
                    const float2 hf = __half22float2(hh);
                    const __half2 ll = __floats2half2_rn((a - hf.x) * 2048.0f, (b - hf.y) * 2048.0f);
                    hi[e] = *reinterpret_cast<const uint32_t *>(&hh);
                    lo[e] = *reinterpret_cast<const uint32_t *>(&ll);
                    omax = fmaxf(omax, fmaxf(fabsf(a), fabsf(b)));
                }
                const uint4 vh = make_uint4(hi[0], hi[1], hi[2], hi[3]), vl = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                img[pmain] = vh; img[2 * rows + pmain] = vl;
                if (pdup >= 0) { img[pdup] = vh; img[2 * rows + pdup] = vl; }
            }
            img += (((co0 + c) >> 3) & 1) ? 3 * rows : rows;         // kcore 0 -> 1: next image; kcore 1 -> next chunk's kcore 0
        }
        if (!(omax < 65000.0f) && p.flag) atomicOr(p.flag, 1);
    }
}

// NT = 32 / 64 / 128 (Cout rounded up); OUT_SD = 0: fp32 channel-blocked output, 1: the next layer's presplit image.
template <int NT, int OUT_SD>
__global__ void __launch_bounds__(PsCfg<NT>::THREADS, 1) conv_ps_kernel(const ConvPsParams p) {
    using C = PsCfg<NT>;
    constexpr int SPU = C::SPU, CH = C::CH, NACC = C::NACC, NRUN = C::NRUN;
    constexpr int BAR_AFULL = 0, BAR_AEMPTY = PS_MAXNA, BAR_BFULL = 2 * PS_MAXNA, BAR_BEMPTY = BAR_BFULL + PS_MAXNBS;
    constexpr int NBARS = BAR_BEMPTY + PS_MAXNBS;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) unsigned long long bars[NBARS];
    __shared__ __align__(16) float bias_s[128];

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int NA = p.NA, NBS = p.nbs, nchunks = p.nchunks;
    const bool resident = p.resident != 0;
    const int n_samples = p.d_n ? min(*p.d_n, p.n) : p.n;
    const int n_units = (n_samples + SPU - 1) / SPU;          // CTA b takes units b, b + gridDim.x, ...
    // shared memory: A ring | weight ring | staging buffer of a finished sample
    float *const stage = reinterpret_cast<float *>(smem + (size_t)NA * PS_CHUNK + (size_t)NBS * C::B_STAGE);

    if (tid == 0) {
        for (int s = 0; s < PS_MAXNA; ++s) {
            mbar_init(smem_u32(&bars[BAR_AFULL + s]), 1);
            mbar_init(smem_u32(&bars[BAR_AEMPTY + s]), SPU == 1 ? PS_NC : 4);    // Cout 128: both warpgroups read a slot
        }
        for (int s = 0; s < PS_MAXNBS; ++s) {
            mbar_init(smem_u32(&bars[BAR_BFULL + s]), 1);
            mbar_init(smem_u32(&bars[BAR_BEMPTY + s]), PS_NC);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (threadIdx.x < 128) bias_s[threadIdx.x] = (int)threadIdx.x < p.Cout ? __ldg(p.bias + threadIdx.x) : 0.0f;
    __syncthreads();
    uint32_t a_base = smem_u32(smem);
    uint32_t b_base = a_base + (uint32_t)NA * PS_CHUNK;
    uint32_t bar_base = smem_u32(&bars[0]);
    asm volatile("" : "+r"(a_base), "+r"(b_base), "+r"(bar_base));

    if (warp < PS_NC) {
        // =========================== MMA warpgroups: wgmma, chunk folds, sample stores ===================================
        ps_setmaxnreg_inc<C::MMA_REGS>();
        const int wg = warp >> 2, tl = tid & 127, wq = warp & 3;
        constexpr uint32_t DESC_HI = 128u >> 4;                              // SBO = 128 B (8 rows x 16 B)
        constexpr uint32_t X_LBO = ((uint32_t)PS_KBYTES >> 4) << 16;        // K-adjacent core matrices: one kcore image apart
        constexpr uint32_t X_SPLIT = (2u * PS_KBYTES) >> 4;
        // weight image [kcore][split][WR][16 B]: K-adjacent core matrices one kcore (2 WR rows) apart, taps 64 WR rows apart;
        // lo (Cout >= 64) / Q (Cout <= 32) WR rows after hi / P; Cout 128: warpgroup g's 64 channels start at row 64 g
        constexpr uint32_t W_LBO = ((uint32_t)(2 * C::WR * 16) >> 4) << 16, W_TAP16 = (64u * C::WR) >> 4, W_LO16 = C::WR;
        const uint32_t co_wg = NT == 128 ? 64u * (uint32_t)wg : 0u;          // first output channel of this warpgroup
        const uint32_t x0 = ((a_base + (SPU == 2 ? (uint32_t)wg * PS_CHUNK : 0u)) >> 4) | X_LBO;
        const uint32_t w0 = ((b_base >> 4) + co_wg) | W_LBO;
        const uint32_t nslots = (uint32_t)NA / SPU;
        // Fragment of thread (warp wq, lane): acc[4j + e] is M row 16 wq + lane / 4 + 8 (e / 2), sample row 8 j + 2 (lane % 4)
        // + e % 2.  Cout >= 64: acc = [main 76 | cross 76], M row = channel.  Cout <= 32: M rows r / r + 8 of a 16-row group
        // are main / cross of channel 8 wq + lane / 4.  run[i]: channel co_wg + ch(i), sample row col(i), 8-row group jb(i).
        auto jb = [](int i) { return NT == 32 ? i >> 1 : i >> 2; };
        auto ch = [&](int i) { return NT == 32 ? 8 * wq + (lane >> 2) : 16 * wq + (lane >> 2) + 8 * ((i & 3) >> 1); };
        auto col = [&](int i) { return 8 * jb(i) + 2 * (lane & 3) + (i & 1); };
        uint32_t slot = 0, a_par = 0, q = 0;
        float run[NRUN], acc[NACC];
        // the wgmmas of one N pass of a chunk (27 for Cout >= 64, 18 for Cout <= 32), then one wait and the fold.  Pass h
        // covers sample rows h * NB0 .. h * NB0 + NB - 1: B descriptors h * NB0 rows on, running sums run[h * NB0 / 2 ...]
        auto pass = [&](auto nb, auto h, uint32_t xc, uint32_t q0) {
            constexpr int NB = decltype(nb)::value, H = decltype(h)::value, HALF = C::NACC / 2;
            wgmma_fence();
#pragma unroll
            for (int g = 0; g < 3; ++g) {
                const uint32_t sq = q0 + (uint32_t)g, sb = sq % (uint32_t)NBS;
                if (H == 0) mbar_wait(bar_base + 8u * (BAR_BFULL + sb), resident ? 0u : (sq / (uint32_t)NBS) & 1u);
                const uint32_t wgt = w0 + sb * ((uint32_t)C::B_STAGE >> 4);
#pragma unroll
                for (int tt = 0; tt < 3; ++tt) {
                    const uint32_t xh = xc + (uint32_t)(H * C::NB0 + 22 * g + tt), xl = xh + X_SPLIT;   // one row = 16 B
                    const uint32_t wh = wgt + (uint32_t)tt * W_TAP16, wl = wh + W_LO16;
                    const uint32_t acc_on = (g == 0 && tt == 0) ? 0u : 1u;
                    if constexpr (NT == 128) {
                        wgmma_ps<NB>(acc, gmma_desc(wh, DESC_HI), gmma_desc(xh, DESC_HI), acc_on);
                        wgmma_ps<NB>(acc + HALF, gmma_desc(wh, DESC_HI), gmma_desc(xl, DESC_HI), acc_on);
                        wgmma_ps<NB>(acc + HALF, gmma_desc(wl, DESC_HI), gmma_desc(xh, DESC_HI), 1u);
                    } else if constexpr (NT == 64) {
                        wgmma_ps<NB>(acc, gmma_desc(wh, DESC_HI), gmma_desc(xh, DESC_HI), acc_on);
                        wgmma_ps<NB>(acc + HALF, gmma_desc(wl, DESC_HI), gmma_desc(xh, DESC_HI), acc_on);
                        wgmma_ps<NB>(acc + HALF, gmma_desc(wh, DESC_HI), gmma_desc(xl, DESC_HI), 1u);
                    } else {      // wh = P, wl = Q
                        wgmma_ps<NB>(acc, gmma_desc(wh, DESC_HI), gmma_desc(xh, DESC_HI), acc_on);
                        wgmma_ps<NB>(acc, gmma_desc(wl, DESC_HI), gmma_desc(xl, DESC_HI), 1u);
                    }
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs<NACC>(acc);
            if constexpr (NT == 32) {
#pragma unroll
                for (int i = 0; i < NRUN; ++i) run[i] += fmaf(acc[4 * (i >> 1) + 2 + (i & 1)], 0.00048828125f, acc[4 * (i >> 1) + (i & 1)]);
            } else {
#pragma unroll
                for (int i = 0; i < NB / 2; ++i) run[H * (C::NB0 / 2) + i] += fmaf(acc[HALF + i], 0.00048828125f, acc[i]);
            }
        };
        // one chunk: its passes, then the release of the A slot and (streamed) the three weight stages
        auto chunk = [&](int c) {
            const uint32_t cs = SPU * slot + (SPU == 2 ? (uint32_t)wg : 0u);
            mbar_wait(bar_base + 8u * (BAR_AFULL + cs), a_par);
            const uint32_t xc = x0 + slot * ((uint32_t)(SPU * PS_CHUNK) >> 4);
            const uint32_t q0 = resident ? (uint32_t)c * 3u : q;
            pass(std::integral_constant<int, C::NB0>{}, std::integral_constant<int, 0>{}, xc, q0);
            if constexpr (C::NP == 2) pass(std::integral_constant<int, PS_N - C::NB0>{}, std::integral_constant<int, 1>{}, xc, q0);
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(bar_base + 8u * (BAR_AEMPTY + cs));
                if (!resident)
                    for (int g = 0; g < 3; ++g) mbar_arrive(bar_base + 8u * (BAR_BEMPTY + (q0 + (uint32_t)g) % (uint32_t)NBS));
            }
            if (++slot == nslots) { slot = 0; a_par ^= 1u; }
            if (!resident) q += 3;
        };
        float *const st = stage + (size_t)wg * PS_SR * CH;                   // this warpgroup's [CH / 4][32 rows][4]
        const float4 *st4 = reinterpret_cast<const float4 *>(st);
        for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
#pragma unroll
            for (int i = 0; i < NRUN; ++i) run[i] = bias_s[co_wg + ch(i)];
            for (int c = 0; c < nchunks; ++c) chunk(c);
            const int s = SPU * u + (SPU == 2 ? wg : 0);
            if (s >= n_samples) continue;                                    // the recomputed sample 2u of an odd count
            // the finished sample, 32 rows at a time: fragments -> staging -> a quarter of a row (CH / 4 channels) per thread
#pragma unroll 1
            for (int h = 0; h < (PS_N + PS_SR - 1) / PS_SR; ++h) {
                asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");    // this warpgroup's staging buffer is free
#pragma unroll
                for (int i = 0; i < NRUN; ++i)
                    if ((jb(i) >> 2) == h) st[((ch(i) >> 2) * PS_SR + (col(i) & (PS_SR - 1))) * 4 + (ch(i) & 3)] = run[i];
                asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
                const int row = tl & (PS_SR - 1), cq = (tl >> 5) * (CH / 4);
                if (h * PS_SR + row < PS_N)
                    ps_store_row<CH / 4, OUT_SD>(p, s, h * PS_SR + row, (int)co_wg + cq, [&](int cc, float (&v)[8]) {
                        const float4 u0 = st4[((cq + cc) >> 2) * PS_SR + row], u1 = st4[(((cq + cc) >> 2) + 1) * PS_SR + row];
                        v[0] = u0.x; v[1] = u0.y; v[2] = u0.z; v[3] = u0.w; v[4] = u1.x; v[5] = u1.y; v[6] = u1.z; v[7] = u1.w;
                    });
            }
            if constexpr (OUT_SD) {
                // zero row y' = 0 of sample s + 1 (and of sample 0): 22 rows of this warpgroup's channels
                const size_t rows = (size_t)p.rows_out;
                const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
                for (int i = tl; i < 22 * (CH / 8); i += 128) {
                    const int b = i / 22, xr = i - 22 * b, co = (int)co_wg + 8 * b;
                    if (co >= p.Cout) continue;
                    uint4 *img = reinterpret_cast<uint4 *>(p.out_sd) + (size_t)((co >> 4) * 4 + ((co >> 3) & 1)) * rows;
                    const size_t r1 = (size_t)(s + 1) * PS_SROWS + (size_t)xr;
                    img[r1] = z; img[2 * rows + r1] = z;
                    if (s == 0) { img[xr] = z; img[2 * rows + xr] = z; }
                }
            }
        }
    } else {
        ps_setmaxnreg_dec<C::PROD_REGS>();
        if (warp == PS_NC) {
            // =========================== A producer: a sample's chunk = four bulk copies of 198 rows ======================
            // Cout <= 64: chunk c of the unit's samples 2u + g goes to slot 2 s + g (sample 2u again when 2u + 1 does not exist).
            if (lane == 0) {
                const uint32_t nslots = (uint32_t)NA / SPU;
                uint32_t slot = 0, par = 0, round = 0;
                for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
                    for (int c = 0; c < nchunks; ++c) {
#pragma unroll
                        for (uint32_t g = 0; g < (uint32_t)SPU; ++g) {
                            const uint32_t cs = slot * SPU + g;
                            const int s = (int)(SPU * (uint32_t)u + g) < n_samples ? (int)(SPU * (uint32_t)u + g) : (int)(SPU * (uint32_t)u);
                            if (round) mbar_wait(bar_base + 8u * (BAR_AEMPTY + cs), par ^ 1u);
                            mbar_arrive_expect_tx(bar_base + 8u * (BAR_AFULL + cs), 4u * (uint32_t)PS_KBYTES);
                            const unsigned char *src = reinterpret_cast<const unsigned char *>(p.in_sd) + ((size_t)(c * 4) * p.rows_in + (size_t)s * PS_SROWS) * 16;
#pragma unroll
                            for (int im = 0; im < 4; ++im)
                                bulk_g2s(a_base + cs * (uint32_t)PS_CHUNK + (uint32_t)im * PS_KBYTES, src + (size_t)im * p.rows_in * 16, (uint32_t)PS_KBYTES,
                                         bar_base + 8u * (BAR_AFULL + cs));
                        }
                        if (++slot == nslots) { slot = 0; par ^= 1u; round = 1; }
                    }
                }
            }
            __syncwarp();
        } else if (warp == PS_WGT_WARP) {
            // =========================== weight producer ========================================================
            if (lane == 0) {
                const int n_st = nchunks * 3;
                uint32_t q = 0;
                for (int u = blockIdx.x; u < n_units; u += gridDim.x) {
                    for (int s = 0; s < n_st; ++s, ++q) {
                        const uint32_t sb = q % (uint32_t)NBS, use = q / (uint32_t)NBS;
                        if (use > 0) mbar_wait(bar_base + 8u * (BAR_BEMPTY + sb), (use - 1) & 1u);
                        mbar_arrive_expect_tx(bar_base + 8u * (BAR_BFULL + sb), (uint32_t)C::B_STAGE);
                        bulk_g2s(b_base + sb * (uint32_t)C::B_STAGE, reinterpret_cast<const unsigned char *>(p.w) + (size_t)s * C::B_STAGE,
                                 (uint32_t)C::B_STAGE, bar_base + 8u * (BAR_BFULL + sb));
                    }
                    if (resident) break;                                // resident weights: loaded for the first unit only
                }
            }
            __syncwarp();
        }
    }
}

template <int NT, int OUT_SD>
int launch_ps(ConvPsParams p, cudaStream_t st) {
    using C = PsCfg<NT>;
    // the whole weight image resident in shared memory when it leaves room for two A chunks per warpgroup stream, else a
    // ring of six stages (two chunks) or as many as leave room for four A chunks
    const int budget = PS_SMEM - C::STAGE_BYTES, n_st = p.nchunks * 3;
    p.resident = n_st <= PS_MAXNBS && budget - n_st * C::B_STAGE >= 2 * C::SPU * PS_CHUNK;
    p.nbs = p.resident ? n_st : 6;
    while (!p.resident && p.nbs > 3 && budget - p.nbs * C::B_STAGE < 4 * PS_CHUNK) --p.nbs;
    int na = (budget - p.nbs * C::B_STAGE) / PS_CHUNK;
    if (na > 2 * C::SPU * p.nchunks) na = 2 * C::SPU * p.nchunks;
    if (na > PS_MAXNA) na = PS_MAXNA;
    na -= na % C::SPU;
    BX_REQUIRE(na >= 2 * C::SPU, "bx_conv_layer_ps: no room for the activation ring");
    p.NA = na;
    const int smem = na * PS_CHUNK + p.nbs * C::B_STAGE + C::STAGE_BYTES;
    static BxPerDevice attr = {};
    if (bx_needs_attr(attr, (size_t)smem))
        BX_CUDA(cudaFuncSetAttribute(conv_ps_kernel<NT, OUT_SD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int sms = bx_device_sm_count();
    if (sms <= 0) sms = 132;
    const int units = (p.n + C::SPU - 1) / C::SPU;
    const int grid = units < sms ? units : sms;
    conv_ps_kernel<NT, OUT_SD><<<grid, C::THREADS, smem, st>>>(p);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

template <int NT>
int dispatch_ps(const ConvPsParams &p, int out_sd, cudaStream_t st) {
    return out_sd ? launch_ps<NT, 1>(p, st) : launch_ps<NT, 0>(p, st);
}

}  // namespace

BX_API int bx_conv_layer_ps(int geom, const void *in, int in_presplit, const void *w_sd, const float *bias, void *out, int out_presplit,
                            int n, const int32_t *d_n, int Cin, int Cout, int D, int W, int relu, int32_t *d_flag, void *stream) {
    (void)D; (void)W;
    BX_REQUIRE(in && w_sd && bias && out, "bx_conv_layer_ps: null pointer");
    BX_REQUIRE(geom == BX_GEOM_CYL3D || geom == BX_GEOM_CYL2D, "bx_conv_layer_ps: geometry must be CYL3D or CYL2D (the descriptor stack)");
    BX_REQUIRE(in_presplit, "bx_conv_layer_ps: the input must be a presplit image (fp32 input: bx_conv_layer_sd)");
    BX_REQUIRE(n >= 0 && Cin >= 16 && Cin % 16 == 0 && Cout >= 4 && Cout % 4 == 0 && Cout <= 128, "bx_conv_layer_ps: bad channels Cin=%d Cout=%d", Cin, Cout);
    BX_REQUIRE(geom != BX_GEOM_CYL3D || Cin == 16, "bx_conv_layer_ps: CYL3D expects 16 input channels x 3 radial slices");
    BX_REQUIRE(!out_presplit || Cout % 16 == 0, "bx_conv_layer_ps: presplit output needs Cout %% 16 == 0");
    BX_REQUIRE(((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(bias) | reinterpret_cast<uintptr_t>(w_sd)) & 15) == 0,
               "bx_conv_layer_ps: activations, weights and bias must be 16-byte aligned");
    if (n == 0) return BX_OK;
    BX_REQUIRE((long long)n * PS_SROWS + 4 * 128 < 0x7fffffffLL, "bx_conv_layer_ps: too many samples (raster rows must stay below 2^31)");
    ConvPsParams p = {};
    p.in_sd = reinterpret_cast<const __half *>(in);
    p.w = reinterpret_cast<const __half *>(w_sd); p.bias = bias; p.flag = d_flag; p.d_n = d_n;
    p.out = out_presplit ? nullptr : reinterpret_cast<float *>(out);
    p.out_sd = out_presplit ? reinterpret_cast<__half *>(out) : nullptr;
    p.n = n; p.Cout = Cout; p.relu = relu;
    p.nchunks = geom == BX_GEOM_CYL3D ? 3 : Cin / 16;
    // same image geometry as bx_conv_layer_sd; a sample's chunk reaches row 176 (n - 1) + 197 < bx_conv_sd_rows(n, 176)
    p.rows_in = bx_conv_sd_rows(n, PS_SROWS);
    p.rows_out = p.rows_in;
    cudaStream_t st = bx_stream(stream);
    if (Cout > 64) return dispatch_ps<128>(p, out_presplit, st);
    if (Cout > 32) return dispatch_ps<64>(p, out_presplit, st);
    return dispatch_ps<32>(p, out_presplit, st);
}
