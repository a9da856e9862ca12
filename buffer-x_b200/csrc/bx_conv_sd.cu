// bx_conv_sd.cu -- the cylindrical descriptor convolutions as a SHIFTED-DESCRIPTOR implicit GEMM on the Hopper tensor cores (wgmma).
//
// For the eight layers of Cylindrical_Net (reference models/patchnet.py:16-84 with the padding of utils/common.py:265-310) an
// activation is written to shared memory ONCE per tile and the nine 3x3 taps are nine VIEWS of the same bytes:
//
//   row space   every sample is a padded (8 x 22) raster: padded row y' = 0 is a zero row (elevation padding, shared with
//               the previous sample's bottom), y' = 1..7 are the elevations; padded column x' = 0 / 21 are the circular
//               copies of azimuth 19 / 0, x' = 1..20 the azimuths.  GEMM row R = 176 s + 22 y + x is output (s, y, x); the
//               input it needs for tap (dy, dx) sits at padded row R + 22 dy + dx -- ONE constant shift per tap for all
//               128 rows of a tile.  Rows with x >= 20 or y == 7 are computed and dropped (140 of 176 rows are real).
//   A operand   a tile's 176 (= 128 + 48 halo) padded rows of one 16-channel chunk live in shared memory as the canonical
//               K-major no-swizzle image [split(hi,lo)][kcore(2)][row][8 x fp16 = 16 B]: rows are linear with a 16-byte
//               stride (SBO = 128 B), so the descriptor of tap (dy, dx) is the chunk's base descriptor with its start
//               address advanced by (22 dy + dx) * 16 B.  The 3x3x3 first layer is the same thing with its three radial
//               slices as three chunks of 16 channels.
//   precision   fp32-grade results (descriptor parity 1e-4 rel) from fp16 tensor-core operands: x = hi + lo * 2^-11 with
//               hi = fp16(x), lo = fp16((x - hi) * 2^11) (22 mantissa bits, the same as the 3xTF32 split, at twice the
//               tensor rate and half the operand bytes):  a*b ~= ah*bh + (al*bh + ah*bl) * 2^-11.  Per 16-channel chunk
//               (K = 144) the products go to a fresh accumulator [main | cross]; the finished chunk's main + cross * 2^-11 is
//               added with round-to-nearest into fp32 running sums that start from the bias, so no accumulation chain is
//               longer than one chunk.  main and cross are disjoint register blocks, each written only by whole wgmmas: a
//               wgmma that accumulates into a sub-range of another in-flight wgmma's registers makes ptxas wait for each
//               wgmma before issuing the next.
//               |x| >= 65504 cannot be represented: the loader raises *flag and the host re-runs the layer on the TF32 kernel.
//
// Two mainloops, both with the shifted activation views as one operand and the weights as the other:
//   rows-as-M         (Cout 128, and every fp32-input kernel)  M = 64 tile rows per warpgroup, N = Cout.  A tap is three
//                     m64nCout wgmmas: ah * bh into main, ah * bl and al * bh into cross.  Cout 128 takes a chunk in one pass
//                     (128 accumulators + 64 running sums per thread, see the register split below), except with fp32 input,
//                     which does two 64-column passes.
//   channels-as-M     (presplit input, Cout <= 64)  M = 64 output channels, N = a whole 128-row tile per warpgroup, so every
//                     wgmma is m64n128k16 whatever Cout is (a narrow N re-reads the activation tile once per few MACs).  The
//                     weight image is the A operand and the activation view the B operand; both have the same K-major
//                     no-swizzle core-matrix layout as before, so a tap is still "base descriptor + (W dy + dx) rows".
//                     Cout 64: three wgmmas per tap, Wh * ah into main, then Wl * ah and Wh * al into cross.  Cout <= 32: the
//                     weight image holds, per (chunk, tap, kcore), two 64-row blocks P and Q; in each 16-row group w, P rows
//                     0-7 / 8-15 are hi / lo of channels 8w .. 8w + 7 and Q rows 0-7 / 8-15 are zero / hi.  P * ah then Q * al
//                     into ONE accumulator leaves main (Wh * ah + exact zeros) in fragment rows r and cross (Wl * ah, then
//                     Wh * al) in rows r + 8 of the same thread: two wgmmas per tap and a thread-local fold.  The cross
//                     products keep the order of the rows-as-M form (ah * bl first), so every element rounds as before.
//
// Persistent warp-specialised CTA, one per SM, of three warpgroups:
//   2 MMA warpgroups  rows-as-M: warpgroup g owns tile rows 64 g .. 64 g + 63 of the CTA's tile.  channels-as-M: the CTA works
//                     on a unit of two tiles 2u, 2u + 1 and warpgroup g owns tile 2u + g (for an odd tile count the last unit's
//                     second warpgroup recomputes tile 2u and stores nothing).  Per (chunk, tap) the wgmmas read the shifted
//                     activation view and the weights straight from shared memory; after a chunk the accumulators are folded
//                     into the running sums and the A slot / weight stages are released.  Both warpgroups walk the chunks in
//                     step, so a streamed weight stage is released when both have used it.  A finished tile goes through a
//                     shared-memory staging buffer (64 columns, or 64 rows of every channel, at a time) so that each thread
//                     then stores (half) a row: ReLU, fp16 hi/lo split and the next layer's wrap columns and zero rows, or
//                     fp32 channel-blocked values.
//   producer warpgroup, warps 0-2 = A producer, warp 3 = weight thread:
//   A producer        presplit input: one thread, a chunk = four 2816-byte bulk copies of the previous layer's presplit image
//                     (ring of NA chunk slots; channels-as-M: slots 2s and 2s + 1 hold the same chunk of the unit's two
//                     tiles).  fp32 input: 3 loader warps convert channel-blocked activations to fp16 hi/lo.
//   weight thread     the host-arranged weight image [chunk][tap][kcore][split][n][8 x fp16] (Cout <= 32: [chunk][tap][kcore]
//                     [P | Q][64][8 x fp16]) in stages of three taps with cp.async.bulk + mbarrier transaction counts; loaded
//                     ONCE and kept resident when the whole image fits next to three A chunks (four for channels-as-M), else
//                     streamed through a ring.
#include <cuda_fp16.h>

#include "bx_common.cuh"
#include "bx_wgmma.cuh"

namespace {

constexpr int SD_BM = 128;                       // GEMM rows per tile
constexpr int SD_AROWS = 176;                    // tile rows + halo (2*22 + 2 = 46 -> 48)
constexpr int SD_SROWS = 176;                    // padded rows per sample (8 x 22)
constexpr int SD_KBYTES = SD_AROWS * 16;         // one (split, kcore) image of a chunk: [row][8 x fp16]
constexpr int SD_CHUNK = 4 * SD_KBYTES;          // [split(hi,lo)][kcore(2)]
constexpr int SD_NL = 3;                         // loader warps (fp32 input)
constexpr int SD_NC = 8;                         // MMA warps: two warpgroups of 64 tile rows
constexpr int SD_WGT_WARP = SD_NC + 3;           // weight thread: last warp of the producer warpgroup
constexpr int SD_MAXNA = 12, SD_MAXNBS = 24;     // A chunk slots; weight stages (resident: every stage of up to 8 chunks)
constexpr int SD_TRING = 32;                     // published tile indices of dynamic scheduling
constexpr int SD_SMEM = 227 * 1024 - 2048;       // dynamic shared memory of one CTA (the rest: barriers, bias)

struct ConvSdParams {
    const float *in;
    const __half *w;
    const float *bias;
    float *out;
    int *flag;
    int n, Cout, nchunks, is3d, S_in, G_in, relu, n_tiles, NA;
    const int *d_n;            // optional device-side sample count (<= n): the match lists of the cost-volume stack
    const float *fa, *fb;      // COSTAB loader: the factor maps A [n,8,3*20,4], B [n,8,3*18,4] of bx_costvol_ab (else NULL)
    int cyl, rs, W, OD, OW, S_out, rs_out;   // raster geometry: rows per sample, row stride, valid output extent, output rasters
    const __half *in_sd;       // IN_SD: presplit padded input  [nchunks][split,kcore (4)][rows_in][8 x fp16]
    __half *out_sd;            // OUT_SD: presplit padded output [Cout/16][4][rows_out][8 x fp16] = the next layer's in_sd
    long long rows_in, rows_out;
    int nbs;                   // weight ring length in stages of three taps (resident: == nchunks * 3, every stage is loaded once)
    int resident;              // the whole weight image stays in shared memory: no re-streaming per tile
    int *tile_ctr;             // dynamic tile scheduling (presplit-input kernels): [0] next tile, [1] CTAs that have finished; NULL = static stride
};

template <int NT, int IN_SD> struct SdCfg {
    // channels-as-M mainloop (see the header): presplit input with Cout <= 64.  The fp32-input kernels keep rows-as-M: their
    // MMA threads have 184 registers, too few for 128 accumulators + 64 running sums.
    static constexpr bool CM = IN_SD && NT < 128;
    static constexpr int TPU = CM ? 2 : 1;                        // tiles per unit of work of a CTA
    // rows-as-M accumulator block: output columns per pass over a chunk.  All of them, except for Cout 128 with fp32 input,
    // whose loader warps keep more registers than the 128 accumulators + 64 running sums of a single pass would leave room for.
    static constexpr int NB = (NT == 128 && !IN_SD) ? 64 : NT;
    static constexpr int NH = NT / NB;                            // passes per chunk
    static constexpr int SB = NT < 64 ? NT : 64;                  // output columns per staging round of a finished tile
    static constexpr int THREADS = (SD_NC + 4) * 32;              // two MMA warpgroups + one producer warpgroup
    // per-thread registers after setmaxnreg: 128 * PROD_REGS + 256 * MMA_REGS = 384 * 168, the CTA's allocation at launch
    // (ptxas reports 168 for every instantiation; a split that asked for more would leave setmaxnreg.inc waiting forever)
    static constexpr int PROD_REGS = IN_SD ? 56 : 136, MMA_REGS = IN_SD ? 224 : 184;
    static constexpr int WR = NT < 64 ? 64 : NT;                  // weight rows per (tap, kcore, split): Cout <= 32 is [P | Q] x 64
    static constexpr int B_STAGE = 3 * 64 * WR;                   // three taps of [kcore][split][WR][16 B]
    // fp32 staging of a finished tile: rows-as-M, one column block of the CTA's tile [SB / 4][128 rows][4]; channels-as-M (SB
    // = NT), 64 rows of every channel of each warpgroup's tile, [warpgroup][NT / 4][64 rows][4] -- the same size
    static constexpr int STAGE_BYTES = SD_BM * SB * 4;
};
static_assert(128 * SdCfg<64, 1>::PROD_REGS + 256 * SdCfg<64, 1>::MMA_REGS == 384 * 168, "register split of the presplit kernels");
static_assert(128 * SdCfg<64, 0>::PROD_REGS + 256 * SdCfg<64, 0>::MMA_REGS == 384 * 168, "register split of the fp32-input kernels");

// Moves registers between warpgroups (all threads of a warpgroup execute it with the same count, a multiple of 8): the
// producer warpgroup gives back what the MMA warpgroups take.  .inc waits until the registers are free.
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// One thread's share of a finished tile: GEMM row R = t * 128 + row, CW consecutive output channels starting at co0; get8
// yields bias + sum of eight of them.  Here: ReLU, then either fp32 channel-blocked stores of the valid rows or the presplit
// images of the next layer (value, wrap-column copies, zero rows).  Rows that produce nothing skip the arithmetic, the index
// arithmetic is 32-bit, the image pointers advance by additions.
template <int CW, int OUT_SD, class Get8>
__device__ __forceinline__ void sd_store_rows(const ConvSdParams &p, int t, int row, int co0, int n_samples, Get8 get8) {
    const uint32_t R = (uint32_t)t * SD_BM + (uint32_t)row;            // host: rows < 2^31
    const uint32_t s = R / (uint32_t)p.rs, q = R - s * (uint32_t)p.rs;
    const uint32_t y = q / (uint32_t)p.W, x = q - y * (uint32_t)p.W;
    const bool live = (int)s < n_samples;
    const bool valid = live && (int)y < p.OD && (int)x < p.OW;
    if constexpr (!OUT_SD) {
        if (!valid) return;
        const int S_out = p.S_out;
        float4 *eo = reinterpret_cast<float4 *>(p.out) + ((size_t)s * (p.Cout >> 2) + (co0 >> 2)) * S_out + (y * p.OW + x);
#pragma unroll
        for (int c = 0; c < CW; c += 8) {
            float r[8];
            get8(c, r);
#pragma unroll
            for (int e = 0; e < 8; ++e) r[e] = p.relu ? fmaxf(r[e], 0.0f) : r[e];
            if (co0 + c < p.Cout) eo[(size_t)(c >> 2) * S_out] = make_float4(r[0], r[1], r[2], r[3]);
            if (co0 + c + 4 < p.Cout) eo[(size_t)((c >> 2) + 1) * S_out] = make_float4(r[4], r[5], r[6], r[7]);
        }
    } else {
        // this row's value goes to padded row R + 23 (= (y + 1) * 22 + (x + 1)); azimuth 19 / 0 are duplicated into the wrap
        // columns x' = 0 / 21; the rows that land on a zero row write zeros; everything else is dropped.
        // (valid-convolution rasters of the cost-volume stack: compact output raster, no padding rows / columns)
        const bool wz = p.cyl && live && ((y == 7 && x <= 20) || (y == 6 && x == 21));       // zero row of sample s + 1
        const bool z0 = p.cyl && R < 22;                                                       // zero row of sample 0
        if (!valid && !wz && !z0) return;
        const size_t rows = (size_t)p.rows_out;
        const size_t pmain = p.cyl ? (size_t)R + 23 : (size_t)s * p.rs_out + y * p.OW + x;
        const long long pdup = !p.cyl ? -1 : (x == 19 ? (long long)R + 3 : (x == 0 ? (long long)R + 43 : -1));
        // image (chunk = co / 16, kcore = (co / 8) & 1): [chunk][split][kcore][row][8]
        uint4 *img = reinterpret_cast<uint4 *>(p.out_sd) + (size_t)((co0 >> 4) * 4 + ((co0 >> 3) & 1)) * rows;
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
        float omax = 0.0f;
#pragma unroll
        for (int c = 0; c < CW; c += 8) {
            if (co0 + c < p.Cout) {
                if (valid) {
                    float r[8];
                    get8(c, r);
                    uint32_t hi[4], lo[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float a = r[2 * e], b = r[2 * e + 1];
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
                } else if (wz) { img[pmain] = z; img[2 * rows + pmain] = z; }
                if (z0) { img[R] = z; img[2 * rows + R] = z; }
            }
            img += (((co0 + c) >> 3) & 1) ? 3 * rows : rows;         // kcore 0 -> 1: next image; kcore 1 -> next chunk's kcore 0
        }
        if (!(omax < 65000.0f) && p.flag) atomicOr(p.flag, 1);
    }
}

// IN_SD = 0: fp32 channel-blocked input converted by the loader warps; 1: presplit padded fp16 images fetched with bulk copies.
// OUT_SD = 0: fp32 channel-blocked output; 1: presplit padded fp16 images (zero rows and wrap columns written here).
template <int NT, int IN_SD, int OUT_SD>
// Registers: 12 warps = 3 per sub-partition of 16 K registers, so every thread starts at 168 (the bound __launch_bounds__
// gives ptxas).  The producer warpgroup then drops to PROD_REGS (56 for the bulk-copy and weight threads, 136 for the fp32
// loaders) and the MMA warpgroups rise to MMA_REGS (224 / 184): room for a whole Cout 128 chunk's accumulators
// [main 64 | cross 64] next to the 64 running sums, and enough for ptxas to keep the wgmma chain of a chunk in flight.
__global__ void __launch_bounds__(SdCfg<NT, IN_SD>::THREADS, 1) conv_sd_kernel(const ConvSdParams p) {
    using C = SdCfg<NT, IN_SD>;
    constexpr int NB = C::NB, NH = C::NH, SB = C::SB, WGT_WARP = SD_WGT_WARP;
    constexpr int BAR_AFULL = 0, BAR_AEMPTY = SD_MAXNA, BAR_BFULL = 2 * SD_MAXNA, BAR_BEMPTY = BAR_BFULL + SD_MAXNBS;
    constexpr int BAR_TILE = BAR_BEMPTY + SD_MAXNBS, NBARS = BAR_TILE + SD_TRING;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) unsigned long long bars[NBARS];
    __shared__ int tile_ring[SD_TRING];
    __shared__ __align__(16) float bias_s[128];        // the running sums of a tile start from the bias

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);       // warp-uniform role index (keeps the wgmma issue convergent)
    const int NA = p.NA, NBS = p.nbs, nchunks = p.nchunks;
    const bool resident = p.resident != 0;
    const int n_samples = p.d_n ? min(*p.d_n, p.n) : p.n;
    const int n_tiles = (int)(((long long)n_samples * p.rs + SD_BM - 1) / SD_BM);   // <= the host's bound the grid was sized for
    const int n_units = (n_tiles + C::TPU - 1) / C::TPU;
    // shared memory: A ring | weight ring | staging buffer of a finished tile (C::STAGE_BYTES)
    float *const stage = reinterpret_cast<float *>(smem + (size_t)NA * SD_CHUNK + (size_t)NBS * C::B_STAGE);

    if (tid == 0) {
        for (int s = 0; s < SD_MAXNA; ++s) {
            mbar_init(smem_u32(&bars[BAR_AFULL + s]), IN_SD ? 1 : SD_NL);
            mbar_init(smem_u32(&bars[BAR_AEMPTY + s]), C::CM ? 4 : SD_NC);     // channels-as-M: a slot is one warpgroup's
        }
        for (int s = 0; s < SD_MAXNBS; ++s) {
            mbar_init(smem_u32(&bars[BAR_BFULL + s]), 1);
            mbar_init(smem_u32(&bars[BAR_BEMPTY + s]), SD_NC);
        }
        for (int s = 0; s < SD_TRING; ++s) mbar_init(smem_u32(&bars[BAR_TILE + s]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (threadIdx.x < 128) bias_s[threadIdx.x] = (int)threadIdx.x < p.Cout ? __ldg(p.bias + threadIdx.x) : 0.0f;
    __syncthreads();
    uint32_t a_base = smem_u32(smem);
    uint32_t b_base = a_base + (uint32_t)NA * SD_CHUNK;
    uint32_t bar_base = smem_u32(&bars[0]);
    asm volatile("" : "+r"(a_base), "+r"(b_base), "+r"(bar_base));

    // Unit sequence of this CTA (a unit is C::TPU tiles).  Static: blockIdx.x, + gridDim.x, ...  Dynamic (presplit input,
    // p.tile_ctr): the A producer draws the next unit from a global counter and publishes it in a shared-memory ring; every
    // other role reads the k-th entry (-1 = no more units).  With several pairs in flight a convolution often starts with some
    // SMs still held by another stream's kernels; with the static stride the CTAs that start late still own their share of
    // the tiles and the whole launch waits for them.
    const bool dyn = IN_SD && p.tile_ctr != nullptr;
    auto tile_of = [&](uint32_t k) -> int {
        if (!dyn) { const long long t = (long long)blockIdx.x + (long long)k * gridDim.x; return t < n_units ? (int)t : -1; }
        mbar_wait(bar_base + 8u * (BAR_TILE + (k & (SD_TRING - 1))), (k / SD_TRING) & 1u);
        return tile_ring[k & (SD_TRING - 1)];
    };

    // Each role branch starts with its warpgroup's setmaxnreg (one instruction for all threads of a warpgroup): the MMA
    // warpgroups take the registers the producer warpgroup gives up.
    if (warp < SD_NC) {
        // =========================== MMA warpgroups: wgmma, chunk folds, tile stores =====================================
        setmaxnreg_inc<C::MMA_REGS>();
        const int wg = warp >> 2, tl = tid & 127;
        constexpr uint32_t DESC_HI = 128u >> 4;                          // SBO = 128 B (8 rows x 16 B)
        constexpr uint32_t A_LBO = ((uint32_t)SD_KBYTES >> 4) << 16;    // K-adjacent core matrices: one kcore image apart
        constexpr uint32_t A_SPLIT = (2u * SD_KBYTES) >> 4;
        // weight image [kcore][split][WR][16 B]: K-adjacent core matrices one kcore (2 WR rows) apart, taps 64 WR rows apart
        constexpr uint32_t B_LBO = ((uint32_t)(2 * C::WR * 16) >> 4) << 16, B_TAP16 = (64u * C::WR) >> 4;
        const uint32_t Wrow = (uint32_t)p.W;                             // tap (g, tt) reads rows R + g * W + tt
        uint32_t slot = 0, a_par = 0, q = 0, k = 0;
        if constexpr (C::CM) {
            // ---- channels-as-M: warpgroup wg owns tile 2u + wg; weights = A operand (64 channel rows), activations = B (128 rows)
            // Fragment of thread (warp w = warp & 3, lane): acc[4j + e] is M row 16 w + lane / 4 + 8 (e / 2), tile row
            // 8 j + 2 (lane % 4) + e % 2.  Cout 64: acc = [main 64 | cross 64], M row = channel.  Cout <= 32: M rows r / r + 8
            // of a 16-row group are main / cross of channel 8 w + lane / 4.  run[i]: channel ch(i), tile row col(i).
            constexpr int NACC = NT == 64 ? 128 : 64;
            constexpr uint32_t W_LO16 = (64u * 16u) >> 4;                // lo (Cout 64) / Q (Cout <= 32): 64 rows after hi / P
            const int wq = warp & 3;
            auto ch = [&](int i) { return NT == 64 ? 16 * wq + (lane >> 2) + 8 * ((i & 3) >> 1) : 8 * wq + (lane >> 2); };
            auto col = [&](int i) { return (NT == 64 ? 8 * (i >> 2) : 8 * (i >> 1)) + 2 * (lane & 3) + (i & 1); };
            auto mi = [](int i) { return NT == 64 ? i : 4 * (i >> 1) + (i & 1); };              // main accumulator of run[i]
            auto xi = [](int i) { return NT == 64 ? 64 + i : 4 * (i >> 1) + 2 + (i & 1); };     // cross accumulator of run[i]
            const uint32_t x0 = ((a_base + (uint32_t)wg * SD_CHUNK) >> 4) | A_LBO;   // slot 2 s + wg: this warpgroup's tile
            const uint32_t w0 = (b_base >> 4) | B_LBO;
            const uint32_t nslots = (uint32_t)NA / 2u;
            float run[NT], acc[NACC];
            // one chunk of this warpgroup's tile: 27 (Cout 64) or 18 (Cout <= 32) wgmmas, one wait, the fold, the release
            auto chunk = [&](int c) {
                const uint32_t cs = 2u * slot + (uint32_t)wg;
                mbar_wait(bar_base + 8u * (BAR_AFULL + cs), a_par);
                const uint32_t xc = x0 + slot * ((2u * SD_CHUNK) >> 4);
                const uint32_t q0 = resident ? (uint32_t)c * 3u : q;    // first weight stage of this chunk
                wgmma_fence();
#pragma unroll
                for (int g = 0; g < 3; ++g) {
                    const uint32_t sq = q0 + (uint32_t)g, sb = sq % (uint32_t)NBS;
                    mbar_wait(bar_base + 8u * (BAR_BFULL + sb), resident ? 0u : (sq / (uint32_t)NBS) & 1u);
                    const uint32_t wgt = w0 + sb * ((uint32_t)C::B_STAGE >> 4);
#pragma unroll
                    for (int tt = 0; tt < 3; ++tt) {
                        const uint32_t xh = xc + (uint32_t)g * Wrow + (uint32_t)tt, xl = xh + A_SPLIT;   // one row = 16 B
                        const uint32_t wh = wgt + (uint32_t)tt * B_TAP16, wl = wh + W_LO16;
                        const uint32_t acc_on = (g == 0 && tt == 0) ? 0u : 1u;
                        if constexpr (NT == 64) {
                            wgmma_f16<128>(acc, gmma_desc(wh, DESC_HI), gmma_desc(xh, DESC_HI), acc_on);
                            wgmma_f16<128>(acc + 64, gmma_desc(wl, DESC_HI), gmma_desc(xh, DESC_HI), acc_on);
                            wgmma_f16<128>(acc + 64, gmma_desc(wh, DESC_HI), gmma_desc(xl, DESC_HI), 1u);
                        } else {      // wh = P, wl = Q
                            wgmma_f16<128>(acc, gmma_desc(wh, DESC_HI), gmma_desc(xh, DESC_HI), acc_on);
                            wgmma_f16<128>(acc, gmma_desc(wl, DESC_HI), gmma_desc(xl, DESC_HI), 1u);
                        }
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs<NACC>(acc);
#pragma unroll
                for (int i = 0; i < NT; ++i) run[i] += fmaf(acc[xi(i)], 0.00048828125f, acc[mi(i)]);
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(bar_base + 8u * (BAR_AEMPTY + cs));
                    if (!resident)
                        for (int g = 0; g < 3; ++g) mbar_arrive(bar_base + 8u * (BAR_BEMPTY + (q0 + (uint32_t)g) % (uint32_t)NBS));
                }
                if (++slot == nslots) { slot = 0; a_par ^= 1u; }
                if (!resident) q += 3;
            };
            float *const st = stage + (size_t)wg * 64 * NT;                  // this warpgroup's [NT / 4][64 rows][4]
            const float4 *st4 = reinterpret_cast<const float4 *>(st);
            for (int u = tile_of(0); u >= 0; u = tile_of(++k)) {
#pragma unroll
                for (int i = 0; i < NT; ++i) run[i] = bias_s[ch(i)];
                // Two chunks per iteration, the second one guarded: the code of a chunk appears twice, so a Cout <= 32 kernel
                // shows a chain of 36 HGMMAs (2 waits) in its SASS, which tests/test_conv_sd_ptxas_cpu.py checks for.
                for (int c = 0; c < nchunks; c += 2) {
                    chunk(c);
                    if (c + 1 < nchunks) chunk(c + 1);
                }
                const int t = 2 * u + wg;
                if (t >= n_tiles) continue;                                   // the recomputed tile 2u of an odd tile count
                // the finished tile, 64 rows at a time: fragments -> staging -> half a row (NT / 2 channels) per thread
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");    // this warpgroup's staging buffer is free
#pragma unroll
                    for (int i = 0; i < NT; ++i)
                        if ((col(i) >> 6) == h) st[((ch(i) >> 2) * 64 + (col(i) & 63)) * 4 + (ch(i) & 3)] = run[i];
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
                    const int row = tl & 63, cs = (tl >> 6) * (NT / 2);
                    sd_store_rows<NT / 2, OUT_SD>(p, t, h * 64 + row, cs, n_samples, [&](int cc, float (&r)[8]) {
                        const float4 u0 = st4[((cs + cc) >> 2) * 64 + row], u1 = st4[(((cs + cc) >> 2) + 1) * 64 + row];
                        r[0] = u0.x; r[1] = u0.y; r[2] = u0.z; r[3] = u0.w; r[4] = u1.x; r[5] = u1.y; r[6] = u1.z; r[7] = u1.w;
                    });
                }
            }
        } else {
            // ---- rows-as-M: warpgroup wg owns rows 64 wg .. 64 wg + 63 of tile t; activations = A operand, weights = B (N = Cout)
            const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);         // fragment rows r0 and r0 + 8 of the tile
            const int cq = 2 * (lane & 3);                                   // fragment column within an 8-column group
            // Cout <= 32 (fp32 input): hi / lo of the B operand are rows 0-7 / 8-15 of each 16-row group of P, so its 8-row core
            // matrices are 256 B apart and lo starts 128 B after hi
            constexpr uint32_t B_DESC_HI = (NT < 64 ? 256u : 128u) >> 4, B_LO16 = (NT < 64 ? 128u : (uint32_t)NT * 16u) >> 4;
            const uint32_t a0 = ((a_base + (uint32_t)wg * 64u * 16u) >> 4) | A_LBO;   // this warpgroup's 64 rows
            const uint32_t b0 = (b_base >> 4) | B_LBO;
            float run[NT / 2], acc[NB];      // acc = [main NB / 2 | cross NB / 2]: disjoint blocks, each written by whole wgmmas
            for (int t = tile_of(0); t >= 0; t = tile_of(++k)) {
#pragma unroll
                for (int i = 0; i < NT / 2; ++i) run[i] = bias_s[(i / (NB / 2)) * NB + 8 * ((i % (NB / 2)) >> 2) + cq + (i & 1)];
                for (int c = 0; c < nchunks; ++c) {
                    mbar_wait(bar_base + 8u * (BAR_AFULL + slot), a_par);
                    const uint32_t ac = a0 + slot * ((uint32_t)SD_CHUNK >> 4);
                    const uint32_t q0 = resident ? (uint32_t)c * 3u : q;    // first weight stage of this chunk
#pragma unroll
                    for (int h = 0; h < NH; ++h) {
                        wgmma_fence();
#pragma unroll
                        for (int g = 0; g < 3; ++g) {
                            const uint32_t sq = q0 + (uint32_t)g, sb = sq % (uint32_t)NBS;
                            if (h == 0) mbar_wait(bar_base + 8u * (BAR_BFULL + sb), resident ? 0u : (sq / (uint32_t)NBS) & 1u);
                            const uint32_t bg = b0 + sb * ((uint32_t)C::B_STAGE >> 4);
#pragma unroll
                            for (int tt = 0; tt < 3; ++tt) {
                                const uint32_t ah = ac + (uint32_t)g * Wrow + (uint32_t)tt, al = ah + A_SPLIT;   // one row = 16 B
                                const uint32_t bh = bg + (uint32_t)tt * B_TAP16 + (uint32_t)(h * NB), bl = bh + B_LO16;   // n rows of 16 B
                                const uint32_t acc_on = (g == 0 && tt == 0) ? 0u : 1u;
                                // ah * bh -> main; al * bh and ah * bl -> cross.  The cross products keep the order of the
                                // earlier forms of this kernel (Cout <= 64: ah * bl first; Cout 128: al * bh first), so the
                                // rounding of every element is unchanged.
                                wgmma_f16<NB>(acc, gmma_desc(ah, DESC_HI), gmma_desc(bh, B_DESC_HI), acc_on);
                                if constexpr (NT < 128) {
                                    wgmma_f16<NB>(acc + NB / 2, gmma_desc(ah, DESC_HI), gmma_desc(bl, B_DESC_HI), acc_on);
                                    wgmma_f16<NB>(acc + NB / 2, gmma_desc(al, DESC_HI), gmma_desc(bh, B_DESC_HI), 1u);
                                } else {
                                    wgmma_f16<NB>(acc + NB / 2, gmma_desc(al, DESC_HI), gmma_desc(bh, B_DESC_HI), acc_on);
                                    wgmma_f16<NB>(acc + NB / 2, gmma_desc(ah, DESC_HI), gmma_desc(bl, B_DESC_HI), 1u);
                                }
                            }
                        }
                        wgmma_commit();
                        wgmma_wait<0>();
                        wgmma_fence_regs<NB>(acc);
#pragma unroll
                        for (int i = 0; i < NB / 2; ++i) run[h * (NB / 2) + i] += fmaf(acc[NB / 2 + i], 0.00048828125f, acc[i]);
                    }
                    __syncwarp();
                    if (lane == 0) {
                        mbar_arrive(bar_base + 8u * (BAR_AEMPTY + slot));
                        if (!resident)
                            for (int g = 0; g < 3; ++g) mbar_arrive(bar_base + 8u * (BAR_BEMPTY + (q0 + (uint32_t)g) % (uint32_t)NBS));
                    }
                    if (++slot == (uint32_t)NA) { slot = 0; a_par ^= 1u; }
                    if (!resident) q += 3;
                }
                // the finished tile, one column block at a time: fragments -> staging -> one row per thread
#pragma unroll
                for (int h = 0; h < NT / SB; ++h) {
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");        // this warpgroup's rows of the staging buffer are free
#pragma unroll
                    for (int i = 0; i < SB / 2; i += 2) {
                        const int col = 8 * (i >> 2) + cq, row = r0 + ((i & 2) ? 8 : 0);
                        *reinterpret_cast<float2 *>(stage + ((size_t)(col >> 2) * SD_BM + row) * 4 + (col & 3)) =
                            make_float2(run[h * (SB / 2) + i], run[h * (SB / 2) + i + 1]);
                    }
                    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
                    const int row = wg * 64 + (tl & 63), cs = (tl >> 6) * (SB / 2);
                    const float4 *st4 = reinterpret_cast<const float4 *>(stage);
                    sd_store_rows<SB / 2, OUT_SD>(p, t, row, h * SB + cs, n_samples, [&](int cc, float (&r)[8]) {
                        const float4 u0 = st4[((cs + cc) >> 2) * SD_BM + row], u1 = st4[(((cs + cc) >> 2) + 1) * SD_BM + row];
                        r[0] = u0.x; r[1] = u0.y; r[2] = u0.z; r[3] = u0.w; r[4] = u1.x; r[5] = u1.y; r[6] = u1.z; r[7] = u1.w;
                    });
                }
        }
        }
    } else {
        setmaxnreg_dec<C::PROD_REGS>();
        if (warp < WGT_WARP) {
            if (IN_SD) {
                // =========================== A producer: presplit images by bulk copy =================================
                // A chunk's four (split, kcore) images are four contiguous 2816-byte runs of the previous layer's output: one
                // thread keeps NA chunks in flight; no register staging, no conversion.  Channels-as-M: chunk c of the unit's
                // tile 2u + g goes to slot 2 s + g (tile 2u again when 2u + 1 does not exist).  The other two warps before the
                // weight warp have no work.
                if (warp == SD_NC && lane == 0) {
                    constexpr uint32_t TPU = C::TPU;
                    const uint32_t nslots = (uint32_t)NA / TPU;
                    uint32_t slot = 0, par = 0, round = 0;
                    for (uint32_t k = 0;; ++k) {
                        int u;
                        if (dyn) {           // draw the next unit and publish it to the other roles
                            u = atomicAdd(p.tile_ctr, 1);
                            if (u >= n_units) u = -1;
                            tile_ring[k & (SD_TRING - 1)] = u;
                            mbar_arrive(bar_base + 8u * (BAR_TILE + (k & (SD_TRING - 1))));
                        } else {
                            u = tile_of(k);
                        }
                        if (u < 0) break;
                        for (int c = 0; c < nchunks; ++c) {
#pragma unroll
                            for (uint32_t g = 0; g < TPU; ++g) {
                                const uint32_t cs = slot * TPU + g;
                                const int t = (int)(TPU * (uint32_t)u + g) < n_tiles ? (int)(TPU * (uint32_t)u + g) : (int)(TPU * (uint32_t)u);
                                if (round) mbar_wait(bar_base + 8u * (BAR_AEMPTY + cs), par ^ 1u);
                                mbar_arrive_expect_tx(bar_base + 8u * (BAR_AFULL + cs), 4u * (uint32_t)SD_KBYTES);
                                const unsigned char *src = reinterpret_cast<const unsigned char *>(p.in_sd) + ((size_t)(c * 4) * p.rows_in + (size_t)t * SD_BM) * 16;
#pragma unroll
                                for (int im = 0; im < 4; ++im)
                                    bulk_g2s(a_base + cs * (uint32_t)SD_CHUNK + (uint32_t)im * SD_KBYTES, src + (size_t)im * p.rows_in * 16, (uint32_t)SD_KBYTES,
                                             bar_base + 8u * (BAR_AFULL + cs));
                            }
                            if (++slot == nslots) { slot = 0; par ^= 1u; round = 1; }
                        }
                    }
                }
                __syncwarp();
            } else {
            // =========================== loaders: fp32 activations -> fp16 hi/lo chunk images ====================
                // A chunk image is 2 x 176 items of (row, 8 channels) = two 16-byte loads each; thread `ltid` owns the items ltid,
                // ltid + 96, ltid + 192, ltid + 288 of EVERY chunk.  The activations come from HBM: all eight loads of a chunk are
                // issued at once and the loads of chunk j + 1 are in flight while chunk j is converted, so no chunk waits a whole
                // exposed round trip.
                constexpr int ITEMS = (2 * SD_AROWS + SD_NL * 32 - 1) / (SD_NL * 32);      // 4
                const int ltid = tid - SD_NC * 32;
                const float4 *in4 = reinterpret_cast<const float4 *>(p.in);
                float amax = 0.0f;
                float4 cur[ITEMS][2], nxt[ITEMS][2];
                auto issue = [&](int t, int c, float4 (&v)[ITEMS][2]) {
                    const long long p0 = (long long)t * SD_BM;
#pragma unroll
                    for (int m = 0; m < ITEMS; ++m) {
                        const int idx = ltid + m * SD_NL * 32;
                        v[m][0] = make_float4(0.f, 0.f, 0.f, 0.f);
                        v[m][1] = v[m][0];
                        if (idx < 2 * SD_AROWS) {
                            const int h = idx >= SD_AROWS ? 1 : 0, r = idx - h * SD_AROWS;
                            const long long pr = p0 + r;
                            const int s = (int)(pr / p.rs), q = (int)(pr - (long long)s * p.rs);
                            const int yp = q / 22, xp = q - yp * 22;
                            if (s < n_samples && (yp != 0 || !p.cyl) && !p.fa) {
                                const int xx = xp == 0 ? 19 : (xp == 21 ? 0 : xp - 1);
                                int pos = p.cyl ? (yp - 1) * 20 + xx : q, g0;       // valid rasters: the row IS the input position
                                if (p.is3d) { pos += c * 140; g0 = h * 2; } else { g0 = c * 4 + h * 2; }
                                const float4 *src = in4 + ((size_t)s * p.G_in + g0) * p.S_in + pos;
                                v[m][0] = __ldg(src);
                                v[m][1] = __ldg(src + p.S_in);
                            }
                        }
                    }
                };
                int j = 0;
                int t = blockIdx.x, c = 0;
                if (t < n_tiles) issue(t, 0, cur);
                while (t < n_tiles) {
                    // position of the chunk after this one
                    int tn = t, cn = c + 1;
                    if (cn == nchunks) { cn = 0; tn = t + gridDim.x; }
                    if (tn < n_tiles) issue(tn, cn, nxt);
                    const int slot = j % NA;
                    if (j >= NA) mbar_wait(bar_base + 8u * (BAR_AEMPTY + slot), (uint32_t)(((j / NA) - 1) & 1));
                    unsigned char *dst = smem + (size_t)slot * SD_CHUNK;
                    if (p.fa) {
                        // second CostNet layer: the first layer's activation relu(A[c][k][(l - n) mod 20] - B[c][k][l]) is regenerated
                        // here from the factor maps (models/BUFFERX.py:39-69 + patchnet.py:192-198, factorised by bx_costvol_ab).  Raster
                        // row q = (n, l) of the 18 x 18 grid; chunk c = (k = c / 2, channels 16 * (c % 2) ...): the k dimension of the
                        // 3x3x3 kernel is folded into the channels, the taps are (dn, dl).  The 14.6 KB of factors per match are L2
                        // hits, so all loads of the chunk are issued here, no cross-chunk prefetch.
                        const long long p0 = (long long)t * SD_BM;
                        const int kk = c >> 1, cb = (c & 1) * 4;
                        float4 va[ITEMS][2], vb[ITEMS][2];
#pragma unroll
                        for (int m = 0; m < ITEMS; ++m) {
                            const int idx = ltid + m * SD_NL * 32;
                            va[m][0] = va[m][1] = vb[m][0] = vb[m][1] = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (idx < 2 * SD_AROWS) {
                                const int h = idx >= SD_AROWS ? 1 : 0, r = idx - h * SD_AROWS;
                                const long long pr = p0 + r;
                                const int s = (int)(pr / 324), q = (int)(pr - (long long)s * 324);
                                const int nn = q / 18, ll = q - nn * 18;
                                if (s < n_samples) {
                                    int sh = ll - nn;
                                    sh = sh < 0 ? sh + 20 : sh;
                                    const float4 *sa = reinterpret_cast<const float4 *>(p.fa) + ((size_t)s * 8 + cb + h * 2) * 60 + kk * 20 + sh;
                                    const float4 *sb = reinterpret_cast<const float4 *>(p.fb) + ((size_t)s * 8 + cb + h * 2) * 54 + kk * 18 + ll;
                                    va[m][0] = __ldg(sa); va[m][1] = __ldg(sa + 60);
                                    vb[m][0] = __ldg(sb); vb[m][1] = __ldg(sb + 54);
                                }
                            }
                        }
#pragma unroll
                        for (int m = 0; m < ITEMS; ++m) {
                            cur[m][0] = make_float4(fmaxf(va[m][0].x - vb[m][0].x, 0.f), fmaxf(va[m][0].y - vb[m][0].y, 0.f), fmaxf(va[m][0].z - vb[m][0].z, 0.f),
                                                    fmaxf(va[m][0].w - vb[m][0].w, 0.f));
                            cur[m][1] = make_float4(fmaxf(va[m][1].x - vb[m][1].x, 0.f), fmaxf(va[m][1].y - vb[m][1].y, 0.f), fmaxf(va[m][1].z - vb[m][1].z, 0.f),
                                                    fmaxf(va[m][1].w - vb[m][1].w, 0.f));
                        }
                    }
#pragma unroll
                    for (int m = 0; m < ITEMS; ++m) {
                        const int idx = ltid + m * SD_NL * 32;
                        if (idx < 2 * SD_AROWS) {
                            const int h = idx >= SD_AROWS ? 1 : 0, r = idx - h * SD_AROWS;
                            const float xs[8] = {cur[m][0].x, cur[m][0].y, cur[m][0].z, cur[m][0].w, cur[m][1].x, cur[m][1].y, cur[m][1].z, cur[m][1].w};
                            uint32_t hi[4], lo[4];
#pragma unroll
                            for (int e = 0; e < 4; ++e) {
                                const __half2 hh = __floats2half2_rn(xs[2 * e], xs[2 * e + 1]);
                                const float2 hf = __half22float2(hh);
                                const __half2 ll = __floats2half2_rn((xs[2 * e] - hf.x) * 2048.0f, (xs[2 * e + 1] - hf.y) * 2048.0f);
                                hi[e] = *reinterpret_cast<const uint32_t *>(&hh);
                                lo[e] = *reinterpret_cast<const uint32_t *>(&ll);
                                amax = fmaxf(amax, fmaxf(fabsf(xs[2 * e]), fabsf(xs[2 * e + 1])));
                            }
                            *reinterpret_cast<uint4 *>(dst + (size_t)h * SD_KBYTES + (size_t)r * 16) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                            *reinterpret_cast<uint4 *>(dst + (size_t)(2 + h) * SD_KBYTES + (size_t)r * 16) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy stores -> tensor-core (async proxy) reads
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_base + 8u * (BAR_AFULL + slot));
#pragma unroll
                    for (int m = 0; m < ITEMS; ++m) { cur[m][0] = nxt[m][0]; cur[m][1] = nxt[m][1]; }
                    t = tn; c = cn; ++j;
                }
                if (!(amax < 65000.0f) && p.flag) atomicOr(p.flag, 1);   // also true for NaN
            }
        } else {
            // =========================== weight producer ========================================================
            if (lane == 0) {
                const int n_st = nchunks * 3;
                uint32_t q = 0;
                for (uint32_t k = 0; tile_of(k) >= 0; ++k) {
                    if (resident && k >= 1) break;                      // resident weights: loaded by the first tile, never again
                    for (int s = 0; s < n_st; ++s, ++q) {
                        const uint32_t sb = q % (uint32_t)NBS, use = q / (uint32_t)NBS;
                        if (use > 0) mbar_wait(bar_base + 8u * (BAR_BEMPTY + sb), (use - 1) & 1u);
                        mbar_arrive_expect_tx(bar_base + 8u * (BAR_BFULL + sb), (uint32_t)C::B_STAGE);
                        bulk_g2s(b_base + sb * (uint32_t)C::B_STAGE, reinterpret_cast<const unsigned char *>(p.w) + (size_t)s * C::B_STAGE,
                                 (uint32_t)C::B_STAGE, bar_base + 8u * (BAR_BFULL + sb));
                    }
                }
            }
            __syncwarp();
        }
    }
    __syncthreads();
    if (dyn && tid == 0) {      // the last CTA to finish rewinds the counters for the next launch that uses them
        __threadfence();
        if (atomicAdd(p.tile_ctr + 1, 1) == (int)gridDim.x - 1) { p.tile_ctr[0] = 0; p.tile_ctr[1] = 0; __threadfence(); }
    }
}

template <int NT, int IN_SD, int OUT_SD>
int launch_sd(ConvSdParams p, cudaStream_t st) {
    using C = SdCfg<NT, IN_SD>;
    // the whole weight image resident in shared memory when it leaves room for three A chunks (channels-as-M: two per
    // warpgroup), else a ring of six stages (two chunks) or as many as leave room for four A chunks.  Channels-as-M slots come
    // in pairs, one per warpgroup.
    const int budget = SD_SMEM - C::STAGE_BYTES, n_st = p.nchunks * 3;
    p.resident = n_st <= SD_MAXNBS && budget - n_st * C::B_STAGE >= (C::CM ? 4 : 3) * SD_CHUNK;
    p.nbs = p.resident ? n_st : 6;
    while (!p.resident && p.nbs > 3 && budget - p.nbs * C::B_STAGE < 4 * SD_CHUNK) --p.nbs;
    int na = (budget - p.nbs * C::B_STAGE) / SD_CHUNK;
    if (na > 2 * C::TPU * p.nchunks) na = 2 * C::TPU * p.nchunks;
    if (na > SD_MAXNA) na = SD_MAXNA;
    na -= na % C::TPU;
    BX_REQUIRE(na >= 2 * C::TPU, "bx_conv_layer_sd: no room for the activation ring");
    p.NA = na;
    const int smem = na * SD_CHUNK + p.nbs * C::B_STAGE + C::STAGE_BYTES;
    static BxPerDevice attr = {};
    if (bx_needs_attr(attr, (size_t)smem))
        BX_CUDA(cudaFuncSetAttribute(conv_sd_kernel<NT, IN_SD, OUT_SD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int sms = bx_device_sm_count();
    if (sms <= 0) sms = 132;
    const int units = (p.n_tiles + C::TPU - 1) / C::TPU;
    const int grid = units < sms ? units : sms;
    conv_sd_kernel<NT, IN_SD, OUT_SD><<<grid, C::THREADS, smem, st>>>(p);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

template <int NT>
int dispatch_sd(const ConvSdParams &p, int in_sd, int out_sd, cudaStream_t st) {
    if (in_sd) return out_sd ? launch_sd<NT, 1, 1>(p, st) : launch_sd<NT, 1, 0>(p, st);
    return out_sd ? launch_sd<NT, 0, 1>(p, st) : launch_sd<NT, 0, 0>(p, st);
}

}  // namespace

// rows of a presplit activation image: n samples of rows_per_sample raster rows (176 for the cylindrical layers: 8 x 22),
// rounded to whole 128-row tiles, + the 48-row halo a tile's operand fetch reaches past its last row
BX_API long long bx_conv_sd_rows(int n, int rows_per_sample) {
    const long long rows = (long long)n * rows_per_sample;
    return (rows + SD_BM - 1) / SD_BM * SD_BM + (SD_AROWS - SD_BM);
}

BX_API int bx_conv_layer_sd(int geom, const void *in, int in_presplit, const void *w_sd, const float *bias, void *out, int out_presplit,
                            int n, const int32_t *d_n, int Cin, int Cout, int D, int W, int relu, int32_t *d_flag, int32_t *d_tile_ctr, void *stream) {
    BX_REQUIRE(in && w_sd && bias && out, "bx_conv_layer_sd: null pointer");
    BX_REQUIRE(geom == BX_GEOM_CYL3D || geom == BX_GEOM_CYL2D || geom == BX_GEOM_VALID3D, "bx_conv_layer_sd: geometry must be CYL3D, CYL2D or VALID3D (k = 3x1x3)");
    BX_REQUIRE(n >= 0 && Cin >= 16 && Cin % 16 == 0 && Cout >= 4 && Cout % 4 == 0 && Cout <= 128, "bx_conv_layer_sd: bad channels Cin=%d Cout=%d", Cin, Cout);
    BX_REQUIRE(geom != BX_GEOM_CYL3D || Cin == 16, "bx_conv_layer_sd: CYL3D expects 16 input channels x 3 radial slices");
    BX_REQUIRE(geom != BX_GEOM_VALID3D || (D >= 3 && W >= 3 && 2 * W + 2 <= SD_AROWS - SD_BM), "bx_conv_layer_sd: VALID3D raster %d x %d out of range (W <= 23)", D, W);
    BX_REQUIRE(!out_presplit || Cout % 16 == 0, "bx_conv_layer_sd: presplit output needs Cout %% 16 == 0");
    BX_REQUIRE(((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(bias) | reinterpret_cast<uintptr_t>(w_sd)) & 15) == 0,
               "bx_conv_layer_sd: activations, weights and bias must be 16-byte aligned");
    if (n == 0) return BX_OK;
    ConvSdParams p = {};
    p.w = reinterpret_cast<const __half *>(w_sd); p.bias = bias; p.flag = d_flag; p.d_n = d_n; p.tile_ctr = d_tile_ctr;
    p.in = in_presplit ? nullptr : reinterpret_cast<const float *>(in);
    p.in_sd = in_presplit ? reinterpret_cast<const __half *>(in) : nullptr;
    p.out = out_presplit ? nullptr : reinterpret_cast<float *>(out);
    p.out_sd = out_presplit ? reinterpret_cast<__half *>(out) : nullptr;
    p.n = n; p.Cout = Cout; p.relu = relu;
    p.is3d = geom == BX_GEOM_CYL3D;
    p.cyl = geom != BX_GEOM_VALID3D;
    p.nchunks = p.is3d ? 3 : Cin / 16;
    p.G_in = Cin / 4;
    if (p.cyl) {
        p.rs = SD_SROWS; p.W = 22; p.OD = 7; p.OW = 20; p.S_out = 140; p.rs_out = SD_SROWS;
        p.S_in = p.is3d ? 420 : 140;
    } else {        // valid k = (3,1,3) convolution over a D x W raster (CostNet layers, models/patchnet.py:151-210)
        p.rs = D * W; p.W = W; p.OD = D - 2; p.OW = W - 2; p.S_out = p.OD * p.OW; p.rs_out = p.S_out;
        p.S_in = D * W;
    }
    const long long rows = (long long)n * p.rs;
    BX_REQUIRE(rows + 4 * SD_BM < 0x7fffffffLL, "bx_conv_layer_sd: too many samples (raster rows must stay below 2^31)");
    p.n_tiles = (int)((rows + SD_BM - 1) / SD_BM);
    p.rows_in = bx_conv_sd_rows(n, p.rs);
    p.rows_out = bx_conv_sd_rows(n, p.rs_out);
    cudaStream_t st = bx_stream(stream);
    if (Cout > 64) return dispatch_sd<128>(p, in_presplit, out_presplit, st);
    if (Cout > 32) return dispatch_sd<64>(p, in_presplit, out_presplit, st);
    return dispatch_sd<32>(p, in_presplit, out_presplit, st);
}

/* Second CostNet layer on the shifted-descriptor kernel: conv 32 -> 64, k = 3x3x3 over the regenerated first activation
 * relu(A - B) [32, 18, 3, 18] (see bx_costvol_ab), computed as a 96 -> 64 convolution with k = (3,1,3) over the 18 x 18 (n, l)
 * raster -- the three k rows become channel chunks.  w_sd: ops.conv_sd_weights_costab image; out: [n,16,256,4] fp32 or the
 * presplit image over the 16 x 16 output raster (rows = bx_conv_sd_rows(n, 256)). */
BX_API int bx_conv_layer_sd_costab(const float *fa, const float *fb, const void *w_sd, const float *bias, void *out, int out_presplit, int n,
                                   const int32_t *d_n, int relu, int32_t *d_flag, void *stream) {
    BX_REQUIRE(fa && fb && w_sd && bias && out, "bx_conv_layer_sd_costab: null pointer");
    BX_REQUIRE(((reinterpret_cast<uintptr_t>(fa) | reinterpret_cast<uintptr_t>(fb) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(bias) |
                 reinterpret_cast<uintptr_t>(w_sd)) & 15) == 0, "bx_conv_layer_sd_costab: pointers must be 16-byte aligned");
    if (n <= 0) return BX_OK;
    ConvSdParams p = {};
    p.w = reinterpret_cast<const __half *>(w_sd); p.bias = bias; p.flag = d_flag; p.d_n = d_n;
    p.fa = fa; p.fb = fb;
    p.in = fa;                     // unused by the COSTAB loader
    p.out = out_presplit ? nullptr : reinterpret_cast<float *>(out);
    p.out_sd = out_presplit ? reinterpret_cast<__half *>(out) : nullptr;
    p.n = n; p.Cout = 64; p.relu = relu;
    p.is3d = 0; p.cyl = 0; p.nchunks = 6; p.G_in = 8;
    p.rs = 324; p.W = 18; p.OD = 16; p.OW = 16; p.S_out = 256; p.rs_out = 256; p.S_in = 324;
    p.n_tiles = (int)(((long long)n * p.rs + SD_BM - 1) / SD_BM);
    p.rows_in = bx_conv_sd_rows(n, p.rs);
    p.rows_out = bx_conv_sd_rows(n, p.rs_out);
    return dispatch_sd<64>(p, 0, out_presplit, bx_stream(stream));
}
