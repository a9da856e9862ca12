// bx_train_desc.cu -- the Desc-stage training step (reference trainer.py:93-167 with cfg.stage "Desc", model.train()):
// MiniSpinNet's forward with batch-statistics BatchNorm and its backward pass, in float64.
//
// Float64 for the reason bx_train_step.cu gives for CostNet: a lower layer's gradient passes through up to ten
// batch-statistics BatchNorm backwards (point layer, seven in the cylindrical stack, two in the pool layer), each of which can
// cancel most of its input.  The forward is float64 as well: the backward consumes its activations and batch statistics.
//
// Activations are channel-blocked float64 [n][C/4][S][4] (the layout of the bx_ts_* kernels); a cylindrical raster is
// 7 elevation x 20 azimuth positions (S = 140 per depth slice).
//
// The cylindrical convolutions (patchnet.py:68-84: padded circularly in azimuth and with zeros in elevation,
// utils/common.py:265-310, then a valid 3x3 or 3x3x3 convolution) run as implicit GEMMs on the fp64 tensor-core MMA
// (mma.sync m16n8k16 .f64, DMMA on sm_90).  The padding lives in the operand loader: a tap that reads outside the
// elevation range loads a zero, an azimuth index wraps.  The data gradient is the same cylindrical convolution with the taps
// flipped and the weight transposed (the padding rule maps onto itself), one launch per input depth slice.
//
// The 1x1 convolution (fp32 and float64) and the BatchNorm + ReLU backward carry the bx_ts_ prefix: the Pose step runs
// them too (its frozen descriptor's pool layer, CostNet's BatchNorms with gamma = 1).
//
// Determinism: every reduction over samples x positions goes through BX_TS_SPLITS per-block partials summed in index
// order by one thread per output; no floating-point atomics.  Two runs on the same inputs are bit-identical.
#include "bx_splits.cuh"

namespace {

constexpr int CYL_E = 7, CYL_A = 20, CYL_S = CYL_E * CYL_A;
constexpr double NORM_EPS = 1e-12;        // F.normalize's eps

__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
        "{%0,%1,%2,%3};\n"
        : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]),
          "d"(b[3]));
}

// input position of output position p under tap t = (d, de, da) of a cylindrical raster, or -1 (zero elevation padding)
__device__ __forceinline__ int cyl_src(int p, int t) {
    const int e = p / CYL_A, a = p - e * CYL_A;
    const int d = t / 9, de = (t / 3) % 3, da = t % 3;
    const int ee = e + de - 1;
    if (ee < 0 || ee >= CYL_E) return -1;
    int aa = a + da - 1;
    aa = aa < 0 ? aa + CYL_A : (aa >= CYL_A ? aa - CYL_A : aa);
    return d * CYL_S + ee * CYL_A + aa;
}

// Cylindrical convolution as a row-major implicit GEMM on DMMA: rows (sample, output position), columns the Nc output
// channels, k = (tap, Kc input channels).
//   forward (!DGRAD): in = x [n][Kc/4][Din*140][4], w [Din*9][Kc][Nc], bias [Nc]; out[s][co][p] = b + sum w x[tap(p)]
//   DGRAD: in = dy [n][Kc/4][140][4], w the forward weight [Dw*9][Nc][Kc] of which depth slice wd is used with flipped
//          taps: out = dx of that slice.
// out is [n][Nc/4][out_S][4], written at positions out_off + p.  CTA: 64 rows x 64 columns, 4 warps of 16 rows x 8
// m16n8 fragments; k-chunks of 16 channels of one tap.  Kc % 16 == 0, Nc % 8 == 0.
constexpr int CM_BM = 64, CM_BN = 64, CM_AP = 20, CM_BP = 68;

template <bool DGRAD>
__global__ void __launch_bounds__(128) cyl_mma_kernel(const double *__restrict__ in, const double *__restrict__ w,
                                                      const double *__restrict__ bias, int n, int Kc, int Nc, int Din, int wd,
                                                      int out_S, int out_off, double *__restrict__ out) {
    __shared__ __align__(16) double As[CM_BM * CM_AP];
    __shared__ __align__(16) double Bs[16 * CM_BP];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tig = lane & 3;
    const long long rows = (long long)n * CYL_S;
    const long long r0 = (long long)blockIdx.x * CM_BM;
    const int n0 = blockIdx.y * CM_BN;
    const int Gk = Kc / 4, S_in = Din * CYL_S;
    // the two (row, channel group) items this thread loads per chunk
    int lrow[2], lgrp[2], ls[2], lp[2];
    bool lval[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int i = tid + 128 * h;
        lrow[h] = i & 63;
        lgrp[h] = i >> 6;
        const long long gr = r0 + lrow[h];
        lval[h] = gr < rows;
        ls[h] = lval[h] ? (int)(gr / CYL_S) : 0;
        lp[h] = lval[h] ? (int)(gr % CYL_S) : 0;
    }
    double acc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0;
    const int T = DGRAD ? 9 : Din * 9;
    for (int t = 0; t < T; ++t) {
        int src[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) src[h] = lval[h] ? cyl_src(lp[h], t) : -1;
        const int tw = DGRAD ? wd * 9 + 8 - t : t;
        for (int k0 = 0; k0 < Kc; k0 += 16) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                double2 v0 = make_double2(0.0, 0.0), v1 = v0;
                if (src[h] >= 0) {
                    const double2 *p =
                        reinterpret_cast<const double2 *>(in + (((size_t)ls[h] * Gk + k0 / 4 + lgrp[h]) * S_in + src[h]) * 4);
                    v0 = p[0];
                    v1 = p[1];
                }
                double *a = As + lrow[h] * CM_AP + 4 * lgrp[h];
                a[0] = v0.x; a[1] = v0.y; a[2] = v1.x; a[3] = v1.y;
            }
#pragma unroll
            for (int h = 0; h < 8; ++h) {
                const int e = tid + 128 * h;
                int c, j;
                double v = 0.0;
                if (!DGRAD) {
                    c = e >> 6; j = e & 63;
                    if (n0 + j < Nc) v = w[((size_t)tw * Kc + k0 + c) * Nc + n0 + j];
                } else {
                    c = e & 15; j = e >> 4;
                    if (n0 + j < Nc) v = w[((size_t)tw * Nc + n0 + j) * Kc + k0 + c];
                }
                Bs[c * CM_BP + j] = v;
            }
            __syncthreads();
            double af[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) af[i] = As[(16 * warp + g + 8 * (i & 1)) * CM_AP + tig + 4 * (i >> 1)];
#pragma unroll
            for (int nb = 0; nb < 8; ++nb) {
                double bf[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) bf[i] = Bs[(tig + 4 * i) * CM_BP + nb * 8 + g];
                dmma16816(acc[nb], af, bf);
            }
            __syncthreads();
        }
    }
    const int Gn = Nc / 4;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const long long row = r0 + 16 * warp + g + 8 * hh;
        if (row >= rows) continue;
        const int s = (int)(row / CYL_S), p = (int)(row % CYL_S);
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) {
            const int col = n0 + nb * 8 + 2 * tig;
            if (col >= Nc) continue;
            double v0 = acc[nb][2 * hh], v1 = acc[nb][2 * hh + 1];
            if (!DGRAD) {
                v0 += bias[col];
                v1 += bias[col + 1];
            }
            *reinterpret_cast<double2 *>(out + (((size_t)s * Gn + col / 4) * out_S + out_off + p) * 4 + (col & 3)) = make_double2(v0, v1);
        }
    }
}

// Weight gradient of the cylindrical convolution on DMMA: dw[t][ci][co] = sum_{s, p} x[s][ci][tap_t(p)] dy[s][co][p]
// (m = ci, n = co, k = rows (s, p)).  CTA = (tap, 32 input channels, 64 output channels) x one of BX_TS_SPLITS contiguous
// row ranges; 4 warps of one m16 fragment x 4 n8 fragments; rows in chunks of 32; partial [split][t][ci][co].
constexpr int WG_RC = 32, WG_XP = 36, WG_DP = 68;

__global__ void __launch_bounds__(128, 1) cyl_wgrad_kernel(const double *__restrict__ x, const double *__restrict__ dy, int n, int Cin,
                                                        int Cout, int Din, double *__restrict__ partial) {
    __shared__ __align__(16) double Xs[WG_RC * WG_XP];
    __shared__ __align__(16) double Ds[WG_RC * WG_DP];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tig = lane & 3;
    const int nci = (Cin + 31) / 32, nco = (Cout + 63) / 64;
    int b = blockIdx.x;
    const int cot = b % nco; b /= nco;
    const int cit = b % nci;
    const int t = b / nci;
    const int T = Din * 9, S_in = Din * CYL_S;
    const long long R = (long long)n * CYL_S;
    const long long per = (R + gridDim.y - 1) / gridDim.y;
    const long long rb = min(R, per * blockIdx.y), re = min(R, rb + per);
    const int Gi = Cin / 4, Go = Cout / 4;
    const int mf = warp & 1, nf0 = (warp >> 1) * 4;
    double acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0;
#pragma unroll 1
    for (long long c0 = rb; c0 < re; c0 += WG_RC) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {            // Xs: 32 rows x 8 channel groups
            const int i = tid + 128 * h, r = i & 31, grp = i >> 5;
            const long long row = c0 + r;
            double2 v0 = make_double2(0.0, 0.0), v1 = v0;
            const int ga = cit * 8 + grp;
            if (row < re && ga < Gi) {
                const int s = (int)(row / CYL_S), p = (int)(row % CYL_S);
                const int src = cyl_src(p, t);
                if (src >= 0) {
                    const double2 *q = reinterpret_cast<const double2 *>(x + (((size_t)s * Gi + ga) * S_in + src) * 4);
                    v0 = q[0];
                    v1 = q[1];
                }
            }
            double *a = Xs + r * WG_XP + 4 * grp;
            a[0] = v0.x; a[1] = v0.y; a[2] = v1.x; a[3] = v1.y;
        }
#pragma unroll
        for (int h = 0; h < 4; ++h) {            // Ds: 32 rows x 16 channel groups
            const int i = tid + 128 * h, r = i & 31, grp = i >> 5;
            const long long row = c0 + r;
            double2 v0 = make_double2(0.0, 0.0), v1 = v0;
            const int gd = cot * 16 + grp;
            if (row < re && gd < Go) {
                const int s = (int)(row / CYL_S), p = (int)(row % CYL_S);
                const double2 *q = reinterpret_cast<const double2 *>(dy + (((size_t)s * Go + gd) * CYL_S + p) * 4);
                v0 = q[0];
                v1 = q[1];
            }
            double *d = Ds + r * WG_DP + 4 * grp;
            d[0] = v0.x; d[1] = v0.y; d[2] = v1.x; d[3] = v1.y;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < WG_RC / 16; ++kk) {
            double af[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) af[i] = Xs[(kk * 16 + tig + 4 * (i >> 1)) * WG_XP + mf * 16 + g + 8 * (i & 1)];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                double bf[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) bf[i] = Ds[(kk * 16 + tig + 4 * i) * WG_DP + (nf0 + j) * 8 + g];
                dmma16816(acc[j], af, bf);
            }
        }
        __syncthreads();
    }
    const size_t L = (size_t)T * Cin * Cout;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int ci = cit * 32 + mf * 16 + g + 8 * hh;
        if (ci >= Cin) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int co = cot * 64 + (nf0 + j) * 8 + 2 * tig;
            if (co >= Cout) continue;
            double *o = partial + (size_t)blockIdx.y * L + ((size_t)t * Cin + ci) * Cout + co;
            o[0] = acc[j][2 * hh];
            o[1] = acc[j][2 * hh + 1];
        }
    }
}

// Point layer, training forward (patch_embedder.py:78-90): per (patch, voxel) and channel c the nv samples
// y = W[c] . inv + b[c], x^ = y scale[c] + shift[c] (affine batch-statistics BatchNorm folded), ReLU, max over the samples
// (the first maximum, as max_pool2d).  feat blocked [K][4][V][4], arg [K][16][V] the index of the maximum.
__global__ void pnt_forward_kernel(const float *__restrict__ inv, const double *__restrict__ W, const double *__restrict__ b,
                                   const double *__restrict__ scale, const double *__restrict__ shift, int K, int V, int nv,
                                   double *__restrict__ feat, unsigned char *__restrict__ arg) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)K * V) return;
    const int k = (int)(i / V), v = (int)(i % V);
    const float *sm = inv + (size_t)i * nv * 3;
    for (int c = 0; c < 16; ++c) {
        double best = 0.0;
        int ba = 0;
        for (int a = 0; a < nv; ++a) {
            const double y = W[3 * c] * (double)sm[3 * a] + W[3 * c + 1] * (double)sm[3 * a + 1] + W[3 * c + 2] * (double)sm[3 * a + 2] + b[c];
            double r = y * scale[c] + shift[c];
            r = r > 0.0 ? r : 0.0;
            if (a == 0 || r > best) {
                best = r;
                ba = a;
            }
        }
        feat[(((size_t)k * 4 + c / 4) * V + v) * 4 + (c & 3)] = best;
        arg[((size_t)k * 16 + c) * V + v] = (unsigned char)ba;
    }
}

// Point layer backward, the sparse pass: the feature gradient goes to the selected sample of each (patch, channel, voxel),
// masked by the ReLU (dz).  Per channel the sums sum dz, sum dz x^ (x^ = (y - mean) rstd) and sum dz inv (3).
// grid (16, BX_TS_SPLITS); partial [split][16][5].
__global__ void __launch_bounds__(TS_THREADS) pnt_bwd_sums_kernel(const float *__restrict__ inv, const unsigned char *__restrict__ arg,
                                                                  const double *__restrict__ dfeat, const double *__restrict__ W,
                                                                  const double *__restrict__ b, const double *__restrict__ mean,
                                                                  const double *__restrict__ rstd, const double *__restrict__ scale,
                                                                  const double *__restrict__ shift, int K, int V, int nv,
                                                                  double *__restrict__ partial) {
    __shared__ double sh[5 * TS_THREADS];
    const int c = blockIdx.x, split = blockIdx.y, nsplit = gridDim.y;
    const long long R = (long long)K * V;
    const long long per = (R + nsplit - 1) / nsplit;
    const long long rb = min(R, per * split), re = min(R, rb + per);
    double acc[5] = {0, 0, 0, 0, 0};
    const double w0 = W[3 * c], w1 = W[3 * c + 1], w2 = W[3 * c + 2];
    for (long long i = rb + threadIdx.x; i < re; i += TS_THREADS) {
        const int k = (int)(i / V), v = (int)(i % V);
        const int a = arg[((size_t)k * 16 + c) * V + v];
        const float *q = inv + ((size_t)i * nv + a) * 3;
        const double x0 = q[0], x1 = q[1], x2 = q[2];
        const double y = w0 * x0 + w1 * x1 + w2 * x2 + b[c];
        if (y * scale[c] + shift[c] > 0.0) {
            const double dz = dfeat[(((size_t)k * 4 + c / 4) * V + v) * 4 + (c & 3)];
            acc[0] += dz;
            acc[1] += dz * ((y - mean[c]) * rstd[c]);
            acc[2] += dz * x0;
            acc[3] += dz * x1;
            acc[4] += dz * x2;
        }
    }
    block_sum<5>(acc, sh);
    if (threadIdx.x == 0)
        for (int j = 0; j < 5; ++j) partial[((size_t)split * 16 + c) * 5 + j] = sh[j * TS_THREADS];
}

// Point layer backward, the closing step (one thread per channel): with S the split sums of pnt_bwd_sums_kernel and the
// moments mo [9] of all R samples (zero slots included),
//   dgamma = S1, dbeta = S0, dy_r = gamma rstd (dz_r - m1 - x^_r m2), m1 = S0 / R, m2 = S1 / R,
//   dW = sum_r dy_r inv_r^T = gamma rstd (S_inv - m1 sum inv - m2 sum x^ inv^T), db = gamma rstd (S0 - R m1 - m2 sum x^),
// where sum x^ inv^T = rstd (W sum inv inv^T + (b - mean) sum inv^T) and sum x^ = rstd (W sum inv + R (b - mean)): the
// dense sums over every sample follow from the moments.  out [16][6] = dW (3), db, dgamma, dbeta.
__global__ void pnt_bwd_final_kernel(const double *__restrict__ partial, int nsplit, const double *__restrict__ mo, double R,
                                     const double *__restrict__ W, const double *__restrict__ b, const double *__restrict__ mean,
                                     const double *__restrict__ rstd, const double *__restrict__ gamma, double *__restrict__ out) {
    const int c = threadIdx.x;
    if (c >= 16) return;
    double S[5] = {0, 0, 0, 0, 0};
    for (int i = 0; i < nsplit; ++i)
        for (int j = 0; j < 5; ++j) S[j] += partial[((size_t)i * 16 + c) * 5 + j];
    const double M[3][3] = {{mo[3], mo[4], mo[5]}, {mo[4], mo[6], mo[7]}, {mo[5], mo[7], mo[8]}};
    const double m1 = S[0] / R, m2 = S[1] / R, rs = rstd[c], G = gamma[c] * rs, off = b[c] - mean[c];
    double sxh = 0.0;
    for (int j = 0; j < 3; ++j) sxh += W[3 * c + j] * mo[j];
    sxh = rs * (sxh + R * off);
    for (int j = 0; j < 3; ++j) {
        double sxi = 0.0;
        for (int l = 0; l < 3; ++l) sxi += W[3 * c + l] * M[l][j];
        sxi = rs * (sxi + off * mo[j]);
        out[6 * c + j] = G * (S[2 + j] - m1 * mo[j] - m2 * sxi);
    }
    out[6 * c + 3] = G * (S[0] - R * m1 - m2 * sxh);
    out[6 * c + 4] = S[1];
    out[6 * c + 5] = S[0];
}

// 1x1 convolution of a blocked image, fp32 or float64: out[s][co][p] (+)= b[co] + sum_ci w[ci][co] x[s][ci][p], the
// accumulator starting at the bias (0 without one), then one fused multiply-add per input channel in channel order.
// Cin, Cout <= 32, multiples of 4.
template <typename T>
__global__ void conv1x1_kernel(const T *__restrict__ x, const T *__restrict__ w, const T *__restrict__ b, int n, int Cin, int Cout,
                               int S, int accumulate, T *__restrict__ out) {
    __shared__ T ws[32 * 32 + 32];
    for (int i = threadIdx.x; i < Cin * Cout; i += blockDim.x) ws[i] = w[i];
    for (int i = threadIdx.x; i < Cout; i += blockDim.x) ws[Cin * Cout + i] = b ? b[i] : T(0);
    __syncthreads();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n * S) return;
    const int s = (int)(t / S), p = (int)(t % S);
    T acc[32];
#pragma unroll
    for (int co = 0; co < 32; ++co) acc[co] = co < Cout ? ws[Cin * Cout + co] : T(0);
    const int Gi = Cin / 4, Go = Cout / 4;
    for (int g = 0; g < Gi; ++g) {
        const T *xp = x + (((size_t)s * Gi + g) * S + p) * 4;
        for (int j = 0; j < 4; ++j) {
            const T a = xp[j];
#pragma unroll
            for (int co = 0; co < 32; ++co)
                if (co < Cout) acc[co] = fma(ws[(4 * g + j) * Cout + co], a, acc[co]);
        }
    }
#pragma unroll
    for (int co = 0; co < 32; ++co) {
        if (co >= Cout) break;
        T *o = out + (((size_t)s * Go + co / 4) * S + p) * 4 + (co & 3);
        *o = accumulate ? *o + acc[co] : acc[co];
    }
}

// sum over (s, p) of X[s][a][p] D[s][b][p] for every channel pair (the weight gradient of a 1x1 convolution); grid
// (Ca/4 * Cb/4, BX_TS_SPLITS), each thread a 4 x 4 block of pairs; partial [split][Ca][Cb]
__global__ void __launch_bounds__(TS_THREADS) cross_sums_kernel(const double *__restrict__ X, const double *__restrict__ D, int n, int Ca,
                                                                int Cb, int S, double *__restrict__ partial) {
    __shared__ double sh[16 * TS_THREADS];
    const int Gb = Cb / 4, ga = blockIdx.x / Gb, gb = blockIdx.x % Gb, split = blockIdx.y, nsplit = gridDim.y;
    const long long R = (long long)n * S;
    const long long per = (R + nsplit - 1) / nsplit;
    const long long rb = min(R, per * split), re = min(R, rb + per);
    double acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.0;
    for (long long r = rb + threadIdx.x; r < re; r += TS_THREADS) {
        const int s = (int)(r / S), p = (int)(r % S);
        const double *xp = X + (((size_t)s * (Ca / 4) + ga) * S + p) * 4;
        const double *dp = D + (((size_t)s * Gb + gb) * S + p) * 4;
        double xv[4], dv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) xv[j] = xp[j], dv[j] = dp[j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[4 * i + j] = fma(xv[i], dv[j], acc[4 * i + j]);
    }
    block_sum<16>(acc, sh);
    if (threadIdx.x == 0)
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j)
                partial[((size_t)split * Ca + 4 * ga + i) * Cb + 4 * gb + j] = sh[(4 * i + j) * TS_THREADS];
}

// Batch-statistics BatchNorm + ReLU backward, float64, blocked (patchnet.py:28,31 with affine = False: gamma = 1; the pool
// layer's, patch_embedder.py:32-39):
//   x^ = (z - mean) rstd, dz = dy [y > 0] with y the forward's ReLU output (bn_apply's fma(z, scale, shift): a mask
//   recomputed from x^ can round to the other sign near the boundary, so it is read from y, as torch's threshold_backward).
// First the per-channel sums sum dz, sum dz x^ (grid (C/4, BX_TS_SPLITS), partial [split][2C], then in split order),
// then dx = gamma rstd (dz - m1 - x^ m2) with m1, m2 those sums over N (one thread per element).
struct BnBwd {
    const double *mean, *rstd, *gamma;
};

__global__ void __launch_bounds__(TS_THREADS) bn_bwd_sums_kernel(const double *__restrict__ dy, const double *__restrict__ z,
                                                                 const double *__restrict__ y, BnBwd q, int n, int G, int S,
                                                                 double *__restrict__ partial) {
    __shared__ double sh[8 * TS_THREADS];
    const int g = blockIdx.x, split = blockIdx.y, nsplit = gridDim.y;
    double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    double mu[4], rs[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) mu[j] = q.mean[4 * g + j], rs[j] = q.rstd[4 * g + j];
    for (int s = split; s < n; s += nsplit) {
        const size_t base = ((size_t)s * G + g) * S * 4;
        for (int p = threadIdx.x; p < S; p += TS_THREADS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const double xh = (z[base + 4 * p + j] - mu[j]) * rs[j];
                const double dz = y[base + 4 * p + j] > 0.0 ? dy[base + 4 * p + j] : 0.0;
                v[j] += dz;
                v[4 + j] += dz * xh;
            }
        }
    }
    block_sum<8>(v, sh);
    if (threadIdx.x == 0) {
        const int C = 4 * G;
        double *o = partial + (size_t)split * 2 * C;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            o[4 * g + j] = sh[j * TS_THREADS];
            o[C + 4 * g + j] = sh[(4 + j) * TS_THREADS];
        }
    }
}

__global__ void bn_bwd_kernel(const double *__restrict__ dy, const double *__restrict__ z, const double *__restrict__ y, BnBwd q,
                              const double *__restrict__ sums, double N, long long total, int G, int S, double *__restrict__ dx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)((i / (4LL * S)) % G) * 4 + (int)(i & 3);
    const double xh = (z[i] - q.mean[c]) * q.rstd[c];
    const double dz = y[i] > 0.0 ? dy[i] : 0.0;
    dx[i] = q.gamma[c] * q.rstd[c] * (dz - sums[c] / N - xh * (sums[4 * G + c] / N));
}

// Attention pooling and the two L2 normalisations (patch_embedder.py:86-90), float64, one CTA per patch:
//   f[c] = mean_p x[c][p] w[p], desc = f / max(|f|, eps), equi[:, p] = x[:, p] / max(|x[:, p]|, eps).
// x blocked [K][8][140][4], w the attention map blocked [K][1][140][4] (channel 0); f [K][32] float64, desc fp32 [K][32],
// equi fp32 [K][32][140].
__global__ void __launch_bounds__(CYL_S) pool_fwd_kernel(const double *__restrict__ x, const double *__restrict__ w, double *__restrict__ f,
                                                         float *__restrict__ desc, float *__restrict__ equi) {
    __shared__ double ws[CYL_S];
    __shared__ double fs[32];
    const int k = blockIdx.x, p = threadIdx.x;
    const double *xk = x + (size_t)k * 32 * CYL_S;
    ws[p] = w[((size_t)k * CYL_S + p) * 4];
    double n2 = 0.0;
    for (int c = 0; c < 32; ++c) {
        const double v = xk[((c / 4) * CYL_S + p) * 4 + (c & 3)];
        n2 += v * v;
    }
    const double nx = fmax(sqrt(n2), NORM_EPS);
    for (int c = 0; c < 32; ++c) equi[((size_t)k * 32 + c) * CYL_S + p] = (float)(xk[((c / 4) * CYL_S + p) * 4 + (c & 3)] / nx);
    __syncthreads();
    if (p < 32) {
        double s = 0.0;
        for (int q = 0; q < CYL_S; ++q) s += xk[((p / 4) * CYL_S + q) * 4 + (p & 3)] * ws[q];
        s /= (double)CYL_S;
        fs[p] = s;
        f[(size_t)k * 32 + p] = s;
    }
    __syncthreads();
    if (p < 32) {
        double s2 = 0.0;
        for (int c = 0; c < 32; ++c) s2 += fs[c] * fs[c];
        desc[(size_t)k * 32 + p] = (float)(fs[p] / fmax(sqrt(s2), NORM_EPS));
    }
}

// backward of pool_fwd_kernel: ddesc [K][32], dequi [K][32][140] (fp32, upstream) -> dx blocked [K][8][140][4] (the equi
// path and the direct x w path) and dw blocked [K][1][140][4] (channel 0; channels 1-3 zero).  Normalisation backward:
// |v| >= eps: (g - y (y . g)) / |v|, else g / eps (torch's clamp_min, whose backward passes the gradient at equality).
__global__ void __launch_bounds__(CYL_S) pool_bwd_kernel(const double *__restrict__ x, const double *__restrict__ w, const double *__restrict__ f,
                                                         const float *__restrict__ ddesc, const float *__restrict__ dequi,
                                                         double *__restrict__ dx, double *__restrict__ dw) {
    __shared__ double df[32];
    const int k = blockIdx.x, p = threadIdx.x;
    const double *xk = x + (size_t)k * 32 * CYL_S;
    if (p == 0) {
        double n2 = 0.0, yg = 0.0;
        const double *fk = f + (size_t)k * 32;
        for (int c = 0; c < 32; ++c) n2 += fk[c] * fk[c];
        const double nf = sqrt(n2);
        const bool big = nf >= NORM_EPS;
        const double den = big ? nf : NORM_EPS;
        for (int c = 0; c < 32; ++c) yg += (fk[c] / den) * (double)ddesc[(size_t)k * 32 + c];
        for (int c = 0; c < 32; ++c) {
            const double g = ddesc[(size_t)k * 32 + c];
            df[c] = big ? (g - (fk[c] / den) * yg) / den : g / NORM_EPS;
        }
    }
    __syncthreads();
    double n2 = 0.0, yg = 0.0;
    for (int c = 0; c < 32; ++c) {
        const double v = xk[((c / 4) * CYL_S + p) * 4 + (c & 3)];
        n2 += v * v;
    }
    const double nx = sqrt(n2);
    const bool big = nx >= NORM_EPS;
    const double den = big ? nx : NORM_EPS;
    for (int c = 0; c < 32; ++c)
        yg += (xk[((c / 4) * CYL_S + p) * 4 + (c & 3)] / den) * (double)dequi[((size_t)k * 32 + c) * CYL_S + p];
    const double wp = w[((size_t)k * CYL_S + p) * 4];
    double dwp = 0.0;
    for (int c = 0; c < 32; ++c) {
        const size_t o = (((size_t)k * 8 + c / 4) * CYL_S + p) * 4 + (c & 3);
        const double v = xk[((c / 4) * CYL_S + p) * 4 + (c & 3)];
        const double g = dequi[((size_t)k * 32 + c) * CYL_S + p];
        const double de = big ? (g - (v / den) * yg) / den : g / NORM_EPS;
        dx[o] = de + df[c] * wp / (double)CYL_S;
        dwp += df[c] * v;
    }
    double *dwo = dw + ((size_t)k * CYL_S + p) * 4;
    dwo[0] = dwp / (double)CYL_S;
    dwo[1] = dwo[2] = dwo[3] = 0.0;
}

// EquiMatch backward (BUFFERX.py:72-86): cor[k][a] = sum_{c, e, l} s[k][c][e][(l - a) mod L] t[k][c][e][l]; from dcor
//   ds[k][c][e][m] = sum_a dcor[k][a] t[k][c][e][(m + a) mod L],  dt[k][c][e][l] = sum_a dcor[k][a] s[k][c][e][(l - a) mod L]
// in float64, stored fp32.  One thread per element of the maps [B][C*E][L].
__global__ void equi_match_bwd_kernel(const float *__restrict__ s, const float *__restrict__ t, const float *__restrict__ dcor, int B, int CE,
                                      int L, float *__restrict__ ds, float *__restrict__ dt) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * CE * L) return;
    const int l = (int)(i % L);
    const long long row = i / L;
    const int k = (int)(row / CE);
    const float *sr = s + row * L, *tr = t + row * L, *dc = dcor + (size_t)k * L;
    double as = 0.0, at = 0.0;
    for (int a = 0; a < L; ++a) {
        const double g = dc[a];
        int ip = l + a;
        if (ip >= L) ip -= L;
        int im = l - a;
        if (im < 0) im += L;
        as += g * (double)tr[ip];
        at += g * (double)sr[im];
    }
    ds[i] = (float)as;
    dt[i] = (float)at;
}

}  // namespace

static bool cyl_sizes_ok(int n, int Kc, int Nc, int Din) {
    return n >= 1 && Kc >= 16 && Kc % 16 == 0 && Nc >= 8 && Nc % 8 == 0 && Din >= 1 && Din <= 3;
}

BX_API int bx_td_cyl_forward(const double *x, const double *w, const double *b, int n, int Cin, int Cout, int Din, double *out,
                             void *stream) {
    BX_REQUIRE(cyl_sizes_ok(n, Cin, Cout, Din), "bx_td_cyl_forward: bad sizes (Cin %% 16, Cout %% 8, 1 <= Din <= 3)");
    BX_REQUIRE(x && w && b && out, "bx_td_cyl_forward: null pointer");
    dim3 grid(blocks_for((long long)n * CYL_S, CM_BM), (Cout + CM_BN - 1) / CM_BN);
    cyl_mma_kernel<false><<<grid, 128, 0, bx_stream(stream)>>>(x, w, b, n, Cin, Cout, Din, 0, CYL_S, 0, out);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_td_cyl_dgrad(const double *dy, const double *w, int n, int Cin, int Cout, int Din, double *dx, void *stream) {
    BX_REQUIRE(cyl_sizes_ok(n, Cout, Cin, Din), "bx_td_cyl_dgrad: bad sizes (Cin %% 8, Cout %% 16, 1 <= Din <= 3)");
    BX_REQUIRE(dy && w && dx, "bx_td_cyl_dgrad: null pointer");
    cudaStream_t st = bx_stream(stream);
    dim3 grid(blocks_for((long long)n * CYL_S, CM_BM), (Cin + CM_BN - 1) / CM_BN);
    for (int d = 0; d < Din; ++d) {
        cyl_mma_kernel<true><<<grid, 128, 0, st>>>(dy, w, nullptr, n, Cout, Cin, 1, d, Din * CYL_S, d * CYL_S, dx);
        BX_LAUNCH_CHECK();
    }
    return BX_OK;
}

BX_API int bx_td_cyl_wgrad(const double *x, const double *dy, int n, int Cin, int Cout, int Din, double *wpartial, double *dw,
                           void *stream) {
    BX_REQUIRE(n >= 1 && Cin >= 4 && Cin % 4 == 0 && Cout >= 8 && Cout % 8 == 0 && Din >= 1 && Din <= 3, "bx_td_cyl_wgrad: bad sizes");
    BX_REQUIRE(x && dy && wpartial && dw, "bx_td_cyl_wgrad: null pointer");
    cudaStream_t st = bx_stream(stream);
    dim3 grid(Din * 9 * ((Cin + 31) / 32) * ((Cout + 63) / 64), BX_TS_SPLITS);
    cyl_wgrad_kernel<<<grid, 128, 0, st>>>(x, dy, n, Cin, Cout, Din, wpartial);
    BX_LAUNCH_CHECK();
    const long long L = (long long)Din * 9 * Cin * Cout;
    sum_splits_kernel<<<blocks_for(L, 256), 256, 0, st>>>(wpartial, BX_TS_SPLITS, L, dw);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_td_pnt_forward(const float *inv, const double *W, const double *b, const double *scale, const double *shift, int K, int V,
                             int nv, double *feat, unsigned char *arg, void *stream) {
    BX_REQUIRE(K >= 1 && V >= 1 && nv >= 1 && nv <= 255, "bx_td_pnt_forward: bad sizes");
    BX_REQUIRE(inv && W && b && scale && shift && feat && arg, "bx_td_pnt_forward: null pointer");
    pnt_forward_kernel<<<blocks_for((long long)K * V, 128), 128, 0, bx_stream(stream)>>>(inv, W, b, scale, shift, K, V, nv, feat, arg);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_td_pnt_backward(const float *inv, const unsigned char *arg, const double *dfeat, const double *W, const double *b,
                              const double *mean, const double *rstd, const double *gamma, const double *scale, const double *shift,
                              const double *mo9, int K, int V, int nv, double *partial, double *out, void *stream) {
    BX_REQUIRE(K >= 1 && V >= 1 && nv >= 1 && nv <= 255, "bx_td_pnt_backward: bad sizes");
    BX_REQUIRE(inv && arg && dfeat && W && b && mean && rstd && gamma && scale && shift && mo9 && partial && out,
               "bx_td_pnt_backward: null pointer");
    cudaStream_t st = bx_stream(stream);
    pnt_bwd_sums_kernel<<<dim3(16, BX_TS_SPLITS), TS_THREADS, 0, st>>>(inv, arg, dfeat, W, b, mean, rstd, scale, shift, K, V, nv, partial);
    BX_LAUNCH_CHECK();
    pnt_bwd_final_kernel<<<1, 32, 0, st>>>(partial, BX_TS_SPLITS, mo9, (double)K * V * nv, W, b, mean, rstd, gamma, out);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

template <typename T>
static int conv1x1(const T *x, const T *w, const T *b, int n, int Cin, int Cout, int S, int accumulate, T *out, void *stream) {
    BX_REQUIRE(n >= 1 && Cin >= 4 && Cin % 4 == 0 && Cin <= 32 && Cout >= 4 && Cout % 4 == 0 && Cout <= 32 && S >= 1, "bx_ts_conv1x1: bad sizes");
    BX_REQUIRE(x && w && out, "bx_ts_conv1x1: null pointer");
    conv1x1_kernel<T><<<blocks_for((long long)n * S, 128), 128, 0, bx_stream(stream)>>>(x, w, b, n, Cin, Cout, S, accumulate, out);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_ts_conv1x1(const float *x, const float *w, const float *b, int n, int Cin, int Cout, int S, int accumulate, float *out,
                         void *stream) {
    return conv1x1<float>(x, w, b, n, Cin, Cout, S, accumulate, out, stream);
}

BX_API int bx_ts_conv1x1_f64(const double *x, const double *w, const double *b, int n, int Cin, int Cout, int S, int accumulate, double *out,
                             void *stream) {
    return conv1x1<double>(x, w, b, n, Cin, Cout, S, accumulate, out, stream);
}

BX_API int bx_td_cross_sums(const double *X, const double *D, int n, int Ca, int Cb, int S, double *partial, double *out, void *stream) {
    BX_REQUIRE(n >= 1 && Ca >= 4 && Ca % 4 == 0 && Cb >= 4 && Cb % 4 == 0 && S >= 1, "bx_td_cross_sums: bad sizes");
    BX_REQUIRE(X && D && partial && out, "bx_td_cross_sums: null pointer");
    cudaStream_t st = bx_stream(stream);
    cross_sums_kernel<<<dim3((Ca / 4) * (Cb / 4), BX_TS_SPLITS), TS_THREADS, 0, st>>>(X, D, n, Ca, Cb, S, partial);
    BX_LAUNCH_CHECK();
    sum_splits_kernel<<<blocks_for((long long)Ca * Cb, 256), 256, 0, st>>>(partial, BX_TS_SPLITS, (long long)Ca * Cb, out);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_ts_bn_backward(const double *dy, const double *z, const double *y, const double *mean, const double *rstd,
                             const double *gamma, int n, int C, int S, double *partial, double *sums, double *dx, void *stream) {
    BX_REQUIRE(n >= 1 && C >= 4 && C % 4 == 0 && S >= 1, "bx_ts_bn_backward: bad sizes");
    BX_REQUIRE(dy && z && y && mean && rstd && gamma && partial && sums && dx, "bx_ts_bn_backward: null pointer");
    cudaStream_t st = bx_stream(stream);
    BnBwd q{mean, rstd, gamma};
    bn_bwd_sums_kernel<<<dim3(C / 4, BX_TS_SPLITS), TS_THREADS, 0, st>>>(dy, z, y, q, n, C / 4, S, partial);
    BX_LAUNCH_CHECK();
    sum_splits_kernel<<<blocks_for(2 * C, 128), 128, 0, st>>>(partial, BX_TS_SPLITS, 2 * C, sums);
    BX_LAUNCH_CHECK();
    const long long total = (long long)n * C * S;
    bn_bwd_kernel<<<blocks_for(total, 256), 256, 0, st>>>(dy, z, y, q, sums, (double)n * S, total, C / 4, S, dx);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_td_pool_forward(const double *x, const double *w, int K, double *f, float *desc, float *equi, void *stream) {
    BX_REQUIRE(K >= 1 && x && w && f && desc && equi, "bx_td_pool_forward: bad arguments");
    pool_fwd_kernel<<<K, CYL_S, 0, bx_stream(stream)>>>(x, w, f, desc, equi);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_td_pool_backward(const double *x, const double *w, const double *f, const float *ddesc, const float *dequi, int K, double *dx,
                               double *dw, void *stream) {
    BX_REQUIRE(K >= 1 && x && w && f && ddesc && dequi && dx && dw, "bx_td_pool_backward: bad arguments");
    pool_bwd_kernel<<<K, CYL_S, 0, bx_stream(stream)>>>(x, w, f, ddesc, dequi, dx, dw);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_td_equi_match_backward(const float *s, const float *t, const float *dcor, int B, int C, int E, int L, float *ds, float *dt,
                                     void *stream) {
    BX_REQUIRE(B >= 1 && C >= 1 && E >= 1 && L >= 1, "bx_td_equi_match_backward: bad sizes");
    BX_REQUIRE(s && t && dcor && ds && dt, "bx_td_equi_match_backward: null pointer");
    const long long total = (long long)B * C * E * L;
    equi_match_bwd_kernel<<<blocks_for(total, 256), 256, 0, bx_stream(stream)>>>(s, t, dcor, B, C * E, L, ds, dt);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
