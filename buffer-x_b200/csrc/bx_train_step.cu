// bx_train_step.cu -- the Pose-stage training step (reference trainer.py:93-167 with cfg.stage "Pose", model.train()):
// batch-statistics BatchNorm for the descriptor network and CostNet, and CostNet's backward pass.
//
// Activations are channel-blocked [n][C/4][S][4] (the layout bx_conv_layer_tc reads and writes).
// Descriptor network (frozen, forward only): fp32; its convolutions run on bx_conv_layer_tc with the unfolded weights (no
//   BatchNorm folded in, ReLU off), the kernels here reduce the batch statistics and normalise.
// CostNet (forward + backward): float64 on CUDA cores, from the cost volume of the fp32 maps to the gradients.  The
//   gradient of a lower layer passes through up to eight batch-statistics BatchNorm backwards, each of which can cancel
//   most of its input (dx = (dz - mean dz - x^ mean dz x^) / sigma); an fp32 evaluation of the chain (3xTF32 forward or
//   plain fp32 on CUDA cores alike) carries that cancellation into the weight gradients of the lower layers, a float64 one
//   does not.
// The channel sums and bn_apply serve the Desc step (bx_train_desc.cu) too; the BatchNorm backward and the 1x1
// convolution that both steps run are in bx_train_desc.cu, beside the pool layer's other kernels.
//
// Determinism: every reduction over samples x positions goes through the fixed-order split reductions of bx_splits.cuh;
// two runs on the same inputs give bit-identical statistics and gradients.
#include "bx_splits.cuh"

namespace {

// per-channel sum x and sum x^2 of a blocked image; grid (C/4, BX_TS_SPLITS); partial [split][2C]: sum x at [c], sum x^2
// at [C + c]
template <typename T>
__global__ void __launch_bounds__(TS_THREADS) chan_sums_kernel(const T *__restrict__ x, int n, int G, int S, double *__restrict__ partial) {
    __shared__ double sh[8 * TS_THREADS];
    const int g = blockIdx.x, split = blockIdx.y, nsplit = gridDim.y;
    double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = split; s < n; s += nsplit) {
        const T *xs = x + ((size_t)s * G + g) * S * 4;
        for (int p = threadIdx.x; p < S; p += TS_THREADS) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const double a = (double)xs[4 * p + j];
                v[j] += a;
                v[4 + j] += a * a;
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

// first and second moments of R 3-vectors: partial [split][9] = sum x, y, z, xx, xy, xz, yy, yz, zz
__global__ void __launch_bounds__(TS_THREADS) moments3_kernel(const float *__restrict__ v3, long long R, double *__restrict__ partial) {
    __shared__ double sh[9 * TS_THREADS];
    double v[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (long long r = (long long)blockIdx.x * TS_THREADS + threadIdx.x; r < R; r += (long long)gridDim.x * TS_THREADS) {
        const double a = v3[3 * r], b = v3[3 * r + 1], c = v3[3 * r + 2];
        v[0] += a; v[1] += b; v[2] += c;
        v[3] += a * a; v[4] += a * b; v[5] += a * c; v[6] += b * b; v[7] += b * c; v[8] += c * c;
    }
    block_sum<9>(v, sh);
    if (threadIdx.x == 0)
        for (int i = 0; i < 9; ++i) partial[(size_t)blockIdx.x * 9 + i] = sh[i * TS_THREADS];
}

// y = z * scale[c] + shift[c] (ReLU if relu), blocked, one element per thread; y may alias z
template <typename T>
__global__ void bn_apply_kernel(const T *__restrict__ z, const T *__restrict__ scale, const T *__restrict__ shift, long long total,
                                int G, int S, int relu, T *__restrict__ y) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)((i / (4LL * S)) % G) * 4 + (int)(i & 3);
    T r = z[i] * scale[c] + shift[c];
    if (relu) r = r > T(0) ? r : T(0);
    y[i] = r;
}

// cost volume of the reference's CostVolume.forward (models/BUFFERX.py:52-64) over elevation rows 1..5 of the full maps:
// cv[m][c][nn][k][l] = s[m][c][k + 1][(l - nn) mod 20] - t[m][c][k + 1][l] (float64: exact); s, t channel-first fp32
// [M,32,7,20]; cv blocked float64 [M][8][20 * 5 * 20][4]
__global__ void costvol_kernel(const float *__restrict__ es, const float *__restrict__ et, int M, double *__restrict__ cv) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // (m, g, pos, j)
    if (i >= (long long)M * 8 * 2000 * 4) return;
    const int j = (int)(i & 3), pos = (int)((i >> 2) % 2000), g = (int)((i >> 2) / 2000 % 8), m = (int)(i / 64000);
    const int nn = pos / 100, k = (pos / 20) % 5, l = pos % 20;
    const size_t base = ((size_t)m * 32 + 4 * g + j) * 140 + (k + 1) * 20;
    cv[i] = (double)es[base + (l - nn + 20) % 20] - (double)et[base + l];
}

// soft arg-max of the reference (BUFFERX.py:66-68), float64: ind = sum_k softmax(logits)_k k.  With g (dL/d ind) the backward
// dlogit_k = g p_k (k - ind) instead.  logits / dlogits [M][L] (the head's blocked output with one position)
__global__ void softargmax_kernel(const double *__restrict__ logits, int M, int L, const double *__restrict__ g, double *__restrict__ ind,
                                  double *__restrict__ dlogits) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const double *lg = logits + (size_t)m * L;
    double mx = lg[0];
    for (int k = 1; k < L; ++k) mx = fmax(mx, lg[k]);
    double se = 0.0, sk = 0.0;
    for (int k = 0; k < L; ++k) {
        const double e = exp(lg[k] - mx);
        se += e;
        sk += e * (double)k;
    }
    const double r = sk / se;
    if (g == nullptr) {
        ind[m] = r;
        return;
    }
    const double gm = g[m];
    for (int k = 0; k < L; ++k) dlogits[(size_t)m * L + k] = gm * (exp(lg[k] - mx) / se) * ((double)k - r);
}

struct ConvGeom {
    int D, H, W, kd, kh, kw, OD, OH, OW;
};

// The two row-major implicit GEMMs of a valid 3-D convolution over blocked float64 images, on CUDA cores:
//   FWD   out[s][co][op] = b[co] + sum_{t, ci} w[t][ci][co] x[s][ci][op + t]     rows (s, op), columns co, k = (t, ci)
//   !FWD  dx[s][ci][ip]  =          sum_{t, co} w[t][ci][co] dy[s][co][ip - t]   rows (s, ip), columns ci, k = (t, co)
// A 64-row x 32-column tile per CTA, k-chunks of 16 channels of one tap; each thread accumulates 2 rows x 4 columns.
// The k channel count is a multiple of 4 (zero-filled to the chunk); the column count a multiple of 4.
template <bool FWD>
__global__ void __launch_bounds__(TS_THREADS) conv_gemm_kernel(const double *__restrict__ in, const double *__restrict__ w,
                                                               const double *__restrict__ bias, int n, int Cin, int Cout, ConvGeom q,
                                                               double *__restrict__ out) {
    __shared__ double As[16][64];
    __shared__ double Bs[16][32];
    const int tid = threadIdx.x;
    const int S_in = q.D * q.H * q.W, S_out = q.OD * q.OH * q.OW;
    const int S_row = FWD ? S_out : S_in, S_a = FWD ? S_in : S_out;
    const int Kc = FWD ? Cin : Cout, Nc = FWD ? Cout : Cin;
    const long long rows = (long long)n * S_row;
    const long long r0 = (long long)blockIdx.x * 64;
    const int c0 = blockIdx.y * 32;
    const int cg = tid % 8, rp = tid / 8;
    const int lr = tid % 64, lcg = tid / 64;
    const long long grow = r0 + lr;
    const bool lvalid = grow < rows;
    int ls = 0, lz = 0, ly = 0, lx = 0;
    if (lvalid) {
        ls = (int)(grow / S_row);
        const int p = (int)(grow % S_row);
        const int HH = FWD ? q.OH : q.H, WW = FWD ? q.OW : q.W;
        lz = p / (HH * WW);
        ly = (p / WW) % HH;
        lx = p % WW;
    }
    const int Ga = Kc / 4;
    double acc[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
    const int T = q.kd * q.kh * q.kw;
    for (int t = 0; t < T; ++t) {
        const int dz = t / (q.kh * q.kw), dyy = (t / q.kw) % q.kh, dxx = t % q.kw;
        bool in_ok;
        int ap;
        if (FWD) {
            in_ok = lvalid;
            ap = ((lz + dz) * q.H + ly + dyy) * q.W + lx + dxx;
        } else {
            const int oz = lz - dz, oy = ly - dyy, ox = lx - dxx;
            in_ok = lvalid && oz >= 0 && oz < q.OD && oy >= 0 && oy < q.OH && ox >= 0 && ox < q.OW;
            ap = (oz * q.OH + oy) * q.OW + ox;
        }
        for (int k0 = 0; k0 < Kc; k0 += 16) {
            {
                const int ga = k0 / 4 + lcg;
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    As[lcg * 4 + j][lr] = (in_ok && ga < Ga) ? in[(((size_t)ls * Ga + ga) * S_a + ap) * 4 + j] : 0.0;
            }
            for (int e = tid; e < 16 * 32; e += TS_THREADS) {
                const int k = e / 32, c = e % 32;
                const int kk = k0 + k, cc = c0 + c;
                double v = 0.0;
                if (kk < Kc && cc < Nc) v = FWD ? w[((size_t)t * Cin + kk) * Cout + cc] : w[((size_t)t * Cin + cc) * Cout + kk];
                Bs[k][c] = v;
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const double a0 = As[k][2 * rp], a1 = As[k][2 * rp + 1];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const double b = Bs[k][4 * cg + j];
                    acc[0][j] = fma(a0, b, acc[0][j]);
                    acc[1][j] = fma(a1, b, acc[1][j]);
                }
            }
            __syncthreads();
        }
    }
    const int Gn = Nc / 4;
    const int cgo = c0 / 4 + cg;
    if (cgo >= Gn) return;
    for (int h = 0; h < 2; ++h) {
        const long long row = r0 + 2 * rp + h;
        if (row >= rows) continue;
        const int s = (int)(row / S_row), p = (int)(row % S_row);
        double *o = out + (((size_t)s * Gn + cgo) * S_row + p) * 4;
#pragma unroll
        for (int j = 0; j < 4; ++j) o[j] = acc[h][j] + (FWD ? bias[4 * cgo + j] : 0.0);
    }
}

// weight gradient of a valid 3-D convolution, blocked float64: dw[t][ci][co] = sum_{s, op} x[s][ci][op + t] dy[s][co][op].
// CTA = (tap, 32 input channels, 32 output channels) x one of BX_TS_SPLITS contiguous ranges of the (sample, position)
// rows; 4 row groups of 64 threads, each thread 4 x 4 outputs; the row groups are added in order and the CTA writes its
// partial [split][t][ci][co].  Cin % 32 == 0 and Cout % 4 == 0.
__global__ void __launch_bounds__(TS_THREADS) wgrad_kernel(const double *__restrict__ x, const double *__restrict__ dy, int n, int Cin,
                                                           int Cout, ConvGeom q, double *__restrict__ partial) {
    __shared__ double sm[2 * 64 * 32];                // Xs | Ds in the loop, then the 4 x 32 x 32 row-group sums
    double(*Xs)[32] = reinterpret_cast<double(*)[32]>(sm);
    double(*Ds)[32] = reinterpret_cast<double(*)[32]>(sm + 64 * 32);
    const int tid = threadIdx.x;
    const int nci = Cin / 32, nco = (Cout + 31) / 32;
    int b = blockIdx.x;
    const int cot = b % nco; b /= nco;
    const int cit = b % nci;
    const int t = b / nci;
    const int T = q.kd * q.kh * q.kw;
    const int dz = t / (q.kh * q.kw), dyy = (t / q.kw) % q.kh, dxx = t % q.kw;
    const int S_in = q.D * q.H * q.W, S_out = q.OD * q.OH * q.OW;
    const long long R = (long long)n * S_out;
    const long long per = (R + gridDim.y - 1) / gridDim.y;
    const long long rb = per * blockIdx.y, re = min(R, rb + per);
    const int Gi = Cin / 4, Go = Cout / 4;
    const int kg = tid / 64, lt = tid % 64, ti = lt / 8, tj = lt % 8;
    double acc[4][4] = {};
    for (long long c0 = rb; c0 < re; c0 += 64) {
        for (int e = tid; e < 64 * 32; e += TS_THREADS) {
            const int r = e / 32, c = e % 32;
            const long long row = c0 + r;
            double xv = 0.0, dv = 0.0;
            if (row < re) {
                const int s = (int)(row / S_out), op = (int)(row % S_out);
                const int oz = op / (q.OH * q.OW), oy = (op / q.OW) % q.OH, ox = op % q.OW;
                const int ip = ((oz + dz) * q.H + oy + dyy) * q.W + ox + dxx;
                xv = x[(((size_t)s * Gi + cit * 8 + c / 4) * S_in + ip) * 4 + (c & 3)];
                if (cot * 8 + c / 4 < Go) dv = dy[(((size_t)s * Go + cot * 8 + c / 4) * S_out + op) * 4 + (c & 3)];
            }
            Xs[r][c] = xv;
            Ds[r][c] = dv;
        }
        __syncthreads();
        for (int r = kg * 16; r < kg * 16 + 16; ++r) {
            double av[4], dv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) av[i] = Xs[r][4 * ti + i], dv[i] = Ds[r][4 * tj + i];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(av[i], dv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) sm[kg * 1024 + (4 * ti + i) * 32 + 4 * tj + j] = acc[i][j];
    __syncthreads();
    const size_t L = (size_t)T * Cin * Cout;
    for (int e = tid; e < 32 * 32; e += TS_THREADS) {
        const int i = e / 32, j = e % 32;
        const int co = cot * 32 + j;
        if (co >= Cout) continue;
        partial[(size_t)blockIdx.y * L + ((size_t)t * Cin + cit * 32 + i) * Cout + co] =
            ((sm[e] + sm[1024 + e]) + sm[2048 + e]) + sm[3072 + e];
    }
}

}  // namespace

BX_API int bx_ts_splits(void) { return BX_TS_SPLITS; }

template <typename T>
static int channel_sums(const T *x, int n, int C, int S, double *partial, double *out, void *stream) {
    BX_REQUIRE(n >= 1 && C >= 4 && C % 4 == 0 && S >= 1, "bx_ts_channel_sums: bad sizes");
    BX_REQUIRE(x && partial && out, "bx_ts_channel_sums: null pointer");
    cudaStream_t st = bx_stream(stream);
    chan_sums_kernel<T><<<dim3(C / 4, BX_TS_SPLITS), TS_THREADS, 0, st>>>(x, n, C / 4, S, partial);
    BX_LAUNCH_CHECK();
    sum_splits_kernel<<<blocks_for(2 * C, 128), 128, 0, st>>>(partial, BX_TS_SPLITS, 2 * C, out);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_ts_channel_sums(const float *x, int n, int C, int S, double *partial, double *out, void *stream) {
    return channel_sums<float>(x, n, C, S, partial, out, stream);
}

BX_API int bx_ts_channel_sums_f64(const double *x, int n, int C, int S, double *partial, double *out, void *stream) {
    return channel_sums<double>(x, n, C, S, partial, out, stream);
}

BX_API int bx_ts_moments3(const float *v3, long long R, double *partial, double *out9, void *stream) {
    BX_REQUIRE(R >= 1 && v3 && partial && out9, "bx_ts_moments3: bad arguments");
    cudaStream_t st = bx_stream(stream);
    moments3_kernel<<<BX_TS_SPLITS, TS_THREADS, 0, st>>>(v3, R, partial);
    BX_LAUNCH_CHECK();
    sum_splits_kernel<<<1, 32, 0, st>>>(partial, BX_TS_SPLITS, 9, out9);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

template <typename T>
static int bn_apply(const T *z, const T *scale, const T *shift, int n, int C, int S, int relu, T *y, void *stream) {
    BX_REQUIRE(n >= 1 && C % 4 == 0 && S >= 1 && z && scale && shift && y, "bx_ts_bn_apply: bad arguments");
    const long long total = (long long)n * C * S;
    bn_apply_kernel<T><<<blocks_for(total, 256), 256, 0, bx_stream(stream)>>>(z, scale, shift, total, C / 4, S, relu, y);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_ts_bn_apply(const float *z, const float *scale, const float *shift, int n, int C, int S, int relu, float *y, void *stream) {
    return bn_apply<float>(z, scale, shift, n, C, S, relu, y, stream);
}

BX_API int bx_ts_bn_apply_f64(const double *z, const double *scale, const double *shift, int n, int C, int S, int relu, double *y,
                              void *stream) {
    return bn_apply<double>(z, scale, shift, n, C, S, relu, y, stream);
}

BX_API int bx_ts_costvol(const float *equi_s, const float *equi_t, int M, double *cv, void *stream) {
    BX_REQUIRE(M >= 1 && equi_s && equi_t && cv, "bx_ts_costvol: bad arguments");
    costvol_kernel<<<blocks_for((long long)M * 64000, 256), 256, 0, bx_stream(stream)>>>(equi_s, equi_t, M, cv);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_ts_softargmax(const double *logits, int M, int L, const double *g, double *ind, double *dlogits, void *stream) {
    BX_REQUIRE(M >= 1 && L >= 1 && logits && (g ? dlogits != nullptr : ind != nullptr), "bx_ts_softargmax: bad arguments");
    softargmax_kernel<<<blocks_for(M, 128), 128, 0, bx_stream(stream)>>>(logits, M, L, g, ind, dlogits);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

static bool conv_sizes_ok(int n, int Cin, int Cout, int D, int H, int W, int kd, int kh, int kw) {
    return n >= 1 && Cin % 32 == 0 && Cout % 4 == 0 && Cout >= 4 && kd >= 1 && kh >= 1 && kw >= 1 && kd <= D && kh <= H && kw <= W;
}

BX_API int bx_ts_conv_forward(const double *x, const double *w, const double *b, int n, int Cin, int Cout, int D, int H, int W, int kd,
                              int kh, int kw, double *out, void *stream) {
    BX_REQUIRE(conv_sizes_ok(n, Cin, Cout, D, H, W, kd, kh, kw), "bx_ts_conv_forward: bad sizes");
    BX_REQUIRE(x && w && b && out, "bx_ts_conv_forward: null pointer");
    ConvGeom q{D, H, W, kd, kh, kw, D - kd + 1, H - kh + 1, W - kw + 1};
    dim3 grid(blocks_for((long long)n * q.OD * q.OH * q.OW, 64), (Cout + 31) / 32);
    conv_gemm_kernel<true><<<grid, TS_THREADS, 0, bx_stream(stream)>>>(x, w, b, n, Cin, Cout, q, out);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_ts_conv_backward(const double *x, const double *dy, const double *w, int n, int Cin, int Cout, int D, int H, int W, int kd,
                               int kh, int kw, double *dx, double *wpartial, double *dw, void *stream) {
    BX_REQUIRE(conv_sizes_ok(n, Cin, Cout, D, H, W, kd, kh, kw), "bx_ts_conv_backward: bad sizes");
    BX_REQUIRE(x && dy && wpartial && dw && (dx == nullptr || w != nullptr), "bx_ts_conv_backward: null pointer");
    cudaStream_t st = bx_stream(stream);
    ConvGeom q{D, H, W, kd, kh, kw, D - kd + 1, H - kh + 1, W - kw + 1};
    const int T = kd * kh * kw;
    dim3 wg(T * (Cin / 32) * ((Cout + 31) / 32), BX_TS_SPLITS);
    wgrad_kernel<<<wg, TS_THREADS, 0, st>>>(x, dy, n, Cin, Cout, q, wpartial);
    BX_LAUNCH_CHECK();
    const long long L = (long long)T * Cin * Cout;
    sum_splits_kernel<<<blocks_for(L, 256), 256, 0, st>>>(wpartial, BX_TS_SPLITS, L, dw);
    BX_LAUNCH_CHECK();
    if (dx) {
        dim3 dg(blocks_for((long long)n * D * H * W, 64), Cin / 32);
        conv_gemm_kernel<false><<<dg, TS_THREADS, 0, st>>>(dy, w, nullptr, n, Cin, Cout, q, dx);
        BX_LAUNCH_CHECK();
    }
    return BX_OK;
}
