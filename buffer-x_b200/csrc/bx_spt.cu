// bx_spt.cu -- a6+a7: spherical-voxel point transformer fused with the point layer and its max-pool.
//
// Replaces MiniSpinNet.SPT (/root/reference/models/patch_embedder.py:150-165) = get_voxel_coordinate +
// sphere_query + var_to_invar (/root/reference/utils/common.py:422-498) and the 1x1 conv + BN + ReLU +
// max over the 10 samples (patch_embedder.py:26-30, 73-77).  The reference writes [K,420,10] indices,
// [K,420,10,3] points (75.6 MB at K=1500) and [K,16,420,10] activations (403 MB) to HBM per call; here
// one CTA owns a patch and only the [4,V,4] feature tile (channel-blocked) leaves the SM (26.9 KB/patch).
//
// The selection "first nv points, in index order, inside each voxel ball" is evaluated point-major instead of
// voxel-major (420 x 512 = 215 K distance tests per patch in the reference's ball query):
//   1. every non-zero point enumerates only the voxels that CAN contain it -- (shell, elevation) rows whose ring is
//      closer than rho to the point in the (planar radius, z) half plane, azimuth bins within asin(rho / R_c) of the
//      point's bin (all bins where the ring is closer than rho to the axis) -- runs the EXACT test on those (~50
//      instead of 420) and records hits in a per-voxel bitmap over the patch indices (atomicOr in shared memory).
//      The points are first counting-sorted by their nearest ring so that the 32 lanes of a warp need the same few
//      rows: the row loop is warp-uniform, rows no lane needs are skipped, and the azimuth window of a row has the
//      same length for every lane (no divergence);
//   2. the exact-zero points (the key-point copies that pad a patch, up to 80 % of it at the finest scale) are
//      one ballot mask that is OR-ed into every voxel whose ball contains the origin;
//   3. a thread per voxel walks its bitmap words in index order and keeps the first nv set bits;
//   4. a thread per (voxel, group of 4 channels) de-rotates the selected non-zero points once, applies the folded
//      3->16 affine map + ReLU and max-reduces (exact-zero points contribute relu(b) like a zeroed slot); one
//      coalesced 16-byte store in the channel-blocked layout.
// The candidate enumeration is conservative (slack 1e-3 on the bands, +1 azimuth bin), membership itself is
// the bit-exact test of oracle bxo_spt: d2 = ((qx-x)^2+(qy-y)^2)+(qz-z)^2 < r*r; slot 0 zeroed when its index
// is 0 (utils/common.py:447-449), padding slots zeroed; x' = x*c + y*(-s), y' = x*s + y*c.  -fmad=false.
#include <cuda_fp16.h>

#include "bx_common.cuh"

namespace {

constexpr int SPT_THREADS = 256;
constexpr int MAX_NV = 16;
constexpr int MAX_RE = 64;   // rad_n * ele_n rows of the voxel table

// SD = 1: the features leave the kernel in the presplit padded fp16 format of bx_conv_layer_sd (three radial slices = three
// 16-channel chunks over the 8 x 22 raster, zero rows and wrap columns included) instead of fp32 channel-blocked.
template <int SD>
__global__ void __launch_bounds__(SPT_THREADS)
spt_pnt_kernel(const float *__restrict__ delta, int K, int P, const float *__restrict__ voxels, int V, int azi_n,
               const float *__restrict__ rot, float voxel_r, int nv, const float *__restrict__ w,
               const float *__restrict__ b, float *__restrict__ feat, int *__restrict__ dbg_vidx,
               float *__restrict__ dbg_inv, long long sd_rows, int *__restrict__ sd_flag, const int *__restrict__ d_K) {
    extern __shared__ float smem[];
    // optional device-side count: patches at or beyond it are not touched (the whole CTA leaves before any barrier)
    const int Kn = d_K ? min(max(*d_K, 0), K) : K;
    if ((int)blockIdx.x >= Kn) return;
    const int NW = (P + 31) >> 5;
    float *px = smem;                                   // P
    float *py = px + P;                                 // P
    float *pz = py + P;                                 // P
    float *vx = pz + P;                                 // 3*V
    float *sw = vx + 3 * V;                             // 64 (w[16][3], b[16])
    float *srot = sw + 64;                              // 2*azi_n
    float *re_s = srot + 2 * azi_n;                     // MAX_RE: planar radius of the row's ring
    float *re_z = re_s + MAX_RE;                        // MAX_RE: c_z of the row
    int *re_h = reinterpret_cast<int *>(re_z + MAX_RE); // MAX_RE: azimuth half width (>= azi_n/2 means "all")
    unsigned *bitmap = reinterpret_cast<unsigned *>(re_h + MAX_RE);   // V*NW
    unsigned *zmask = bitmap + (size_t)V * NW;                         // NW
    unsigned short *sel = reinterpret_cast<unsigned short *>(zmask + NW);  // V*MAX_NV
    unsigned short *order = sel + (size_t)V * MAX_NV;                  // P: non-zero point indices, ring-sorted
    int *cell_cnt = reinterpret_cast<int *>(order + ((P + 1) & ~1));   // MAX_RE + 1
    unsigned short *snz = reinterpret_cast<unsigned short *>(cell_cnt + MAX_RE + 1);   // V: slots holding a non-zero point
    unsigned char *pkey = reinterpret_cast<unsigned char *>(snz + V);   // P: ring of a point, 0xFF = zero point
    unsigned char *scnt = pkey + P;                                     // V

    const int k = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31;
    const int n_re = V / azi_n;
    const float *dl = delta + (size_t)k * P * 3;
    for (int i = tid; i < 3 * P; i += SPT_THREADS) {
        const float v = dl[i];
        const int s = i / 3, c = i - 3 * s;
        (c == 0 ? px : (c == 1 ? py : pz))[s] = v;
    }
    for (int i = tid; i < 3 * V; i += SPT_THREADS) vx[i] = voxels[i];
    if (tid < 48) sw[tid] = w[tid];
    if (tid < 16) sw[48 + tid] = b[tid];
    for (int i = tid; i < 2 * azi_n; i += SPT_THREADS) srot[i] = rot[i];
    for (int i = tid; i < V * NW; i += SPT_THREADS) bitmap[i] = 0u;
    __syncthreads();

    const float r2 = voxel_r * voxel_r;
    const float slack = voxel_r + 1e-3f;
    const float slack2 = slack * slack;
    const float step = 6.283185307179586f / (float)azi_n;
    // ---- per (shell, elevation) row: |c|, c_z, azimuth half width ------------------------------------
    if (tid < n_re) {
        const float cx = vx[3 * (tid * azi_n)], cy = vx[3 * (tid * azi_n) + 1], cz = vx[3 * (tid * azi_n) + 2];
        const float Rc = sqrtf(cx * cx + cy * cy);
        re_s[tid] = Rc;                                 // the ring of the row in the (planar radius, z) half plane
        re_z[tid] = cz;
        int h = azi_n;  // all bins
        if (Rc > slack) h = (int)ceilf(asinf(fminf(1.0f, slack / Rc)) / step) + 1;
        re_h[tid] = h;
    }
    // ---- zero mask (exact zeros: the key-point copies) -----------------------------------------------
    for (int base = 0; base < NW * 32; base += SPT_THREADS) {
        const int i = base + tid;
        const bool z = (i < P) && (px[i] == 0.0f) && (py[i] == 0.0f) && (pz[i] == 0.0f);
        const unsigned m = __ballot_sync(BX_FULL, z);
        if (lane == 0 && (i >> 5) < NW) zmask[i >> 5] = m;
    }
    __syncthreads();
    // ---- 1. voxels whose ball contains the origin take every zero point --------------------------------
    for (int v = tid; v < V; v += SPT_THREADS) {
        const float qx = vx[3 * v], qy = vx[3 * v + 1], qz = vx[3 * v + 2];
        if (bx_d2(qx - 0.0f, qy - 0.0f, qz - 0.0f) < r2)
            for (int wd = 0; wd < NW; ++wd) bitmap[(size_t)v * NW + wd] = zmask[wd];
    }
    __syncthreads();
    // ---- 2. non-zero points: exact test on their candidate voxels --------------------------------------
    // 2a. counting sort of the points by their nearest (shell, elevation) ring in the (planar radius, z) half plane:
    //     the 32 points of a warp then share the few rows that can contain them, and rows no lane needs are skipped
    //     warp-wide.
    if (tid < MAX_RE) cell_cnt[tid] = 0;
    __syncthreads();
    for (int i = tid; i < P; i += SPT_THREADS) {
        unsigned char key = 0xFF;
        if (!((zmask[i >> 5] >> (i & 31)) & 1u)) {
            const float x = px[i], y = py[i], z = pz[i];
            const float rp = sqrtf(x * x + y * y);
            float best = 3.0e38f;
            int kb = 0;
            for (int re = 0; re < n_re; ++re) {
                const float dr = rp - re_s[re], dz = z - re_z[re];
                const float d = dr * dr + dz * dz;
                if (d < best) { best = d; kb = re; }
            }
            key = (unsigned char)kb;
            atomicAdd(&cell_cnt[kb], 1);
        }
        pkey[i] = key;
    }
    __syncthreads();
    if (tid == 0) {
        int acc = 0;
        for (int re = 0; re < n_re; ++re) { const int c = cell_cnt[re]; cell_cnt[re] = acc; acc += c; }
        cell_cnt[MAX_RE] = acc;   // number of non-zero points
    }
    __syncthreads();
    for (int i = tid; i < P; i += SPT_THREADS) {
        const unsigned char key = pkey[i];
        if (key != 0xFF) order[atomicAdd(&cell_cnt[key], 1)] = (unsigned short)i;
    }
    __syncthreads();
    // 2b. lane = point (ring-sorted); the row loop is warp-uniform and a row's azimuth window has the same length for
    //     every lane, so there is no divergence inside it.
    const int n_nz = cell_cnt[MAX_RE];
    for (int base = (tid & ~31); base < n_nz; base += SPT_THREADS) {
        const bool valid = base + lane < n_nz;
        const int i = valid ? order[base + lane] : 0;
        const float x = px[i], y = py[i], z = pz[i];
        const float rp = sqrtf(x * x + y * y);
        float al = atan2f(y, x);
        if (al < 0.0f) al += 6.283185307179586f;
        int ap = (int)floorf(al / step);
        ap = min(max(ap, 0), azi_n - 1);
        const unsigned bit = 1u << (i & 31);
        unsigned *bm = bitmap + (i >> 5);
        for (int re = 0; re < n_re; ++re) {
            // a voxel centre of the row is at least the in-plane distance to the row's ring away from the point
            const float dr = rp - re_s[re], dz = z - re_z[re];
            const bool act = valid && (dr * dr + dz * dz) < slack2;
            if (!__any_sync(BX_FULL, act)) continue;
            const int h = re_h[re];
            const bool all = 2 * h + 1 >= azi_n;
            const int cnt = all ? azi_n : 2 * h + 1;
            int a = all ? 0 : ap - h;
            a = a < 0 ? a + azi_n : a;
            const int vb = re * azi_n;
            for (int j = 0; j < cnt; ++j) {
                const int v = vb + a;
                if (act && bx_d2(vx[3 * v] - x, vx[3 * v + 1] - y, vx[3 * v + 2] - z) < r2) atomicOr(bm + (size_t)v * NW, bit);
                a = (a + 1 == azi_n) ? 0 : a + 1;
            }
        }
    }
    __syncthreads();
    // ---- 3. first nv set bits per voxel, in index order -------------------------------------------------
    for (int v = tid; v < V; v += SPT_THREADS) {
        int c = 0;
        for (int wd = 0; wd < NW && c < nv; ++wd) {
            unsigned m = bitmap[(size_t)v * NW + wd];
            while (m && c < nv) {
                const int bpos = __ffs(m) - 1;
                m &= m - 1;
                sel[(size_t)v * MAX_NV + c] = (unsigned short)(wd * 32 + bpos);
                ++c;
            }
        }
        scnt[v] = (unsigned char)c;
        // slots whose point is an exact zero (key-point copies) contribute relu(b) like a zeroed slot: the feature
        // pass only visits the others
        unsigned nzm = 0;
        for (int l = 0; l < c; ++l) {
            const int i = sel[(size_t)v * MAX_NV + l];
            if (!((zmask[i >> 5] >> (i & 31)) & 1u) && !(l == 0 && i == 0)) nzm |= 1u << l;
        }
        snz[v] = (unsigned short)nzm;
        if (dbg_vidx || dbg_inv) {
            const int first = c > 0 ? sel[(size_t)v * MAX_NV] : 0;
            const int a = v % azi_n;
            const float cs = srot[2 * a], sn = srot[2 * a + 1];
            for (int l = 0; l < nv; ++l) {
                const int i = (l < c) ? sel[(size_t)v * MAX_NV + l] : first;
                const size_t o = ((size_t)k * V + v) * nv + l;
                if (dbg_vidx) dbg_vidx[o] = i;
                if (dbg_inv) {
                    const bool live = (l < c) && !(l == 0 && first == 0);
                    float xr = 0.f, yr = 0.f, zr = 0.f;
                    if (live) {
                        xr = (px[i] * cs) + (py[i] * (-sn));
                        yr = (px[i] * sn) + (py[i] * cs);
                        zr = pz[i];
                    }
                    dbg_inv[3 * o] = xr; dbg_inv[3 * o + 1] = yr; dbg_inv[3 * o + 2] = zr;
                }
            }
        }
    }
    __syncthreads();
    // ---- 4. features in the channel-blocked layout [K][16/4][V][4] the tensor-core convolution reads: thread = (group
    //         of 4 channels, voxel); the selected non-zero points are de-rotated once per thread; one 16-byte store ----
    if (SD) {
        // thread = (kcore of 8 channels, voxel): one 16-byte hi and one 16-byte lo store (x = hi + lo * 2^-11, the split the
        // convolution's own loader would apply to the fp32 features -- bit-identical operands)
        uint4 *img = reinterpret_cast<uint4 *>(feat);
        float omax = 0.0f;
        for (int t = tid; t < 2 * V; t += SPT_THREADS) {
            const int h = t / V, v = t - h * V;
            float w0[8], w1[8], w2[8], bb[8], best[8];
            const int c = scnt[v];
            unsigned nzm = snz[v];
            const bool any_zero = (c < nv) || (__popc(nzm) < c);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const int ch = h * 8 + q;
                w0[q] = sw[3 * ch]; w1[q] = sw[3 * ch + 1]; w2[q] = sw[3 * ch + 2]; bb[q] = sw[48 + ch];
                best[q] = any_zero ? fmaxf(bb[q], 0.0f) : -INFINITY;
            }
            const int a = v % azi_n;
            const float cs = srot[2 * a], sn = srot[2 * a + 1];
            while (nzm) {
                const int l = __ffs(nzm) - 1;
                nzm &= nzm - 1;
                const int i = sel[(size_t)v * MAX_NV + l];
                const float x = px[i], y = py[i], z = pz[i];
                const float xr = (x * cs) + (y * (-sn));
                const float yr = (x * sn) + (y * cs);
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float val = (((w0[q] * xr) + (w1[q] * yr)) + (w2[q] * z)) + bb[q];
                    best[q] = fmaxf(best[q], fmaxf(val, 0.0f));
                }
            }
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const __half2 hh = __floats2half2_rn(best[2 * e], best[2 * e + 1]);
                const float2 hf = __half22float2(hh);
                const __half2 ll = __floats2half2_rn((best[2 * e] - hf.x) * 2048.0f, (best[2 * e + 1] - hf.y) * 2048.0f);
                hi[e] = *reinterpret_cast<const uint32_t *>(&hh);
                lo[e] = *reinterpret_cast<const uint32_t *>(&ll);
                omax = fmaxf(omax, fmaxf(fabsf(best[2 * e]), fabsf(best[2 * e + 1])));
            }
            const int r = v / (7 * 20), rem = v - r * 140, ey = rem / 20, ax = rem - ey * 20;
            uint4 *im = img + (size_t)(r * 4 + h) * sd_rows + (size_t)k * 176 + (ey + 1) * 22;
            const uint4 vh = make_uint4(hi[0], hi[1], hi[2], hi[3]), vl = make_uint4(lo[0], lo[1], lo[2], lo[3]);
            im[ax + 1] = vh;
            im[2 * sd_rows + ax + 1] = vl;
            if (ax == 19) { im[0] = vh; im[2 * sd_rows] = vl; }          // wrap column x' = 0
            if (ax == 0) { im[21] = vh; im[2 * sd_rows + 21] = vl; }     // wrap column x' = 21
        }
        // the zero row above this sample's first elevation (and, from the last sample, the one below its last)
        const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
        for (int t = tid; t < 12 * 22; t += SPT_THREADS) {
            const int im = t / 22, xp = t - im * 22;
            img[(size_t)im * sd_rows + (size_t)k * 176 + xp] = z4;
            if (k == Kn - 1) img[(size_t)im * sd_rows + (size_t)Kn * 176 + xp] = z4;
        }
        if (!(omax < 65000.0f) && sd_flag) atomicOr(sd_flag, 1);
        return;
    }
    float4 *out4 = reinterpret_cast<float4 *>(feat + (size_t)k * 16 * V);
    for (int t = tid; t < 4 * V; t += SPT_THREADS) {
        const int cg = t / V, v = t - cg * V;
        float w0[4], w1[4], w2[4], bb[4], best[4];
        const int c = scnt[v];
        unsigned nzm = snz[v];
        const bool any_zero = (c < nv) || (__popc(nzm) < c);     // padding slot, slot 0 with index 0, or an exact-zero point
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int ch = cg * 4 + q;
            w0[q] = sw[3 * ch]; w1[q] = sw[3 * ch + 1]; w2[q] = sw[3 * ch + 2]; bb[q] = sw[48 + ch];
            best[q] = any_zero ? fmaxf(bb[q], 0.0f) : -INFINITY;   // a zeroed slot contributes relu(bn(conv(0)))
        }
        const int a = v % azi_n;
        const float cs = srot[2 * a], sn = srot[2 * a + 1];
        while (nzm) {
            const int l = __ffs(nzm) - 1;
            nzm &= nzm - 1;
            const int i = sel[(size_t)v * MAX_NV + l];
            const float x = px[i], y = py[i], z = pz[i];
            const float xr = (x * cs) + (y * (-sn));
            const float yr = (x * sn) + (y * cs);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float val = (((w0[q] * xr) + (w1[q] * yr)) + (w2[q] * z)) + bb[q];
                best[q] = fmaxf(best[q], fmaxf(val, 0.0f));
            }
        }
        out4[t] = make_float4(best[0], best[1], best[2], best[3]);
    }
}

size_t spt_smem_bytes(int P, int V, int azi_n) {
    const int NW = (P + 31) >> 5;
    size_t bytes = sizeof(float) * (3 * (size_t)P + 3 * (size_t)V + 64 + 2 * (size_t)azi_n + 3 * MAX_RE);
    bytes += sizeof(unsigned) * ((size_t)V * NW + NW);
    bytes += sizeof(unsigned short) * ((size_t)V * MAX_NV + (size_t)((P + 1) & ~1) + (size_t)V);
    bytes += sizeof(int) * (MAX_RE + 1);
    bytes += (size_t)P + (size_t)V + 16;
    return bytes;
}

}  // namespace

BX_API int bx_spt_pnt(const float *delta, int K, int P, const float *voxels, int V, int azi_n, const float *rot,
                      float voxel_r, int nv, const float *w, const float *b, float *feat, int32_t *dbg_vidx,
                      float *dbg_inv, void *stream) {
    BX_REQUIRE(delta && voxels && rot && w && b && feat, "bx_spt_pnt: null pointer");
    BX_REQUIRE(K >= 0 && P >= 1 && P <= 65535 && V >= 1 && azi_n >= 1 && nv >= 1 && nv <= MAX_NV, "bx_spt_pnt: bad sizes");
    BX_REQUIRE(V % azi_n == 0 && V / azi_n <= MAX_RE, "bx_spt_pnt: V must be (rad_n*ele_n <= %d) * azi_n", MAX_RE);
    if (K == 0) return BX_OK;
    const size_t smem = spt_smem_bytes(P, V, azi_n);
    BX_REQUIRE(smem <= 200 * 1024, "bx_spt_pnt: P=%d V=%d needs %zu bytes of shared memory", P, V, smem);
    static BxPerDevice attr = {};
    if (bx_needs_attr(attr, smem))
        BX_CUDA(cudaFuncSetAttribute(spt_pnt_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    spt_pnt_kernel<0><<<K, SPT_THREADS, smem, bx_stream(stream)>>>(delta, K, P, voxels, V, azi_n, rot, voxel_r, nv, w, b,
                                                                feat, dbg_vidx, dbg_inv, 0, nullptr, nullptr);
    BX_LAUNCH_CHECK();
    return BX_OK;
}

BX_API int bx_spt_pnt_sd(const float *delta, int K, int P, const float *voxels, int V, int azi_n, const float *rot,
                         float voxel_r, int nv, const float *w, const float *b, void *feat_sd, long long rows, int32_t *d_flag,
                         void *stream) {
    return bx_spt_pnt_sd_n(delta, K, P, voxels, V, azi_n, rot, voxel_r, nv, w, b, feat_sd, rows, d_flag, nullptr, stream);
}

BX_API int bx_spt_pnt_sd_n(const float *delta, int K, int P, const float *voxels, int V, int azi_n, const float *rot,
                           float voxel_r, int nv, const float *w, const float *b, void *feat_sd, long long rows, int32_t *d_flag,
                           const int32_t *d_K, void *stream) {
    BX_REQUIRE(delta && voxels && rot && w && b && feat_sd, "bx_spt_pnt_sd: null pointer");
    BX_REQUIRE(K >= 0 && P >= 1 && P <= 65535 && nv >= 1 && nv <= MAX_NV, "bx_spt_pnt_sd: bad sizes");
    BX_REQUIRE(V == 420 && azi_n == 20, "bx_spt_pnt_sd: the presplit raster is 3 radial x 7 elevation x 20 azimuth voxels");
    BX_REQUIRE(rows >= (long long)K * 176 + 22 && (reinterpret_cast<uintptr_t>(feat_sd) & 15) == 0, "bx_spt_pnt_sd: image too small or misaligned");
    if (K == 0) return BX_OK;
    const size_t smem = spt_smem_bytes(P, V, azi_n);
    BX_REQUIRE(smem <= 200 * 1024, "bx_spt_pnt_sd: P=%d V=%d needs %zu bytes of shared memory", P, V, smem);
    static BxPerDevice attr = {};
    if (bx_needs_attr(attr, smem))
        BX_CUDA(cudaFuncSetAttribute(spt_pnt_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    spt_pnt_kernel<1><<<K, SPT_THREADS, smem, bx_stream(stream)>>>(delta, K, P, voxels, V, azi_n, rot, voxel_r, nv, w, b,
                                                                reinterpret_cast<float *>(feat_sd), nullptr, nullptr, rows, d_flag, d_K);
    BX_LAUNCH_CHECK();
    return BX_OK;
}
