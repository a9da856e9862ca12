/*
 * bufferx_b200.h -- C-ABI of the H100-native (sm_90a) BUFFER-X per-pair registration hot path.
 *
 * Boundary contract
 *   - extern "C", plain pointers and sizes only.  Every pointer is a DEVICE pointer unless the
 *     parameter name starts with `h_`.  No ownership transfer: the caller allocates every input,
 *     output and workspace buffer (PyTorch does, in the host mirror buffer-x_b200/ops.py).
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Every call only
 *     ENQUEUES work; none synchronises the host.  Data-dependent sizes (number of mutual matches,
 *     consensus inliers, RANSAC early stop) live in device memory as int32 counters so that a
 *     whole pair can be enqueued without a host round trip.
 *   - Return value: 0 = ok, negative = error (BX_ERR_*); bx_last_error() gives the message for
 *     the calling thread.
 *   - Layouts are row-major, fp32 / int32 unless stated.
 *
 * Each entry point names the reference interface it replaces (paths relative to /root/reference;
 * third-party ops that the reference calls but does not vendor are named with their package).
 * The in-tree precedent for this ABI style is the reference's dead CPython modules
 * cpp_wrappers/cpp_neighbors/wrapper.cpp:58-239 and cpp_wrappers/cpp_subsampling/wrapper.cpp:631-859
 * (C-contiguous float32/int32 arrays in, arrays out, error on bad shapes).
 */
#ifndef BUFFERX_B200_H_
#define BUFFERX_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BX_OK 0
#define BX_ERR_INVALID_ARG (-1)
#define BX_ERR_CUDA (-2)
#define BX_ERR_UNSUPPORTED (-3)

#define BX_RADIUS_BINS 8192 /* candidate radii r_m = 5*m/8192 probed by the reference's bisection */
#define BX_RADIUS_SUBSAMPLE 200000 /* a larger cloud is histogrammed on this many drawn points (models/BUFFERX.py:664-665) */

/* ---- library ------------------------------------------------------------------------------ */
const char *bx_last_error(void);
int bx_version(void);          /* 10000*major + 100*minor + patch */
int bx_device_sm_count(void);  /* SM count of the current device (132 on an H100 SXM), <0 on error */
unsigned long long bx_launch_count(void); /* kernels launched by this library since it was loaded */

/* ---- a1: farthest point sampling ------------------------------------------------------------
 * Replaces pointnet2_ops.furthest_point_sample + gather_operation
 * (models/BUFFERX.py:286-290, 338-346).  B clouds stored back to back in `xyz` ([sum N,3]);
 * `h_offsets` (HOST, B+1 ints) gives each cloud's first point.  Starts at index 0, skips
 * candidates with |p|^2 <= 1e-3, tie rule of the upstream 512-thread block reduction.
 * One thread-block cluster per cloud; the cloud lives in registers across the cluster.
 * idx: [B,npoint] int32 (index inside the cloud); kpts: [B,npoint,3] (may be NULL).
 * Limit: N <= 131072 per cloud. */
int bx_fps(const float *xyz, const int32_t *h_offsets, int B, int npoint, int32_t *idx, float *kpts, void *stream);
/* With device-side point counts (size-class buffers: one captured launch serves every cloud up to a capacity).  h_offsets
 * give each cloud's first point and its CAPACITY (h_offsets[b+1] - h_offsets[b]); cloud b holds its first
 * n_b = min(max(d_counts[b], 1), capacity) points, and points beyond n_b are never read.  The launch configuration and
 * the grid follow the capacities; indices and key-points are those of bx_fps on the n_b-point clouds (the tie rule's
 * block size bs is derived from n_b).  d_counts NULL = bx_fps. */
int bx_fps_n(const float *xyz, const int32_t *h_offsets, int B, int npoint, int32_t *idx, float *kpts,
             const int32_t *d_counts, void *stream);
/* Size class of an n-point cloud: the largest point count that gets the same FPS launch configuration (register tier,
 * CTAs per cloud) as n -- the capacity whose buffers keep the kernel on n's tier.  0 for n <= 0, -1 above the
 * 524288-point limit. */
int bx_fps_size_class(int n);
/* One cloud of any size up to 1638400 points (models/BUFFERX.py:286-290 on the first-downsampled clouds of dense sensors,
 * which bx_fps refuses above 524288 points): xyz [n,3], idx [npoint] int32, kpts [npoint,3] (may be NULL).  Same result
 * contract as bx_fps, so any n gives bx_fps's indices.  The cloud is spread over ceil(n / 18432) SMs of one cooperative
 * grid (coordinates in shared memory, running distances in registers) that exchanges one candidate per SM and iteration
 * through global memory; capturable into a CUDA graph.  workspace: bx_fps_large_workspace_bytes(n) bytes, 16-byte aligned,
 * not shared with a launch in flight.  1638400 is the limit of the patch gatherer's shared-memory bitmap
 * (bx_select_patches_grid): a larger n is refused. */
int bx_fps_large(const float *xyz, int n, int npoint, int32_t *idx, float *kpts, void *workspace, void *stream);
long long bx_fps_large_workspace_bytes(int n);
/* Count form (size-class buffers): the grid is sized for the capacity cap (ceil(cap / 18432) CTAs) and the cloud is the first
 * n = min(max(*d_n, 1), cap) points of xyz; points beyond n are never read.  Indices and key-points are those of
 * bx_fps_large on the n-point cloud.  workspace: bx_fps_large_workspace_bytes(cap) bytes. */
int bx_fps_large_n(const float *xyz, int cap, const int32_t *d_n, int npoint, int32_t *idx, float *kpts, void *workspace,
                   void *stream);
/* Size class of an n-point cloud up to 1638400 points: bx_fps_size_class(n) up to 524288 points; above, the
 * capacities 18432 * {35, 43, 53, 66, 82} and 1638400 (bx_fps_large_n's grid), each at most 1.25x the smallest cloud of its
 * class.  0 for n <= 0, -1 above 1638400. */
int bx_fps_large_size_class(int n);

/* ---- a2: density-aware radius estimation ----------------------------------------------------
 * Replaces density_aware_radius_estimation + squared_cdist (models/BUFFERX.py:610-696) without
 * the [Kr,N] distance matrix and without host syncs: one pass builds the histogram of d2 over
 * the 8192 radii the bisection can probe, then the bisection runs on the device.
 * hist: [BX_RADIUS_BINS+2] uint32 workspace (zeroed by the call).
 * round_table: [BX_RADIUS_BINS+1] fp32, round(5*m/8192, 2) as computed by Python on the host.
 * thresholds: HOST array of n_thr percentages; out_r: [n_thr] fp32 radii; out_m: [n_thr] int32 (may be NULL).
 * denom = (original cloud size) * Kr as in the reference. */
int bx_radius_estimate(const float *kpts, int Kr, const float *pts, int N, int64_t denom,
                       const double *h_thresholds, int n_thr, double tolerance, const float *round_table,
                       uint32_t *hist, float *out_r, int32_t *out_m, void *stream);
/* Pair form with device-side point counts: both clouds (capacities cap_s, cap_t) and both key-point sets ([Kr,3] each);
 * d_counts [2] (device, required) = (ns, nt), clamped to the capacities.  The device picks the source iff ns > nt (the
 * reference's rule, models/BUFFERX.py:654) and uses denom = N * Kr of the chosen cloud; points beyond a count are never
 * read.  Same radii and m as bx_radius_estimate on the chosen exact cloud.  No sub-sampling: for a chosen cloud of more
 * than BX_RADIUS_SUBSAMPLE points use bx_radius_estimate_n_sub. */
int bx_radius_estimate_n(const float *kpts_s, const float *pts_s, int cap_s, const float *kpts_t, const float *pts_t, int cap_t,
                         int Kr, const int32_t *d_counts, const double *h_thresholds, int n_thr, double tolerance,
                         const float *round_table, uint32_t *hist, float *out_r, int32_t *out_m, void *stream);
/* The same with the reference's sub-sample: when the chosen cloud has N > BX_RADIUS_SUBSAMPLE points, the histogram runs
 * over its points d_sub[i], i < BX_RADIUS_SUBSAMPLE (device int32 indices, clamped to [0, N)), with denom = N * Kr; otherwise
 * d_sub is not read.  The draw sizes itself by N, which the caller knows on the host when it uploads the counts, so it is made
 * there (torch.randint(0, N, (200000,)) on torch's CPU generator, as the reference) and uploaded with them.  Same histogram,
 * radii and m as bx_radius_estimate on the gathered cloud pts[d_sub] with that denom. */
int bx_radius_estimate_n_sub(const float *kpts_s, const float *pts_s, int cap_s, const float *kpts_t, const float *pts_t, int cap_t,
                             int Kr, const int32_t *d_counts, const int32_t *d_sub, const double *h_thresholds, int n_thr,
                             double tolerance, const float *round_table, uint32_t *hist, float *out_r, int32_t *out_m, void *stream);

/* ---- a3: order-preserving radius-neighbour patch gathering ----------------------------------
 * Replaces MiniSpinNet.select_patches (models/patch_embedder.py:92-120) =
 * pointnet2_ops.ball_query + grouping_operation + the centre fix-up, and (as the GPU
 * counterpart) the reference's CPU radius search cpp_wrappers/cpp_neighbors.
 * bx_permute_cloud: out4[i] = (pts[perm[i]], 0) as float4 (perm may be NULL = identity).
 * bx_select_patches: for each key-point the FIRST P points of the permuted cloud (index order)
 * with d2 < r*r; r = *d_radius if d_radius != NULL else `radius`.
 * idx: [K,P] int32 raw ball-query indices (may be NULL); patches: [K,P,3]. */
int bx_permute_cloud(const float *pts, const int32_t *perm, int N, float *out4, void *stream);
/* With a device-side point count (d_N NULL = bx_permute_cloud): rows i < min(*d_N, N) are written, the others left
 * untouched; perm entries beyond the count are never read.  The grid is sized by the capacity N. */
int bx_permute_cloud_n(const float *pts, const int32_t *perm, int N, const int32_t *d_N, float *out4, void *stream);
int bx_select_patches(const float *pts4, int N, const float *kpts, int K, float radius, const float *d_radius,
                      int P, int32_t *idx, float *patches, void *stream);
/* The same for several (permuted cloud, key-point set, device radius) jobs in ONE launch (all 2 x num_scales jobs of a pair):
 * job j reads pts4[j] (N[j] points), kpts[j] (K[j] key-points), *d_radius[j]; its patches are rows
 * [sum_{i<j} K[i], ...) of `patches`.  The pointer arrays are HOST arrays of device pointers (<= 16 jobs). */
int bx_select_patches_batched(int njobs, const void *const *pts4, const int32_t *N, const void *const *kpts, const int32_t *K,
                              const void *const *d_radius, int P, float *patches, void *stream);
/* Hash-grid form for large clouds (N >= ~50 k points): the permuted cloud is binned into a spatial hash of cells of edge >=
 * radius, a key-point tests the cells around it only (27; up to 64 beyond ~2900 cells from the origin, the whole cloud
 * beyond 2^21 cells, so that fp32 rounding of the cell coordinates never loses a neighbour), hits set bits in a per-key-point bitmap over the point indices that
 * is read back in index order -- same contract and bit-identical output as bx_select_patches (device-side radius required).
 * workspace: bx_select_patches_grid_workspace_bytes(N) bytes, 16-byte aligned. */
int bx_select_patches_grid(const float *pts4, int N, const float *kpts, int K, const float *d_radius, int P, int32_t *idx,
                           float *patches, void *workspace, void *stream);
long long bx_select_patches_grid_workspace_bytes(int N);
/* All (cloud, scale) jobs of a pair through the hash grid, one launch per phase (arguments like bx_select_patches_batched;
 * workspace = the sum of bx_select_patches_grid_workspace_bytes(N[j]) bytes). */
int bx_select_patches_grid_batched(int njobs, const void *const *pts4, const int32_t *N, const void *const *kpts, const int32_t *K,
                                   const void *const *d_radius, int P, float *patches, void *workspace, void *stream);
/* Device-side key-point counts (early-exit pairs: the later scales' work is sized on the device).  d_K: host array of njobs
 * device int32 pointers (an entry or the array may be NULL = no count).  Job j processes its first min(*d_K[j], K[j])
 * key-points; the patch rows of the others are left untouched.  In the grid form a job whose count is 0 also skips its
 * binning phases (count, scan, scatter).  Otherwise identical to the calls above (which pass NULL). */
int bx_select_patches_batched_n(int njobs, const void *const *pts4, const int32_t *N, const void *const *kpts, const int32_t *K,
                                const void *const *d_radius, const void *const *d_K, int P, float *patches, void *stream);
int bx_select_patches_grid_batched_n(int njobs, const void *const *pts4, const int32_t *N, const void *const *kpts, const int32_t *K,
                                     const void *const *d_radius, const void *const *d_K, int P, float *patches, void *workspace,
                                     void *stream);
/* Device-side point counts as well (size-class buffers).  N[j] is job j's CAPACITY; d_N: host array of njobs device int32
 * pointers (an entry or the array may be NULL = no count): job j's permuted cloud holds min(max(*d_N[j], 1), N[j]) points
 * and points beyond that are never read.  Grids, the grid form's workspace (bx_select_patches_grid_workspace_bytes(N[j])
 * per job) and its shared-memory bitmap are sized by the capacities.  Output is bit-identical to the calls above on the
 * exact clouds; d_N NULL = the _n calls above. */
int bx_select_patches_batched_counts(int njobs, const void *const *pts4, const int32_t *N, const void *const *d_N, const void *const *kpts,
                                     const int32_t *K, const void *const *d_radius, const void *const *d_K, int P, float *patches,
                                     void *stream);
int bx_select_patches_grid_batched_counts(int njobs, const void *const *pts4, const int32_t *N, const void *const *d_N,
                                          const void *const *kpts, const int32_t *K, const void *const *d_radius,
                                          const void *const *d_K, int P, float *patches, void *workspace, void *stream);

/* Plain ordered ball query (pointnet2_ops.ball_query; utils/common.py:442): xyz [n,3] packed. */
int bx_ball_query(const float *xyz, int n, const float *qry, int m, float radius, int nsample, int32_t *idx,
                  void *stream);
/* The same over B clouds of n points each (pointnet2_ops.ball_query as the reference calls it: models/patch_embedder.py:99
 * with B = 1 and one large cloud, utils/common.py:62,442 sphere_query with B = K patches of 512 points): xyz [B,n,3],
 * qry [B,m,3], idx [B,m,nsample]; row j of cloud b holds the first nsample indices i (index order) with
 * ((dx*dx)+(dy*dy))+(dz*dz) < radius*radius, padded with the first hit, all zero when nothing is hit.  Clouds of up to
 * 4096 points are staged in shared memory (one CTA per cloud when B is large, several when B is small); larger clouds are
 * scanned by one warp per query like bx_ball_query.  B <= 65535. */
int bx_ball_query_batched(const float *xyz, int B, int n, const float *qry, int m, float radius, int nsample, int32_t *idx,
                          void *stream);

/* ---- pointnet2 channel-first gathers ---------------------------------------------------------
 * Replace pointnet2_ops gather_operation (models/BUFFERX.py:289-290, 342-345) and grouping_operation
 * (models/patch_embedder.py:101, utils/common.py:64,453): out[b][c][k] = features[b][c][idx[b][k]], features [B,C,N],
 * idx [B,K] int32 (grouping: idx [B,M,S] with K = M*S, out [B,C,M,S]).  An index outside [0,N) gives NaN. */
int bx_gather_channels(const float *features, int B, int C, int N, const int32_t *idx, int K, float *out, void *stream);

/* ---- k = 1 nearest neighbour ----------------------------------------------------------------
 * Replaces knn_cuda.KNN(k=1, transpose_mode=True)(ref, query) (models/BUFFERX.py:481,486,511): for each of B problems,
 * every query row [Nq,D] finds the ref row [Nr,D] with the smallest d2 = sum over D in order, without FMA, of (q - r)^2
 * (the arithmetic of bx_mutual_nn); the first minimum in ref order wins.  ref [B,Nr,D], qry [B,Nq,D]; keys [B*Nq] uint64
 * workspace; dist [B,Nq] = sqrtf(d2), idx [B,Nq] int64.  Nr >= 1. */
int bx_knn1(const float *ref, int Nr, const float *qry, int Nq, int D, int B, unsigned long long *keys, float *dist,
            int64_t *idx, void *stream);

/* ---- batched 3x3 SVD ------------------------------------------------------------------------
 * Replaces torch_batch_svd.svd (utils/common.py:715, cal_Z_axis): A [B,3,3] -> U [B,3,3], S [B,3] descending,
 * V [B,3,3] with A = U diag(S) V^T.  One thread per matrix, fp64 one-sided Jacobi; general (non-symmetric, singular)
 * matrices; U and V orthonormal; singular-vector signs unspecified. */
int bx_svd3(const float *A, int B, float *U, float *S, float *V, void *stream);

/* ---- a4+a5: local reference frame + normalisation -------------------------------------------
 * Replaces MiniSpinNet.axis_align / normalize (models/patch_embedder.py:122-148, 167-170),
 * cal_Z_axis (utils/common.py:709-726, torch_batch_svd) and RodsRotatFormula (:501-525).
 * delta: [K,P,3]; Rt: [K,3,3] (the reference's returned "R"); rand_axis: [K,3].
 * flags: bit 0 = is_aligned_to_global_z (identity frame); bit 1 = well-conditioned Rodrigues (cos = z_z/|z|,
 * sin = |z x e_z|/|z|) instead of the reference's theta = acos(cos) -> sin(theta), cos(theta) (default, literal). */
int bx_lrf(const float *patches, int K, int P, float des_r, const float *d_des_r, int flags, float *delta,
           float *Rt, float *rand_axis, void *stream);
/* The same over the patches of several (cloud, scale) key-point sets in one launch: patch k uses the device radius
 * d_des_r[k / r_group] (r_group > 0; r_group == 0: d_des_r[0] / des_r like bx_lrf). */
int bx_lrf_batched(const float *patches, int K, int P, float des_r, const float *d_des_r, int r_group, int flags, float *delta,
                   float *Rt, float *rand_axis, void *stream);
/* With device-side counts: r_group > 0: d_K[g] per radius group g, patch k is processed iff k % r_group < d_K[k / r_group];
 * r_group == 0: iff k < *d_K.  Rows of the other patches (delta, Rt, rand_axis) are left untouched.  d_K NULL = bx_lrf_batched. */
int bx_lrf_batched_n(const float *patches, int K, int P, float des_r, const float *d_des_r, int r_group, const int32_t *d_K, int flags,
                     float *delta, float *Rt, float *rand_axis, void *stream);

/* ---- a6+a7: spherical-voxel transformer + point layer ---------------------------------------
 * Replaces MiniSpinNet.SPT (models/patch_embedder.py:150-165: get_voxel_coordinate,
 * sphere_query, var_to_invar of utils/common.py:422-498) fused with pnt_layer + max-pool
 * (patch_embedder.py:26-30, 73-77); the [K,420,10,3] tensor is never written.
 * voxels: [V,3] (V = rad_n*ele_n*azi_n, azimuth fastest); rot: [azi_n,2] (cos,sin of -a*2pi/azi_n);
 * w: [16,3], b: [16] = 1x1 conv with BatchNorm folded in.  feat: [K,4,V,4] (channel-blocked, the layout
 * bx_conv_layer_tc reads: element (c, v) at ((c/4)*V + v)*4 + c%4).
 * dbg_vidx [K,V,nv] / dbg_inv [K,V,nv,3] are optional parity taps (NULL in production). */
int bx_spt_pnt(const float *delta, int K, int P, const float *voxels, int V, int azi_n, const float *rot,
               float voxel_r, int nv, const float *w, const float *b, float *feat, int32_t *dbg_vidx,
               float *dbg_inv, void *stream);
/* Same computation; the features are written in the presplit padded fp16 format that bx_conv_layer_sd reads with bulk
 * copies: feat_sd [3 (radial slice = 16-channel chunk)][4 (split, kcore)][rows][8 x fp16], rows = bx_conv_sd_rows(K, 176),
 * zero rows and wrap columns included; V must be 3*7*20.  *d_flag |= 1 if a feature is outside fp16 range. */
int bx_spt_pnt_sd(const float *delta, int K, int P, const float *voxels, int V, int azi_n, const float *rot,
                  float voxel_r, int nv, const float *w, const float *b, void *feat_sd, long long rows, int32_t *d_flag,
                  void *stream);
/* With a device-side count (d_K NULL = bx_spt_pnt_sd): the first n = min(*d_K, K) patches are written, with the zero row
 * that follows patch n - 1 (as bx_conv_layer_sd writes the zero row of sample s + 1 for a live sample s); the rows of the
 * later patches are left untouched. */
int bx_spt_pnt_sd_n(const float *delta, int K, int P, const float *voxels, int V, int azi_n, const float *rot,
                    float voxel_r, int nv, const float *w, const float *b, void *feat_sd, long long rows, int32_t *d_flag,
                    const int32_t *d_K, void *stream);

/* ---- a8/a11: convolution stacks -------------------------------------------------------------
 * Every conv layer of Cylindrical_Net (models/patchnet.py:16-84, circular-azimuth / zero-elevation padding of
 * utils/common.py:265-310) and CostNet (models/patchnet.py:151-210, un-padded) is an implicit GEMM, rows = (sample,
 * output position), cols = Cout, K = taps*Cin, on bx_conv_layer_sd (production) or bx_conv_layer_tc (TF32 fall-back).
 * BatchNorm is folded into the weights.  geom: BX_GEOM_*; n = *d_n if d_n != NULL else n. */
#define BX_GEOM_CYL3D 0    /* in [C,3,7,20] -> out [C,7,20], taps 27 */
#define BX_GEOM_CYL2D 1    /* in [C,7,20]   -> out [C,7,20], taps 9  */
#define BX_GEOM_VALID3D 2  /* in [C,D,H,W]  -> out [C,D-kd+1,H-kh+1,W-kw+1] */
#define BX_GEOM_COSTAB 4   /* VALID3D 3x3x3 on [32,18,3,18] whose input is the first CostNet activation regenerated from
                              bx_costvol_ab's factors: relu(A[c][k][(l-n) mod 20] - B[c][k][l]); equi_s = A, equi_t = B
                              (channel-blocked [n][8][3*20][4] / [n][8][3*18][4]) (bx_conv_layer_tc only) */

/* Shifted-descriptor implicit GEMM, fp16-split operands.
 * The production kernel of the eight Cylindrical_Net layers (models/patchnet.py:16-84; padding utils/common.py:265-310)
 * and of the k = (3,1,3) layers of CostNet (models/patchnet.py:151-210).
 * geom = BX_GEOM_CYL3D (16 channels x 3 radial slices, k=3x3x3), BX_GEOM_CYL2D (k=3x3; circular azimuth / zero elevation
 * padding) or BX_GEOM_VALID3D (un-padded k=3x1x3 over a D x W raster, D and W given; output (D-2) x (W-2)).
 * Activations come in two formats, chosen per side:
 *   presplit = 0  fp32 channel-blocked: in [n,Cin/4,S_in,4], out [n,Cout/4,S_out,4];
 *   presplit = 1  the layer-to-layer format: fp16 images [C/16][split(hi,lo)][kcore(2)][rows][8], x = hi + lo * 2^-11, over
 *                 the GEMM row raster (cylindrical: 176 rows per sample = 8 x 22, one zero row + 7 elevations, 20 azimuths +
 *                 2 wrap columns, written by the producing kernel; valid: D*W rows per sample), rows =
 *                 bx_conv_sd_rows(n, rows per sample).  The consumer's operand tiles are plain cp.async.bulk copies.
 * n = sample capacity; *d_n (optional, device) = the number of samples actually present (match count).
 * w_sd: fp16 hi/lo weight image [chunk][tap][kcore][split][NT][8] (ops.conv_sd_weights; NT = bx_conv_tc_ntile(Cout)); for
 * Cout <= 32 it is [chunk][tap][kcore][P | Q][64][8] (hi / lo and zero / hi of 8 channels per 16-row group, see bx_conv_sd.cu);
 * bias fp32 [Cout].  An activation with |x| >= 65000 cannot be split into fp16 operands -> *d_flag |= 1 (d_flag may be
 * NULL) and the caller re-runs the stack with bx_conv_layer_tc. */
int bx_conv_layer_sd(int geom, const void *in, int in_presplit, const void *w_sd, const float *bias, void *out, int out_presplit,
                     int n, const int32_t *d_n, int Cin, int Cout, int D, int W, int relu, int32_t *d_flag, void *stream);
long long bx_conv_sd_rows(int n, int rows_per_sample);
/* The descriptor-stack layers (geom = BX_GEOM_CYL3D / BX_GEOM_CYL2D, presplit input) on the per-sample kernel
 * (bx_conv_ps.cu): same arguments, weight image and bytes written as bx_conv_layer_sd, bit-identical values.  A sample's
 * 152 live raster rows are one wgmma operand, so the 24 dead rows (y = 7) of every sample are never computed.  D, W
 * unused. */
int bx_conv_layer_ps(int geom, const void *in, int in_presplit, const void *w_sd, const float *bias, void *out, int out_presplit,
                     int n, const int32_t *d_n, int Cin, int Cout, int D, int W, int relu, int32_t *d_flag, void *stream);
/* The second CostNet layer (32 -> 64, k = 3x3x3 over relu(A - B) regenerated from the factor maps of bx_costvol_ab) as a
 * 96 -> 64, k = (3,1,3) convolution over the 18 x 18 (n, l) raster on the same kernel.  fa [n,8,60,4], fb [n,8,54,4] fp32;
 * w_sd: ops.conv_sd_weights_costab; out: fp32 [n,16,256,4] or presplit over the 16 x 16 raster (rows = bx_conv_sd_rows(n, 256)). */
int bx_conv_layer_sd_costab(const float *fa, const float *fb, const void *w_sd, const float *bias, void *out, int out_presplit, int n,
                            const int32_t *d_n, int relu, int32_t *d_flag, void *stream);

/* Tensor-core variant (wgmma .tf32, 3xTF32 split, fp32 accumulators in registers; same geometry
 * arguments).  Activations are CHANNEL-BLOCKED here: in [n][Cin/4][S_in][4], out [n][Cout/4][S_out][4] (a GEMM row
 * fetches its 16 input channels with four 16-byte loads that coalesce across the warp's 32 consecutive rows; the
 * epilogue stores the same way); Cout % 4 == 0; in, out, bias 16-byte aligned.  w_tc is the host-prepared operand image: for every stage it = chunk*T + tap (chunk = 16
 * input channels) the block [kstep(2)][split(2: hi,lo)][kunit(2)][n(NT)][4 floats], NT = bx_conv_tc_ntile(Cout),
 * rows n >= Cout zero, hi = round-to-nearest tf32 of the folded weight, lo = w - hi.  Cin % 16 == 0, Cout <= 128. */
int bx_conv_tc_ntile(int Cout);
/* Tuning knob: stages (16 channels x 1 tap) accumulated per tensor-core segment before the rounded fp32 add (default 4);
 * returns the previous value.  Used by tools/tc_precision.py. */
int bx_conv_tc_set_segment_stages(int stages);
int bx_conv_layer_tc(int geom, const float *in, const float *w_tc, const float *bias, float *out, int n,
                     const int32_t *d_n, int Cin, int Cout, int D, int H, int W, int kd, int kh, int kw, int relu,
                     const float *equi_s, const float *equi_t, void *stream);

/* Factorised first CostNet layer (models/patchnet.py:196 applied to the cost volume of models/BUFFERX.py:51-65):
 * the layer is linear before its ReLU, so out0[co][n][k][l] = relu(A[co][k][(l-n) mod 20] - B[co][k][l]) with
 * A/B small convolutions of the source/target equivariant maps (60 + 54 positions per match instead of 972).
 * wa: [32 c][3 dk][5 e][32 co] = sum over (dn,dl) with dl-dn = e-2 of the folded weight; wb: [32][3][3 dl][32] = sum
 * over dn; bias [32] is added into A.  A: [maxM][8][3*20][4], B: [maxM][8][3*18][4] (channel-blocked like the
 * activations of bx_conv_layer_tc; 16-byte aligned); rows >= *d_M untouched.  *d_M <= maxM is the caller's to keep:
 * the kernel does not clamp it. */
int bx_costvol_ab(const float *equi_s, const float *equi_t, const int32_t *s_mids, const int32_t *t_mids,
                  const int32_t *d_M, int maxM, const float *wa, const float *wb, const float *bias, float *A,
                  float *B, void *stream);

/* ---- a9: attention pooling + normalisation --------------------------------------------------
 * Replaces pool_layer / avg-pool / F.normalize (models/patch_embedder.py:32-39, 80-83).
 * x: [K,32,S], or channel-blocked [K,8,S,4] when channels_last != 0 (the layout bx_conv_layer_tc writes); w1 [32,16] (in-major),
 * b1 [16], w2 [16], b2 [1] (BatchNorm folded); desc: [K,32]; equi: [K,32,S] (always channel-first). */
int bx_pool_desc(const float *x, int K, int C, int S, int channels_last, const float *w1, const float *b1,
                 const float *w2, const float *b2, float *desc, float *equi, void *stream);
/* With a device-side count (d_K NULL = bx_pool_desc): rows k < min(*d_K, K) are written, the others left untouched. */
int bx_pool_desc_n(const float *x, int K, int C, int S, int channels_last, const float *w1, const float *b1,
                   const float *w2, const float *b2, float *desc, float *equi, const int32_t *d_K, void *stream);

/* ---- a10: mutual nearest-neighbour matching -------------------------------------------------
 * Replaces BufferX.mutual_matching (models/BUFFERX.py:469-496) -> knn_cuda.KNN(k=1) both ways.
 * keys: [Ka+Kb] uint64 workspace.  s_mids/t_mids: [Ka] int32 (ascending s); d_M: [1] int32;
 * snn [Ka] / tnn [Kb] optional. */
int bx_mutual_nn(const float *a, int Ka, const float *b, int Kb, int C, unsigned long long *keys, int32_t *s_mids,
                 int32_t *t_mids, int32_t *d_M, int32_t *snn, int32_t *tnn, void *stream);
/* With device-side counts on either side (NULL = no count; both NULL = bx_mutual_nn): matches the first min(*d_Ka, Ka)
 * rows of a against the first min(*d_Kb, Kb) rows of b, exactly as bx_mutual_nn on those rows.  A count of 0 on either
 * side writes *d_M = 0 and nothing else. */
int bx_mutual_nn_n(const float *a, int Ka, const float *b, int Kb, int C, const int32_t *d_Ka, const int32_t *d_Kb,
                   unsigned long long *keys, int32_t *s_mids, int32_t *t_mids, int32_t *d_M, int32_t *snn, int32_t *tnn,
                   void *stream);

/* Concatenate the S per-scale match lists (s_lists/t_lists: [S][stride] int32, counts d_counts[S] on the device)
 * into one list in scale order, adding the per-scale row offsets h_s_off/h_t_off[S] (host arrays) so the entries
 * index the batched descriptor buffers of a pair; d_offs[S+1] receives the prefix sums (d_offs[S] = total).
 * Lets CostNet and the hypothesis build of all scales run as one batch (same order as the reference's per-scale
 * torch.cat, models/BUFFERX.py:391-402). */
int bx_concat_matches(const int32_t *s_lists, const int32_t *t_lists, const int32_t *d_counts, int S, int stride,
                      const int32_t *h_s_off, const int32_t *h_t_off, int32_t *s_all, int32_t *t_all,
                      int32_t *d_offs, void *stream);

/* ---- a11 tail + a12: soft arg-max and pose hypotheses ---------------------------------------
 * Replaces softmax/expectation of CostVolume.forward (models/BUFFERX.py:66-69) and the hypothesis
 * build (:382-389, kornia axis_angle_to_rotation_matrix).  logits: [maxM, azi_n].
 * Appends M = *d_M rows at row offset *d_off of the accumulators and writes *d_off_out = off + M.  *d_M <= maxM is the
 * caller's to keep: the kernel does not clamp it. */
int bx_hypotheses(const float *logits, int azi_n, const float *kpts_s, const float *kpts_t, const float *Rt_s,
                  const float *Rt_t, const int32_t *s_mids, const int32_t *t_mids, const int32_t *d_M, int maxM,
                  const int32_t *d_off, int32_t *d_off_out, float *ind_out, float *R_acc, float *t_acc,
                  float *ss_acc, float *tt_acc, void *stream);

/* ---- a13: cross-scale consensus -------------------------------------------------------------
 * Replaces models/BUFFERX.py:404-417.  Mc = *d_Mc (<= maxMc).  counts: [maxMc] int32 workspace;
 * inlier_ind: [maxMc] int32 ascending; d_I: [1]; d_best: [1]. */
int bx_consensus(const float *ss, const float *tt, const float *R, const float *t, const int32_t *d_Mc, int maxMc,
                 int azi_n, float inlier_th, int32_t *counts, int32_t *inlier_ind, int32_t *d_I, int32_t *d_best,
                 void *stream);

/* ---- a14: RANSAC ----------------------------------------------------------------------------
 * Replaces PoseEstimator._estimate_ransac (models/pose_estimator.py:84-117) -> Open3D 0.18
 * registration_ransac_based_on_correspondence (3-point, EdgeLength + Distance checkers,
 * confidence early stop).  Sampling is an explicit function of (seed, iteration): Philox4x32-10.
 * workspace: bx_ransac_workspace_bytes(max_iter) bytes.  result: 16 doubles T (row-major 4x4)
 * followed by int32 {num_inliers, best_itr, iters_run, reserved} = 144 bytes. */
int64_t bx_ransac_workspace_bytes(int max_iter);
int bx_ransac(const float *ss, const float *tt, const int32_t *inlier_ind, const int32_t *d_I, int maxI,
              double dist_th, double similar_th, double confidence, int max_iter, uint64_t seed, void *workspace,
              void *result, void *stream);
/* Early-exit decision of a multi-scale pair (models/pose_estimator.py compute_confidence_score) on the device: the pair
 * stops after scale 0 when result->num_inliers >= min_inliers.  Writes d_counts[i] = 0 (stop) or h_caps[i] (continue) for
 * i < n (n <= 32; h_caps is a host array: the capacities the later scales' launches were sized for), and, if
 * d_scales_used != NULL, *d_scales_used = 1 (stop) or num_scales. */
int bx_early_exit_gate(const void *result, int min_inliers, int n, const int32_t *h_caps, int32_t *d_counts, int num_scales,
                       double *d_scales_used, void *stream);

/* ---- a15: post refinement -------------------------------------------------------------------
 * Replaces BufferX.post_refinement + rigid_transform_3d (models/BUFFERX.py:522-603).
 * T_in: 16 doubles (the RANSAC result) cast to fp32 like the reference; T_out: 16 fp32. */
int bx_refine(const float *ss, const float *tt, const int32_t *d_n, int maxn, const double *T_in, float dist_th,
              float *T_out, int32_t *d_rounds, void *stream);

/* ---- a17: batched fixed-radius neighbours (distance-sorted, padded) ---------------------------
 * Replaces radius_neighbors.batch_query (cpp_wrappers/cpp_neighbors/wrapper.cpp:58-239 ->
 * neighbors/neighbors.cpp:334-480 batch_nanoflanntbb_neighbors).  h_q_batches / h_s_batches: HOST arrays
 * (1..8 query batches, 1..2 support clouds; query batch b searches support cloud b % 2 like the reference).
 * out == NULL: counting pass (only *d_max_count is written).  Otherwise out is [nq, cap] int32, rows sorted by
 * (fp64 distance, index) and padded with ns; *d_max_count = largest true neighbour count.  The reference orders equal
 * distances by std::sort, which is not stable: its rows have the same distance sequence and, within each run of equal
 * distances, the same index set, but not necessarily the same order.  Balls of up to 4096 neighbours are sorted in shared
 * memory; cap > 4096 needs scratch_d [nq, cap] doubles + scratch_i [nq, cap] int32 (global rank sort of the large balls;
 * both may be NULL when cap <= 4096). */
int bx_radius_neighbors(const float *queries, int nq, const float *supports, int ns, const int32_t *h_q_batches, int nqb,
                        const int32_t *h_s_batches, int nsb, float radius, int32_t *out, int cap, int32_t *d_max_count,
                        double *scratch_d, int32_t *scratch_i, void *stream);

/* ---- a18: voxel-grid barycentre sub-sampling ------------------------------------------------
 * Replaces grid_subsampling.subsample (cpp_wrappers/cpp_subsampling/wrapper.cpp:631-859 ->
 * grid_subsampling/grid_subsampling.cpp:5-106, points only).  table_keys [table_cap] u64 and table_acc
 * [table_cap,4] f32 are workspaces (table_cap = power of two >= 2n), minmax6 a 6-float workspace.
 * keys_out [n] (reference cell id iX + NX*iY + NX*NY*iZ, u64 arithmetic), xyz_out [n,3], cnt_out [n] (may be NULL),
 * *d_m = cells.  The fp32 origin floor(min/dl)*dl can round above the minimum; the cell index -1 then wraps to 2^64-1
 * as in the reference's x86 build, so such points share the reference's (aliased) cell; NX and NY wrap the same way
 * (a flat axis below its rounded-up origin gives NX or NY = 0).
 * Cells are emitted in hash-table order (the reference emits in unordered_map order). */
int bx_grid_subsample(const float *pts, int n, float dl, unsigned long long *table_keys, float *table_acc, int table_cap,
                      float *minmax6, unsigned long long *keys_out, float *xyz_out, int32_t *cnt_out, int32_t *d_m,
                      void *stream);

/* ---- SURVEY 8(f) row 1: loader-side geometric bootstrapping ---------------------------------------
 * bx_pca_analysis replaces compute_pca_alignment (utils/tools.py:132-149) = sklearn PCA(n_components=3) of the
 * sampled points pts[sample_idx[0..n_sample)] (sample_idx NULL: all n points), fp64; n_sample >= 3, as sklearn
 * refuses fewer samples than components.  acc9: 9-double workspace.
 * out15: mean[3], explained variance[3] (descending), components[3][3] (rows; largest-magnitude entry positive).
 * bx_project_range: min / max over the whole cloud of (p - mean) . axis (mean_axis6 = mean[3], axis[3], on the
 * device) = the z-range of pca.transform (utils/tools.py:181-182).  work2: 2 x u64 workspace, out2: {min, max}.
 * bx_voxel_down_sample replaces open3d PointCloud.voxel_down_sample (Open3D 0.18; dataset/*.py, utils/tools.py:
 * 218-219): voxel_min_bound = min - voxel/2, index = floor((p - voxel_min_bound)/voxel) in fp64, output = mean of the
 * points of a voxel.  table_keys [table_cap] u64, table_acc [table_cap,4] f64 (table_cap = power of two >= 2n) and
 * minmax6 [6] u64 are workspaces; keys_out [n] = ix | iy << 21 | iz << 42, xyz_out [n,3], cnt_out [n] (may be NULL),
 * *d_m = voxels.  Emitted in hash-table order (Open3D: unordered_map order).  Keys are distinct only while every
 * axis spans fewer than 2^21 voxels: the caller reads minmax6 (min xyz, max xyz, order-preserving u64 encoding of
 * the doubles) with *d_m and refuses floor((max - voxel_min_bound)/voxel) >= 2^21, as ops.voxel_down_sample does. */
int bx_pca_analysis(const float *pts, int n, const int32_t *sample_idx, int n_sample, double *acc9, double *out15,
                    void *stream);
int bx_project_range(const float *pts, int n, const double *mean_axis6, unsigned long long *work2, double *out2,
                     void *stream);
int bx_voxel_down_sample(const float *pts, int n, double voxel, unsigned long long *table_keys, double *table_acc,
                         int table_cap, unsigned long long *minmax6, unsigned long long *keys_out, float *xyz_out,
                         int32_t *cnt_out, int32_t *d_m, void *stream);

/* ---- SURVEY 8(f) row 3: the training stages' validation forward (cfg.stage "Desc" / "Pose", eval mode) ----------
 * bx_gt_matches replaces BufferX.get_matching_indices (models/BUFFERX.py:498-520): every source point is moved by the
 * row-major 4x4 T (utils/SE3.transform, each row ((r0*x + r1*y) + r2*z) + t), its nearest target point is found by a
 * brute-force scan (knn_cuda k = 1: the first minimum in target order wins ties) and [i, nn(i)] is kept when
 * sqrt(d2) < voxel.  nn_ws [N] int32 workspace; pairs [N,2] int32 in source order; *d_count = pairs kept.
 * bx_so2_augment is the SO(2) augmentation of MiniSpinNet.forward (models/patch_embedder.py:54-67): patch k of delta
 * [K,P,3] and rand_axis [K,3] are rotated in place by the kornia axis-angle matrix of (0, 0, angles[k]); aug_R [K,3,3]
 * (may be NULL) receives the rotations.
 * bx_equi_match is EquiMatch (models/BUFFERX.py:16-36): cor[b,a] = sum_{c,k,l} D1[b,c,k,(l-a) mod L] * D2[b,c,k,l] over
 * [B,C,K,L] maps (L <= 32, both maps of a patch in shared memory), fixed fp32 summation order.
 * bx_so2_gt is BufferX.cal_so2_gt (models/BUFFERX.py:86-126) on s_rand_axis [P,3], the LRFs s_R / t_R [P,3,3], the
 * ground-truth pose T [4,4] and optional aug_R [P,3,3]: exactly one of label_int [P] (rounded, azi_n -> 0) and
 * label_float [P] is written. */
int bx_gt_matches(const float *src, int N, const float *tgt, int M, const float *T, float voxel, int32_t *nn_ws,
                  int32_t *pairs, int32_t *d_count, void *stream);
int bx_so2_augment(float *delta, int K, int P, float *rand_axis, const float *angles, float *aug_R, void *stream);
int bx_equi_match(const float *D1, const float *D2, int B, int C, int K, int L, float *cor, void *stream);
int bx_so2_gt(const float *s_rand_axis, const float *s_R, const float *t_R, const float *T, const float *aug_R, int P,
              int azi_n, long long *label_int, float *label_float, void *stream);

/* ---- SURVEY 8(f) row 3: the Pose-stage training step (trainer.py:93-167 with cfg.stage "Pose", model.train()) -------
 * Activations are channel-blocked [n][C/4][S][4]: fp32 for the frozen descriptor network, float64 for CostNet (forward and
 * backward).  Every reduction over samples x positions writes BX_TS_SPLITS per-block partials (workspace `partial`) that
 * one thread per output then adds in split order in float64: no atomics, bit-identical across runs.
 * bx_ts_channel_sums(_f64): out [2C] float64 = sum x and sum x^2 per channel (the batch statistics of the BatchNorm
 *   layers in training mode, models/patchnet.py:28,31 and patch_embedder.py:26-39).  partial [BX_TS_SPLITS * 2C] float64.
 * bx_ts_moments3: the 3 first and 6 second moments (xx, xy, xz, yy, yz, zz) of R fp32 3-vectors, out9 float64, partial
 *   [BX_TS_SPLITS * 9]: the batch statistics of the linear 3 -> 16 point layer follow from them (patch_embedder.py:26-30).
 * bx_ts_bn_apply(_f64): y = z scale + shift per channel (ReLU if relu); y may alias z.
 * bx_ts_bn_backward: batch-statistics BatchNorm + ReLU backward, float64 (CostNet's and Cylindrical_Net's BatchNorms
 *   with affine = False, patchnet.py:28,31, pass gamma = 1; the pool layer's pool_layer.{1,4}): x^ = (z - mean) rstd,
 *   dz = dy [y > 0] with y the forward's ReLU output (bn_apply's, so the mask is the forward's bit for bit); sums [2C] =
 *   (sum dz, sum dz x^) (= dbeta, dgamma), dx = gamma rstd (dz - m1 - x^ m2) with m1, m2 the sums over n*S.  partial
 *   [BX_TS_SPLITS * 2C].
 * bx_ts_conv1x1(_f64): out (+= if accumulate) b + w^T x, fp32 or float64, for w [Cin][Cout], b [Cout] or NULL (the pool
 *   layer's 1x1 convolutions, patch_embedder.py:32-39, and their data gradients); Cin, Cout <= 32, multiples of 4.
 * bx_ts_costvol: the cost volume of CostVolume.forward (models/BUFFERX.py:52-64) on elevation rows 1..5 of the fp32 maps
 *   equi_s, equi_t [M,32,7,20]: cv float64 [M][8][20*5*20][4], cv[c][n][k][l] = s[c][k+1][(l-n) mod 20] - t[c][k+1][l].
 * bx_ts_softargmax: float64 ind [M] = sum_k softmax(logits)_k k (BUFFERX.py:66-68); with g = dL/dind [M] instead
 *   dlogits [M][L] = g p_k (k - ind).
 * bx_ts_conv_forward / bx_ts_conv_backward: a valid 3-D convolution of CostNet (models/patchnet.py:192-210) and its
 *   backward, float64 on CUDA cores, with input x [n][Cin/4][D*H*W][4], output [n][Cout/4][OD*OH*OW][4], weight w
 *   [kd*kh*kw][Cin][Cout] and bias b [Cout]; the backward gives dw [T][Cin][Cout] (wpartial [BX_TS_SPLITS * T*Cin*Cout]
 *   workspace) and, when dx is not NULL, dx shaped like x.  Cin % 32 == 0, Cout % 4 == 0. */
#define BX_TS_SPLITS 64
int bx_ts_splits(void);
int bx_ts_channel_sums(const float *x, int n, int C, int S, double *partial, double *out, void *stream);
int bx_ts_channel_sums_f64(const double *x, int n, int C, int S, double *partial, double *out, void *stream);
int bx_ts_moments3(const float *v3, long long R, double *partial, double *out9, void *stream);
int bx_ts_bn_apply(const float *z, const float *scale, const float *shift, int n, int C, int S, int relu, float *y, void *stream);
int bx_ts_bn_apply_f64(const double *z, const double *scale, const double *shift, int n, int C, int S, int relu, double *y, void *stream);
int bx_ts_bn_backward(const double *dy, const double *z, const double *y, const double *mean, const double *rstd, const double *gamma,
                      int n, int C, int S, double *partial, double *sums, double *dx, void *stream);
int bx_ts_conv1x1(const float *x, const float *w, const float *b, int n, int Cin, int Cout, int S, int accumulate, float *out,
                  void *stream);
int bx_ts_conv1x1_f64(const double *x, const double *w, const double *b, int n, int Cin, int Cout, int S, int accumulate, double *out,
                      void *stream);
int bx_ts_costvol(const float *equi_s, const float *equi_t, int M, double *cv, void *stream);
int bx_ts_softargmax(const double *logits, int M, int L, const double *g, double *ind, double *dlogits, void *stream);
int bx_ts_conv_forward(const double *x, const double *w, const double *b, int n, int Cin, int Cout, int D, int H, int W, int kd, int kh,
                       int kw, double *out, void *stream);
int bx_ts_conv_backward(const double *x, const double *dy, const double *w, int n, int Cin, int Cout, int D, int H, int W, int kd, int kh,
                        int kw, double *dx, double *wpartial, double *dw, void *stream);

/* ---- SURVEY 8(f) row 3: the Desc-stage training step (trainer.py:93-167 with cfg.stage "Desc", model.train()) -------
 * MiniSpinNet's forward with batch-statistics BatchNorm and its backward, float64 throughout (bx_train_desc.cu).  Images are
 * channel-blocked float64 [n][C/4][S][4]; a cylindrical raster has S = 140 (7 elevation x 20 azimuth) positions per depth
 * slice.  Reductions over samples x positions go through BX_TS_SPLITS partials (workspace `partial` / `wpartial`) added in
 * split order: bit-identical across runs.
 * bx_td_cyl_forward: one layer of Cylindrical_Net (models/patchnet.py:68-84) without its BatchNorm: the input padded
 *   circularly in azimuth and with zeros in elevation (utils/common.py:265-310), then a valid 3x3 (Din = 1) or 3x3x3
 *   (Din = 3, the depth collapsed) convolution.  x [n][Cin/4][Din*140][4], w [Din*9][Cin][Cout] (tap = (d, e, a) row-major),
 *   b [Cout] -> out [n][Cout/4][140][4].  Runs on the fp64 tensor-core MMA.  Cin % 16 == 0, Cout % 8 == 0.
 * bx_td_cyl_dgrad: its data gradient dx [n][Cin/4][Din*140][4] from dy [n][Cout/4][140][4] (replaces autograd through
 *   F.conv3d / F.conv2d of patchnet.py:68-84 and the padding of utils/common.py:265-310).  Cin % 8 == 0, Cout % 16 == 0.
 * bx_td_cyl_wgrad: its weight gradient dw [Din*9][Cin][Cout]; wpartial [BX_TS_SPLITS * Din*9*Cin*Cout].  The bias
 *   gradient is bx_ts_channel_sums_f64 of dy.
 * bx_td_pnt_forward: the point layer in training mode (patch_embedder.py:78-90: pnt_layer = 1x1 conv 3 -> 16, affine
 *   BatchNorm, ReLU, then max_pool2d over the nv samples): inv [K][V][nv][3] fp32 (the de-rotated samples, zero slots
 *   included), W [16][3], b [16], the BatchNorm as x^ = y scale + shift [16] -> feat [K][4][V][4] and arg [K][16][V] (the
 *   first maximal sample).
 * bx_td_pnt_backward: its backward from dfeat (shaped like feat): one pass over the K*16*V selected samples gives sum dz,
 *   sum dz x^ and sum dz inv; the dense sums over every sample follow from mo9 (bx_ts_moments3 of inv).  mean, rstd, gamma
 *   [16] are the batch statistics and BatchNorm weight, scale / shift as in the forward.  out [16][6] = dW[c][0..2], db[c],
 *   dgamma[c], dbeta[c]; partial [BX_TS_SPLITS * 80].
 * bx_td_cross_sums: out [Ca][Cb] = sum over (s, p) of X[s][a][p] D[s][b][p] (a 1x1 convolution's weight gradient);
 *   partial [BX_TS_SPLITS * Ca*Cb].
 * bx_td_pool_forward / bx_td_pool_backward: attention pooling and the L2 normalisations (patch_embedder.py:86-90):
 *   x [K][8][140][4], w the attention [K][1][140][4] (channel 0) -> f [K][32] float64, desc [K][32] and equi [K][32][140]
 *   fp32 (v / max(|v|, 1e-12)); the backward from ddesc, dequi (fp32) gives dx like x and dw like w.
 * bx_td_equi_match_backward: the gradients ds, dt [B][C][E][L] (fp32, float64 accumulation) of bx_equi_match's
 *   cor[b][a] = sum s[b][c][e][(l - a) mod L] t[b][c][e][l] (EquiMatch, models/BUFFERX.py:72-86) from dcor [B][L]. */
int bx_td_cyl_forward(const double *x, const double *w, const double *b, int n, int Cin, int Cout, int Din, double *out, void *stream);
int bx_td_cyl_dgrad(const double *dy, const double *w, int n, int Cin, int Cout, int Din, double *dx, void *stream);
int bx_td_cyl_wgrad(const double *x, const double *dy, int n, int Cin, int Cout, int Din, double *wpartial, double *dw, void *stream);
int bx_td_pnt_forward(const float *inv, const double *W, const double *b, const double *scale, const double *shift, int K, int V, int nv,
                      double *feat, unsigned char *arg, void *stream);
int bx_td_pnt_backward(const float *inv, const unsigned char *arg, const double *dfeat, const double *W, const double *b, const double *mean,
                       const double *rstd, const double *gamma, const double *scale, const double *shift, const double *mo9, int K, int V,
                       int nv, double *partial, double *out, void *stream);
int bx_td_cross_sums(const double *X, const double *D, int n, int Ca, int Cb, int S, double *partial, double *out, void *stream);
int bx_td_pool_forward(const double *x, const double *w, int K, double *f, float *desc, float *equi, void *stream);
int bx_td_pool_backward(const double *x, const double *w, const double *f, const float *ddesc, const float *dequi, int K, double *dx,
                        double *dw, void *stream);
int bx_td_equi_match_backward(const float *s, const float *t, const float *dcor, int B, int C, int E, int L, float *ds, float *dt,
                              void *stream);

/* ---- sharded training: the cross-rank mean of one step (driver.train_sharded, DESIGN.md §8) -------------------------
 * gathered [W][n + 1] fp32 (row-major, device) holds one record per rank: n values (the trainable parameters' gradients,
 * then the BatchNorm buffers) followed by the rank's contribution flag.  With count = the number of rows whose flag is not
 * 0, out[i] = fl32((sum over those rows r, ascending, of (double) gathered[r][i]) / count) for i < n: the float64 sum starts
 * from the first contributing row (one contributor is the identity, bit for bit) and is neither reordered nor contracted;
 * NaN and inf propagate.  *count (device int32) is always written; out is not written when count = 0.  Every rank that
 * runs this on the same gathered matrix gets the same bits.  Refuses NULL pointers, W < 1 and n < 0 before any launch. */
int bx_dp_mean(const float *gathered, int W, long long n, float *out, int32_t *count, void *stream);

/* ---- loader-side ground truth: point-to-point ICP ---------------------------------------------------
 * Replaces open3d.pipelines.registration.registration_icp(source, target, r, init, TransformationEstimationPointToPoint(),
 * ICPConvergenceCriteria(...)) (Open3D 0.18), which the KITTI loader runs on the CPU to refine every pair's ground-truth
 * pose (dataset/kitti.py:95-102: the two raw scans, r = 0.20, init = I, max_iteration = 200).  Open3D's loop: evaluate
 * (nearest target with float64 d2 < r*r per source point; fitness = correspondences / n_src, inlier_rmse = sqrt(sum d2 /
 * correspondences), 0 without any), then up to max_iteration times: Umeyama update (with_scaling = false; the identity
 * without correspondences), transformation = update * transformation, source copy transformed by the update, re-evaluate,
 * stop when |d fitness| < relative_fitness and |d rmse| < relative_rmse.  Assumptions where Open3D defers to FLANN: the
 * radius test is strict and ties between equidistant targets go to the lowest target index.
 * src [n_src,3], tgt [n_tgt,3] and init [16] (row-major 4x4) are float64; n_src, n_tgt >= 1; r > 0 and finite.
 * corr [n_src] int32: each source point's target of the final evaluation, or -1.  result (8-byte aligned): 16 doubles T,
 * double fitness, double inlier_rmse, int32 {num_correspondences, iterations (updates applied), converged, reserved} =
 * 160 bytes.  workspace: bx_icp_workspace_bytes(n_src, n_tgt) bytes, 256-byte aligned.  All max_iteration steps are
 * enqueued at once; the steps after the stop return at once on the device. */
int64_t bx_icp_workspace_bytes(int n_src, int n_tgt);
int bx_icp(const double *src, int n_src, const double *tgt, int n_tgt, double max_correspondence_distance, const double *init,
           double relative_fitness, double relative_rmse, int max_iteration, int32_t *corr, void *result, void *workspace,
           void *stream);

#ifdef __cplusplus
}
#endif
#endif /* BUFFERX_B200_H_ */
