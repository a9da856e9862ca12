"""Torch-tensor front end of the C-ABI library (``include/bufferx_b200.h``).

PyTorch is plumbing here: it owns device memory and the CUDA stream; every kernel lives in
``libbufferx_b200.so`` and is reached through ctypes with raw ``data_ptr()`` values -- no torch types
cross the boundary.  There is NO fallback: if the shared library is missing or a tensor is not on a
CUDA device the call raises.
"""
from __future__ import annotations

import ctypes
import math
import os
from ctypes import c_double, c_float, c_int, c_int64, c_uint64, c_void_p

import numpy as np
import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libbufferx_b200.so")

SYMBOLS = [
    "bx_last_error", "bx_version", "bx_device_sm_count", "bx_launch_count", "bx_fps", "bx_radius_estimate", "bx_permute_cloud",
    "bx_select_patches", "bx_ball_query", "bx_lrf", "bx_spt_pnt", "bx_conv_tc_ntile", "bx_conv_layer_tc",
    "bx_pool_desc", "bx_mutual_nn",
    "bx_hypotheses", "bx_consensus", "bx_ransac_workspace_bytes", "bx_ransac", "bx_refine", "bx_conv_tc_set_segment_stages",
    "bx_radius_neighbors", "bx_grid_subsample", "bx_costvol_ab", "bx_concat_matches",
    "bx_pca_analysis", "bx_project_range", "bx_voxel_down_sample", "bx_conv_layer_sd", "bx_conv_sd_rows", "bx_spt_pnt_sd", "bx_fps_set_sync_mode", "bx_conv_layer_sd_costab", "bx_lrf_batched", "bx_select_patches_batched", "bx_fps_ex", "bx_select_patches_grid", "bx_select_patches_grid_workspace_bytes", "bx_select_patches_grid_batched",
    "bx_gt_matches", "bx_so2_augment", "bx_equi_match", "bx_so2_gt",
    "bx_select_patches_batched_n", "bx_select_patches_grid_batched_n", "bx_lrf_batched_n", "bx_spt_pnt_sd_n", "bx_pool_desc_n",
    "bx_mutual_nn_n", "bx_early_exit_gate",
    "bx_fps_n", "bx_fps_size_class", "bx_radius_estimate_n", "bx_permute_cloud_n", "bx_select_patches_batched_counts",
    "bx_select_patches_grid_batched_counts",
    "bx_ball_query_batched", "bx_gather_channels", "bx_knn1", "bx_svd3", "bx_icp_workspace_bytes", "bx_icp",
    "bx_fps_large", "bx_fps_large_workspace_bytes", "bx_fps_large_n", "bx_fps_large_size_class", "bx_radius_estimate_n_sub",
    "bx_ts_splits", "bx_ts_channel_sums", "bx_ts_channel_sums_f64", "bx_ts_moments3", "bx_ts_bn_apply", "bx_ts_bn_apply_f64",
    "bx_ts_bn_backward", "bx_ts_conv1x1", "bx_ts_conv1x1_f64", "bx_ts_costvol", "bx_ts_softargmax", "bx_ts_conv_forward",
    "bx_ts_conv_backward", "bx_td_cyl_forward", "bx_td_cyl_dgrad", "bx_td_cyl_wgrad", "bx_td_pnt_forward", "bx_td_pnt_backward",
    "bx_td_cross_sums", "bx_td_pool_forward", "bx_td_pool_backward", "bx_td_equi_match_backward", "bx_dp_mean",
]

GEOM_CYL3D, GEOM_CYL2D, GEOM_VALID3D, GEOM_COSTAB = 0, 1, 2, 4
RADIUS_BINS = 8192

_lib = None


class BufferXError(RuntimeError):
    pass


def load_library():
    """Load the CUDA library; raises (never falls back) if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BufferXError(
            f"{LIB_PATH} not found: build it with `python buffer-x_b200/csrc/build.py` "
            "(or __graft_entry__.build()); bufferx_b200 has no CPU / eager fallback")
    lib = ctypes.CDLL(LIB_PATH)
    missing = [s for s in SYMBOLS if not hasattr(lib, s)]
    if missing:
        raise BufferXError(f"{LIB_PATH} lacks symbols {missing}")
    lib.bx_last_error.restype = ctypes.c_char_p
    lib.bx_launch_count.restype = ctypes.c_ulonglong
    lib.bx_ransac_workspace_bytes.restype = c_int64
    lib.bx_ransac_workspace_bytes.argtypes = [c_int]
    P = c_void_p
    lib.bx_fps.argtypes = [P, P, c_int, c_int, P, P, P]
    lib.bx_fps_ex.argtypes = [P, P, c_int, c_int, P, P, c_int, P]
    lib.bx_fps_n.argtypes = [P, P, c_int, c_int, P, P, c_int, P, P]
    lib.bx_fps_size_class.argtypes = [c_int, c_int]
    lib.bx_fps_large.argtypes = [P, c_int, c_int, P, P, P, P]
    lib.bx_fps_large_workspace_bytes.argtypes = [c_int]
    lib.bx_fps_large_workspace_bytes.restype = c_int64
    lib.bx_fps_large_n.argtypes = [P, c_int, P, c_int, P, P, P, P]
    lib.bx_fps_large_size_class.argtypes = [c_int, c_int]
    lib.bx_radius_estimate_n_sub.argtypes = [P, P, c_int, P, P, c_int, c_int, P, P, P, c_int, c_double, P, P, P, P, P]
    lib.bx_radius_estimate_n.argtypes = [P, P, c_int, P, P, c_int, c_int, P, P, c_int, c_double, P, P, P, P, P]
    lib.bx_permute_cloud_n.argtypes = [P, P, c_int, P, P, P]
    lib.bx_select_patches_batched_counts.argtypes = [c_int, P, P, P, P, P, P, P, c_int, P, P]
    lib.bx_select_patches_grid_batched_counts.argtypes = [c_int, P, P, P, P, P, P, P, c_int, P, P, P]
    lib.bx_radius_estimate.argtypes = [P, c_int, P, c_int, c_int64, P, c_int, c_double, P, P, P, P, P]
    lib.bx_permute_cloud.argtypes = [P, P, c_int, P, P]
    lib.bx_select_patches.argtypes = [P, c_int, P, c_int, c_float, P, c_int, P, P, P]
    lib.bx_select_patches_batched.argtypes = [c_int, P, P, P, P, P, c_int, P, P]
    lib.bx_select_patches_grid.argtypes = [P, c_int, P, c_int, P, c_int, P, P, P, P]
    lib.bx_select_patches_grid_workspace_bytes.argtypes = [c_int]
    lib.bx_select_patches_grid_batched.argtypes = [c_int, P, P, P, P, P, c_int, P, P, P]
    lib.bx_select_patches_batched_n.argtypes = [c_int, P, P, P, P, P, P, c_int, P, P]
    lib.bx_select_patches_grid_batched_n.argtypes = [c_int, P, P, P, P, P, P, c_int, P, P, P]
    lib.bx_select_patches_grid_workspace_bytes.restype = c_int64
    lib.bx_ball_query.argtypes = [P, c_int, P, c_int, c_float, c_int, P, P]
    lib.bx_ball_query_batched.argtypes = [P, c_int, c_int, P, c_int, c_float, c_int, P, P]
    lib.bx_gather_channels.argtypes = [P, c_int, c_int, c_int, P, c_int, P, P]
    lib.bx_knn1.argtypes = [P, c_int, P, c_int, c_int, c_int, P, P, P, P]
    lib.bx_svd3.argtypes = [P, c_int, P, P, P, P]
    lib.bx_lrf.argtypes = [P, c_int, c_int, c_float, P, c_int, P, P, P, P]
    lib.bx_lrf_batched.argtypes = [P, c_int, c_int, c_float, P, c_int, c_int, P, P, P, P]
    lib.bx_lrf_batched_n.argtypes = [P, c_int, c_int, c_float, P, c_int, P, c_int, P, P, P, P]
    lib.bx_spt_pnt.argtypes = [P, c_int, c_int, P, c_int, c_int, P, c_float, c_int, P, P, P, P, P, P]
    lib.bx_conv_layer_tc.argtypes = [c_int, P, P, P, P, c_int, P] + [c_int] * 9 + [P, P, P]
    lib.bx_conv_tc_ntile.argtypes = [c_int]
    lib.bx_conv_layer_sd.argtypes = [c_int, P, c_int, P, P, P, c_int, c_int, P, c_int, c_int, c_int, c_int, c_int, P, P, P]
    lib.bx_conv_sd_rows.argtypes = [c_int, c_int]
    lib.bx_conv_layer_sd_costab.argtypes = [P, P, P, P, P, c_int, c_int, P, c_int, P, P]
    lib.bx_fps_set_sync_mode.argtypes = [c_int]
    lib.bx_spt_pnt_sd.argtypes = [P, c_int, c_int, P, c_int, c_int, P, c_float, c_int, P, P, P, c_int64, P, P]
    lib.bx_spt_pnt_sd_n.argtypes = [P, c_int, c_int, P, c_int, c_int, P, c_float, c_int, P, P, P, c_int64, P, P, P]
    lib.bx_conv_sd_rows.restype = c_int64
    lib.bx_costvol_ab.argtypes = [P, P, P, P, P, c_int, P, P, P, P, P, P]
    lib.bx_concat_matches.argtypes = [P, P, P, c_int, c_int, P, P, P, P, P, P]
    lib.bx_pca_analysis.argtypes = [P, c_int, P, c_int, P, P, P]
    lib.bx_project_range.argtypes = [P, c_int, P, P, P, P]
    lib.bx_voxel_down_sample.argtypes = [P, c_int, ctypes.c_double, P, P, c_int, P, P, P, P, P, P]
    lib.bx_pool_desc.argtypes = [P, c_int, c_int, c_int, c_int, P, P, P, P, P, P, P]
    lib.bx_pool_desc_n.argtypes = [P, c_int, c_int, c_int, c_int, P, P, P, P, P, P, P, P]
    lib.bx_mutual_nn.argtypes = [P, c_int, P, c_int, c_int, P, P, P, P, P, P, P]
    lib.bx_mutual_nn_n.argtypes = [P, c_int, P, c_int, c_int, P, P, P, P, P, P, P, P, P]
    lib.bx_early_exit_gate.argtypes = [P, c_int, c_int, P, P, c_int, P, P]
    lib.bx_hypotheses.argtypes = [P, c_int, P, P, P, P, P, P, P, c_int, P, P, P, P, P, P, P, P]
    lib.bx_consensus.argtypes = [P, P, P, P, P, c_int, c_int, c_float, P, P, P, P, P]
    lib.bx_ransac.argtypes = [P, P, P, P, c_int, c_double, c_double, c_double, c_int, c_uint64, P, P, P]
    lib.bx_refine.argtypes = [P, P, P, c_int, P, c_float, P, P, P]
    lib.bx_radius_neighbors.argtypes = [P, c_int, P, c_int, P, c_int, P, c_int, c_float, P, c_int, P, P, P, P]
    lib.bx_grid_subsample.argtypes = [P, c_int, c_float, P, P, c_int, P, P, P, P, P, P]
    lib.bx_gt_matches.argtypes = [P, c_int, P, c_int, P, c_float, P, P, P, P]
    lib.bx_so2_augment.argtypes = [P, c_int, c_int, P, P, P, P]
    lib.bx_equi_match.argtypes = [P, P, c_int, c_int, c_int, c_int, P, P]
    lib.bx_so2_gt.argtypes = [P, P, P, P, P, c_int, c_int, P, P, P]
    lib.bx_icp_workspace_bytes.argtypes = [c_int, c_int]
    lib.bx_icp_workspace_bytes.restype = c_int64
    lib.bx_icp.argtypes = [P, c_int, P, c_int, c_double, P, c_double, c_double, c_int, P, P, P, P]
    lib.bx_ts_channel_sums.argtypes = [P, c_int, c_int, c_int, P, P, P]
    lib.bx_ts_channel_sums_f64.argtypes = [P, c_int, c_int, c_int, P, P, P]
    lib.bx_ts_bn_apply_f64.argtypes = [P, P, P, c_int, c_int, c_int, c_int, P, P]
    lib.bx_ts_conv_forward.argtypes = [P, P, P] + [c_int] * 9 + [P, P]
    lib.bx_ts_moments3.argtypes = [P, c_int64, P, P, P]
    lib.bx_ts_bn_apply.argtypes = [P, P, P, c_int, c_int, c_int, c_int, P, P]
    lib.bx_ts_bn_backward.argtypes = [P] * 6 + [c_int, c_int, c_int, P, P, P, P]
    lib.bx_ts_conv1x1.argtypes = [P, P, P, c_int, c_int, c_int, c_int, c_int, P, P]
    lib.bx_ts_conv1x1_f64.argtypes = [P, P, P, c_int, c_int, c_int, c_int, c_int, P, P]
    lib.bx_ts_costvol.argtypes = [P, P, c_int, P, P]
    lib.bx_ts_softargmax.argtypes = [P, c_int, c_int, P, P, P, P]
    lib.bx_ts_conv_backward.argtypes = [P, P, P] + [c_int] * 9 + [P, P, P, P]
    lib.bx_td_cyl_forward.argtypes = [P, P, P, c_int, c_int, c_int, c_int, P, P]
    lib.bx_td_cyl_dgrad.argtypes = [P, P, c_int, c_int, c_int, c_int, P, P]
    lib.bx_td_cyl_wgrad.argtypes = [P, P, c_int, c_int, c_int, c_int, P, P, P]
    lib.bx_td_pnt_forward.argtypes = [P, P, P, P, P, c_int, c_int, c_int, P, P, P]
    lib.bx_td_pnt_backward.argtypes = [P] * 11 + [c_int, c_int, c_int, P, P, P]
    lib.bx_td_cross_sums.argtypes = [P, P, c_int, c_int, c_int, c_int, P, P, P]
    lib.bx_td_pool_forward.argtypes = [P, P, c_int, P, P, P, P]
    lib.bx_td_pool_backward.argtypes = [P, P, P, P, P, c_int, P, P, P]
    lib.bx_td_equi_match_backward.argtypes = [P, P, P, c_int, c_int, c_int, c_int, P, P, P]
    lib.bx_dp_mean.argtypes = [P, c_int, ctypes.c_longlong, P, P, P]
    _lib = lib
    return lib


def _check(rc, what):
    if rc != 0:
        raise BufferXError(f"{what} failed ({rc}): {load_library().bx_last_error().decode()}")


def _dp(t, dtype=None, name="tensor"):
    """device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise BufferXError(f"{name}: expected a CUDA tensor (bufferx_b200 has no CPU path)")
    if dtype is not None and t.dtype != dtype:
        raise BufferXError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise BufferXError(f"{name}: tensor must be contiguous")
    if t.device.index != torch.cuda.current_device():
        # the C-ABI launches on the CURRENT device and stream: a tensor of another GPU would be dereferenced by a kernel
        # running on the wrong one.  BufferX.forward enters torch.cuda.device(model device) itself.
        raise BufferXError(f"{name}: tensor lives on {t.device} but the current CUDA device is cuda:{torch.cuda.current_device()}; "
                           "call under `with torch.cuda.device(tensor.device):`")
    return t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


F32, I32 = torch.float32, torch.int32


# --------------------------------------------------------------------------- #
def sm_count() -> int:
    return int(load_library().bx_device_sm_count())


def launch_count() -> int:
    """Kernels launched by libbufferx_b200.so since it was loaded (host-side counter)."""
    return int(load_library().bx_launch_count())


class Profiler:
    """Optional CUDA-event brackets around selected C-ABI calls (bench.py roofline figures).
    Events are recorded on the current stream -- the stream the kernels are launched on."""

    def __init__(self):
        self.spans = {}   # name -> list of (start_event, end_event, work)

    def span(self, name, work=0.0):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self.spans.setdefault(name, []).append((a, b, work))
        return a, b

    def summary(self):
        out = {}
        for name, lst in self.spans.items():
            ms = sum(a.elapsed_time(b) for a, b, _ in lst)
            out[name] = dict(launches=len(lst), ms=ms, work=sum(w for _, _, w in lst))
        return out


profiler = None  # set to a Profiler() to record spans


class _Span:
    """with _Span("name"): <C-ABI call>  -- no-op unless ops.profiler is set"""

    def __init__(self, name, work=0.0):
        self.ev = profiler.span(name, work) if profiler else None

    def __enter__(self):
        if self.ev:
            self.ev[0].record()

    def __exit__(self, *exc):
        if self.ev:
            self.ev[1].record()
        return False


def fps(xyz: torch.Tensor, offsets, npoint: int, want_kpts=True, max_cluster=0, d_counts=None):
    """xyz [sumN,3] f32 cuda; offsets: host sequence of B+1 ints.  Returns idx [B,npoint] i32, kpts [B,npoint,3].
    max_cluster 2 / 4: throughput form (fewer SMs per cloud, same indices).  d_counts: optional [B] int32 CUDA tensor of
    point counts; the offsets then give each cloud's capacity and cloud b is its first min(d_counts[b], capacity) points."""
    lib = load_library()
    off = np.ascontiguousarray(offsets, dtype=np.int32)
    B = len(off) - 1
    idx = torch.empty((B, npoint), dtype=I32, device=xyz.device)
    kp = torch.empty((B, npoint, 3), dtype=F32, device=xyz.device) if want_kpts else None
    with _Span("fps"):
        if d_counts is None:
            _check(lib.bx_fps_ex(_dp(xyz, F32, "xyz"), off.ctypes.data_as(c_void_p), B, npoint, _dp(idx), _dp(kp), int(max_cluster), _stream()), "bx_fps")
        else:
            assert d_counts.numel() >= B
            _check(lib.bx_fps_n(_dp(xyz, F32, "xyz"), off.ctypes.data_as(c_void_p), B, npoint, _dp(idx), _dp(kp), int(max_cluster),
                                _dp(d_counts, I32, "d_counts"), _stream()), "bx_fps_n")
    return idx, kp


FPS_MAX_POINTS = 524288          # bx_fps: one 16-CTA cluster's registers
FPS_LARGE_MAX_POINTS = 1638400   # bx_fps_large: the patch gatherer's shared-memory bitmap bounds every cloud of a pair


def fps_large(xyz: torch.Tensor, npoint: int, want_kpts=True, d_count=None):
    """One cloud xyz [N,3] f32 cuda, 1 <= N <= FPS_LARGE_MAX_POINTS, on the grid-wide kernel (bx_fps_large).  Returns idx
    [npoint] i32, kpts [npoint,3] (None unless want_kpts): for any N the indices ops.fps gives where it accepts N.
    d_count: optional 1-element int32 CUDA point count (bx_fps_large_n); xyz is then a capacity buffer, the grid is sized
    for its N rows and the cloud is its first min(max(d_count, 1), N) points."""
    if xyz.dim() != 2 or xyz.shape[1] != 3 or xyz.shape[0] < 1:
        raise BufferXError(f"fps_large: xyz must be [N,3] with N >= 1, got {tuple(xyz.shape)}")
    if d_count is not None and d_count.numel() != 1:
        raise BufferXError(f"fps_large: d_count must hold one point count, got {d_count.numel()} elements")
    lib = load_library()
    N = xyz.shape[0]
    idx = torch.empty(npoint, dtype=I32, device=xyz.device)
    kp = torch.empty((npoint, 3), dtype=F32, device=xyz.device) if want_kpts else None
    ws = torch.empty(int(lib.bx_fps_large_workspace_bytes(N)), dtype=torch.uint8, device=xyz.device)
    with _Span("fps_large"):
        if d_count is None:
            _check(lib.bx_fps_large(_dp(xyz, F32, "xyz"), N, int(npoint), _dp(idx), _dp(kp), _dp(ws), _stream()), "bx_fps_large")
        else:
            _check(lib.bx_fps_large_n(_dp(xyz, F32, "xyz"), N, _dp(d_count, I32, "d_count"), int(npoint), _dp(idx), _dp(kp), _dp(ws),
                                      _stream()), "bx_fps_large_n")
    return idx, kp


def fps_size_class(n: int, max_cluster=0) -> int:
    """The largest point count that gets the same FPS launch configuration as an n-point cloud (-1 above the FPS limit)."""
    return int(load_library().bx_fps_size_class(int(n), int(max_cluster)))


def fps_large_size_class(n: int, max_cluster=0) -> int:
    """Capacity of an n-point cloud's size class up to FPS_LARGE_MAX_POINTS: fps_size_class(n, max_cluster) up to
    FPS_MAX_POINTS; above, multiples of 18432 points (bx_fps_large_n's CTAs) each at most 1.25x the smallest cloud of its
    class, then FPS_LARGE_MAX_POINTS.  -1 above FPS_LARGE_MAX_POINTS."""
    return int(load_library().bx_fps_large_size_class(int(n), int(max_cluster)))


_round_tables = {}


def radius_round_table(device) -> torch.Tensor:
    """round(5*m/8192, 2) for every radius the reference's bisection can probe (models/BUFFERX.py:694)."""
    key = str(device)
    if key not in _round_tables:
        tab = np.array([round(5.0 * m / RADIUS_BINS, 2) for m in range(RADIUS_BINS + 1)], dtype=np.float32)
        _round_tables[key] = torch.from_numpy(tab).to(device)
    return _round_tables[key]


def radius_estimate(kpts: torch.Tensor, pts: torch.Tensor, thresholds, denom=None, tolerance=0.01, hist=None):
    """kpts [Kr,3], pts [N,3] (the larger cloud and its key-points).  Returns (r [n_thr] f32 device, m [n_thr] i32 device)."""
    lib = load_library()
    th = np.ascontiguousarray(thresholds, dtype=np.float64)
    Kr, N = kpts.shape[0], pts.shape[0]
    if hist is None:
        hist = torch.empty(RADIUS_BINS + 2, dtype=I32, device=pts.device)
    out_r = torch.empty(len(th), dtype=F32, device=pts.device)
    out_m = torch.empty(len(th), dtype=I32, device=pts.device)
    denom = int(N) * int(Kr) if denom is None else int(denom)
    _check(lib.bx_radius_estimate(_dp(kpts, F32, "kpts"), Kr, _dp(pts, F32, "pts"), N, denom, th.ctypes.data_as(c_void_p),
                                  len(th), float(tolerance), _dp(radius_round_table(pts.device)), _dp(hist), _dp(out_r),
                                  _dp(out_m), _stream()), "bx_radius_estimate")
    return out_r, out_m, hist


RADIUS_SUBSAMPLE = 200000       # the reference's sub-sample of a larger cloud (BUFFERX.py:664-665)


def radius_estimate_pair(kpts_s, pts_s, kpts_t, pts_t, thresholds, d_counts, tolerance=0.01, hist=None, d_sub=None):
    """Both clouds (capacity buffers) and their [Kr,3] key-points, d_counts [2] int32 CUDA = (ns, nt): the device picks the
    larger cloud (source iff ns > nt) and denom = N * Kr.  Returns (r, m, hist) like radius_estimate.
    d_sub: optional int32 CUDA indices into the chosen cloud, read when it has more than RADIUS_SUBSAMPLE points
    (bx_radius_estimate_n_sub):
      [RADIUS_SUBSAMPLE]: one histogram over pts[d_sub] serves every threshold, as
        radius_estimate(kpts, pts[d_sub], thresholds, denom=N * Kr);
      [len(thresholds), RADIUS_SUBSAMPLE]: one row per threshold (the reference draws one sub-sample per scale): threshold i
        has its own histogram (hist [len(thresholds), RADIUS_BINS + 2]) over pts[d_sub[i]], as
        radius_estimate(kpts, pts[d_sub[i]], thresholds[i:i + 1], denom=N * Kr), one launch per threshold."""
    lib = load_library()
    th = np.ascontiguousarray(thresholds, dtype=np.float64)
    Kr = kpts_s.shape[0]
    assert kpts_t.shape[0] == Kr
    per_threshold = d_sub is not None and d_sub.dim() == 2
    if d_sub is not None and tuple(d_sub.shape) not in ((RADIUS_SUBSAMPLE,), (len(th), RADIUS_SUBSAMPLE)):
        raise BufferXError(f"radius_estimate_pair: d_sub must be [{RADIUS_SUBSAMPLE}] or [{len(th)}, {RADIUS_SUBSAMPLE}], "
                           f"got {tuple(d_sub.shape)}")
    dev = pts_s.device
    if hist is None:
        hist = torch.empty((len(th), RADIUS_BINS + 2) if per_threshold else (RADIUS_BINS + 2,), dtype=I32, device=dev)
    out_r = torch.empty(len(th), dtype=F32, device=dev)
    out_m = torch.empty(len(th), dtype=I32, device=dev)
    if d_sub is None:
        _check(lib.bx_radius_estimate_n(_dp(kpts_s, F32, "kpts_s"), _dp(pts_s, F32, "pts_s"), pts_s.shape[0], _dp(kpts_t, F32, "kpts_t"),
                                        _dp(pts_t, F32, "pts_t"), pts_t.shape[0], Kr, _dp(d_counts, I32, "d_counts"), th.ctypes.data_as(c_void_p),
                                        len(th), float(tolerance), _dp(radius_round_table(dev)), _dp(hist), _dp(out_r), _dp(out_m), _stream()),
               "bx_radius_estimate_n")
        return out_r, out_m, hist
    if not per_threshold:
        _check(lib.bx_radius_estimate_n_sub(_dp(kpts_s, F32, "kpts_s"), _dp(pts_s, F32, "pts_s"), pts_s.shape[0], _dp(kpts_t, F32, "kpts_t"),
                                            _dp(pts_t, F32, "pts_t"), pts_t.shape[0], Kr, _dp(d_counts, I32, "d_counts"), _dp(d_sub, I32, "d_sub"),
                                            th.ctypes.data_as(c_void_p), len(th), float(tolerance), _dp(radius_round_table(dev)), _dp(hist),
                                            _dp(out_r), _dp(out_m), _stream()), "bx_radius_estimate_n_sub")
        return out_r, out_m, hist
    for i in range(len(th)):
        _check(lib.bx_radius_estimate_n_sub(_dp(kpts_s, F32, "kpts_s"), _dp(pts_s, F32, "pts_s"), pts_s.shape[0], _dp(kpts_t, F32, "kpts_t"),
                                            _dp(pts_t, F32, "pts_t"), pts_t.shape[0], Kr, _dp(d_counts, I32, "d_counts"), _dp(d_sub[i], I32, "d_sub"),
                                            th[i:i + 1].ctypes.data_as(c_void_p), 1, float(tolerance), _dp(radius_round_table(dev)), _dp(hist[i]),
                                            _dp(out_r[i:i + 1]), _dp(out_m[i:i + 1]), _stream()), "bx_radius_estimate_n_sub")
    return out_r, out_m, hist


def permute_cloud(pts: torch.Tensor, perm: torch.Tensor | None, out4: torch.Tensor | None = None, d_N=None):
    """d_N: optional 1-element int32 CUDA point count; rows of out4 from the count on are left untouched."""
    N = pts.shape[0]
    if out4 is None:
        out4 = torch.empty((N, 4), dtype=F32, device=pts.device)
    if d_N is None:
        _check(load_library().bx_permute_cloud(_dp(pts, F32, "pts"), _dp(perm, I32, "perm"), N, _dp(out4), _stream()), "bx_permute_cloud")
    else:
        _check(load_library().bx_permute_cloud_n(_dp(pts, F32, "pts"), _dp(perm, I32, "perm"), N, _dp(d_N, I32, "d_N"), _dp(out4), _stream()),
               "bx_permute_cloud_n")
    return out4


def select_patches(pts4: torch.Tensor, kpts: torch.Tensor, radius, P: int, want_idx=False, patches=None):
    """radius: python float or a 1-element CUDA f32 tensor (device-side radius, no sync)."""
    K, N = kpts.shape[0], pts4.shape[0]
    if patches is None:
        patches = torch.empty((K, P, 3), dtype=F32, device=pts4.device)
    idx = torch.empty((K, P), dtype=I32, device=pts4.device) if want_idx else None
    rv, rp = (0.0, _dp(radius, F32, "radius")) if isinstance(radius, torch.Tensor) else (float(radius), None)
    ev = profiler.span("select_patches", 16.0 * N + 12.0 * K + K * P * (12.0 + (4.0 if want_idx else 0.0))) if profiler else None
    if ev:
        ev[0].record()
    _check(load_library().bx_select_patches(_dp(pts4, F32, "pts4"), N, _dp(kpts, F32, "kpts"), K, rv, rp, P, _dp(idx), _dp(patches), _stream()),
           "bx_select_patches")
    if ev:
        ev[1].record()
    return patches, idx


# clouds of at least this many points gather their patches through the spatial hash grid (bx_select_patches_grid) instead of the
# streaming scan: a ball then holds so small a part of the cloud that reading the cloud front to back costs more than binning it.
# The threshold was chosen on the B200 and has not been re-measured on the H100.
GRID_MIN_POINTS = int(os.environ.get("BX_PATCHES_GRID_MIN", "12000"))


def select_patches_grid(pts4: torch.Tensor, kpts: torch.Tensor, radius: torch.Tensor, P: int, want_idx=False, patches=None):
    """Hash-grid form of select_patches (device-side radius tensor); bit-identical output."""
    K, N = kpts.shape[0], pts4.shape[0]
    if patches is None:
        patches = torch.empty((K, P, 3), dtype=F32, device=pts4.device)
    idx = torch.empty((K, P), dtype=I32, device=pts4.device) if want_idx else None
    lib = load_library()
    ws = torch.empty((int(lib.bx_select_patches_grid_workspace_bytes(N)) + 15) // 16 * 4, dtype=I32, device=pts4.device)
    with _Span("select_patches", 16.0 * N + 12.0 * K + K * P * (12.0 + (4.0 if want_idx else 0.0))):
        _check(lib.bx_select_patches_grid(_dp(pts4, F32, "pts4"), N, _dp(kpts, F32, "kpts"), K, _dp(radius, F32, "radius"), P, _dp(idx), _dp(patches, F32, "patches"),
                                          _dp(ws), _stream()), "bx_select_patches_grid")
    return patches, idx


def select_patches_batched(jobs, P: int, patches: torch.Tensor, grid=False, d_K=None, d_N=None):
    """jobs: [(pts4 [N,4], kpts [K,3], radius 1-element CUDA tensor)]; patches [sum K, P, 3] is filled job after job by ONE launch
    (grid=True: the hash-grid form, one launch per phase).  d_K: optional per-job 1-element int32 CUDA tensors (or None
    entries): job j gathers only its first min(d_K[j], K_j) key-points.  d_N: the same for points: pts4 of job j is then a
    capacity buffer whose first min(d_N[j], N_j) rows are the permuted cloud."""
    import ctypes
    n = len(jobs)
    VP, I = ctypes.c_void_p * n, ctypes.c_int32 * n
    pts = VP(*[_dp(j[0], F32, "pts4") for j in jobs])
    kps = VP(*[_dp(j[1], F32, "kpts") for j in jobs])
    rad = VP(*[_dp(j[2], F32, "radius") for j in jobs])
    cnt = None if d_K is None else VP(*[_dp(c, I32, "d_K") for c in d_K])
    npt = None if d_N is None else VP(*[_dp(c, I32, "d_N") for c in d_N])
    Ns, Ks = I(*[int(j[0].shape[0]) for j in jobs]), I(*[int(j[1].shape[0]) for j in jobs])
    assert patches.shape[0] == sum(Ks) and patches.is_contiguous()
    lib = load_library()
    ws = None
    if grid:
        ws = torch.empty(sum(int(lib.bx_select_patches_grid_workspace_bytes(int(a))) for a in Ns) // 4, dtype=I32, device=patches.device)
    with _Span("select_patches", sum(16.0 * a + 12.0 * b + b * P * 12.0 for a, b in zip(Ns, Ks))):
        if grid and npt is not None:
            _check(lib.bx_select_patches_grid_batched_counts(n, pts, Ns, npt, kps, Ks, rad, cnt, P, _dp(patches, F32, "patches"), _dp(ws),
                                                             _stream()), "bx_select_patches_grid_batched_counts")
        elif grid:
            _check(lib.bx_select_patches_grid_batched_n(n, pts, Ns, kps, Ks, rad, cnt, P, _dp(patches, F32, "patches"), _dp(ws), _stream()),
                   "bx_select_patches_grid_batched")
        elif npt is not None:
            _check(lib.bx_select_patches_batched_counts(n, pts, Ns, npt, kps, Ks, rad, cnt, P, _dp(patches, F32, "patches"), _stream()),
                   "bx_select_patches_batched_counts")
        else:
            _check(lib.bx_select_patches_batched_n(n, pts, Ns, kps, Ks, rad, cnt, P, _dp(patches, F32, "patches"), _stream()), "bx_select_patches_batched")
    return patches


def ball_query(xyz: torch.Tensor, qry: torch.Tensor, radius: float, nsample: int):
    idx = torch.empty((qry.shape[0], nsample), dtype=I32, device=xyz.device)
    _check(load_library().bx_ball_query(_dp(xyz, F32, "xyz"), xyz.shape[0], _dp(qry, F32, "qry"), qry.shape[0], float(radius), nsample,
                                        _dp(idx), _stream()), "bx_ball_query")
    return idx


def dropin_tensor(t, name: str, shape: str, dtype=F32):
    """Argument check of the drop-in modules under dropin/: a CUDA tensor of `dtype` with as many dims as `shape` names
    (e.g. "[B,N,3]"), returned contiguous.  Inputs that require grad raise NotImplementedError (no backward is built)."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: expected a torch.Tensor {shape}, got {type(t).__name__}")
    if t.requires_grad:
        raise NotImplementedError(f"{name}: inputs that require grad are not supported (forward only; no backward is built)")
    if not t.is_cuda:
        raise BufferXError(f"{name}: expected a CUDA tensor (bufferx_b200 has no CPU path)")
    if t.dim() != shape.count(",") + 1:
        raise BufferXError(f"{name}: expected shape {shape}, got {tuple(t.shape)}")
    if t.dtype != dtype:
        raise NotImplementedError(f"{name}: only {dtype} {shape} is supported, got {t.dtype}")
    return t.contiguous()


def ball_query_batched(xyz: torch.Tensor, qry: torch.Tensor, radius: float, nsample: int):
    """xyz [B,N,3], qry [B,M,3] f32 -> idx [B,M,nsample] int32: per cloud, the first nsample points (index order) with
    d2 < radius^2, padded with the first hit, all zero when nothing is hit."""
    B, N, M = xyz.shape[0], xyz.shape[1], qry.shape[1]
    idx = torch.empty((B, M, nsample), dtype=I32, device=xyz.device)
    if B == 0 or M == 0:
        return idx
    _check(load_library().bx_ball_query_batched(_dp(xyz, F32, "xyz"), B, N, _dp(qry, F32, "qry"), M, float(radius), int(nsample), _dp(idx),
                                                _stream()), "bx_ball_query_batched")
    return idx


def gather_channels(features: torch.Tensor, idx: torch.Tensor):
    """features [B,C,N] f32, idx [B,...] int32 -> [B,C,...]: out[b,c,k] = features[b,c,idx[b,k]] (NaN for an index outside
    [0,N))."""
    B, C, N = features.shape
    out = torch.empty((B, C) + tuple(idx.shape[1:]), dtype=F32, device=features.device)
    if out.numel() == 0:
        return out
    K = idx[0].numel()
    _check(load_library().bx_gather_channels(_dp(features, F32, "features"), B, C, N, _dp(idx, I32, "idx"), K, _dp(out), _stream()),
           "bx_gather_channels")
    return out


def knn1(ref: torch.Tensor, qry: torch.Tensor):
    """ref [B,Nr,D], qry [B,Nq,D] f32 -> (dist [B,Nq] f32 = sqrtf(d2), idx [B,Nq] int64): the first nearest ref row of each
    query row, d2 summed over D in order without FMA."""
    B, Nr, D = ref.shape
    Nq = qry.shape[1]
    dist = torch.empty((B, Nq), dtype=F32, device=ref.device)
    idx = torch.empty((B, Nq), dtype=torch.int64, device=ref.device)
    if B == 0 or Nq == 0:
        return dist, idx
    keys = torch.empty(B * Nq, dtype=torch.int64, device=ref.device)
    _check(load_library().bx_knn1(_dp(ref, F32, "ref"), Nr, _dp(qry, F32, "qry"), Nq, D, B, _dp(keys), _dp(dist), _dp(idx), _stream()),
           "bx_knn1")
    return dist, idx


def svd3(A: torch.Tensor):
    """A [B,3,3] f32 -> (U [B,3,3], S [B,3] descending, V [B,3,3]) with A = U diag(S) V^T (fp64 one-sided Jacobi)."""
    B = A.shape[0]
    U = torch.empty((B, 3, 3), dtype=F32, device=A.device)
    S = torch.empty((B, 3), dtype=F32, device=A.device)
    V = torch.empty((B, 3, 3), dtype=F32, device=A.device)
    if B:
        _check(load_library().bx_svd3(_dp(A, F32, "A"), B, _dp(U), _dp(S), _dp(V), _stream()), "bx_svd3")
    return U, S, V


def lrf(patches: torch.Tensor, des_r, aligned: bool, delta=None, Rt=None, ra=None, r_group=0, d_K=None):
    """d_K: optional int32 CUDA counts, one per radius group (r_group > 0) or one in all: patches beyond a count are not touched."""
    K, P, _ = patches.shape
    dev = patches.device
    if delta is None:
        delta = torch.empty_like(patches)
    if Rt is None:
        Rt = torch.empty((K, 3, 3), dtype=F32, device=dev)
    if ra is None:
        ra = torch.empty((K, 3), dtype=F32, device=dev)
    rv, rp = (0.0, _dp(des_r, F32, "des_r")) if isinstance(des_r, torch.Tensor) else (float(des_r), None)
    with _Span("lrf", 24.0 * K * P):
        flags = int(bool(aligned)) | (2 if os.environ.get("BX_LRF", "").lower() == "stable" else 0)
        _check(load_library().bx_lrf_batched_n(_dp(patches, F32, "patches"), K, P, rv, rp, int(r_group), _dp(d_K, I32, "d_K"), flags, _dp(delta), _dp(Rt),
                                               _dp(ra), _stream()), "bx_lrf")
    return delta, Rt, ra


def spt_pnt_sd(delta, voxels, rot, voxel_r: float, nv: int, w, b, azi_n: int, flag=None, d_K=None):
    """SPT + point layer with the features in the presplit padded fp16 format: [3, 4, conv_sd_rows(K), 8] fp16.
    d_K: optional int32[1] CUDA count: only the first min(d_K, K) patches are written."""
    K, P, _ = delta.shape
    V = voxels.shape[0]
    feat = conv_sd_buffer(K, 48, delta.device)
    with _Span("spt", 12.0 * K * P + 64.0 * K * V):
        _check(load_library().bx_spt_pnt_sd_n(_dp(delta, F32, "delta"), K, P, _dp(voxels, F32), V, azi_n, _dp(rot, F32), float(voxel_r), nv,
                                              _dp(w, F32), _dp(b, F32), _dp(feat), feat.shape[2], _dp(flag, I32, "flag"), _dp(d_K, I32, "d_K"),
                                              _stream()), "bx_spt_pnt_sd")
    return feat


def spt_pnt(delta, voxels, rot, voxel_r: float, nv: int, w, b, azi_n: int, debug=False, feat=None):
    K, P, _ = delta.shape
    V = voxels.shape[0]
    dev = delta.device
    if feat is None:
        feat = torch.empty((K, 4, V, 4), dtype=F32, device=dev)    # channel-blocked (see to_blocked)
    vidx = torch.empty((K, V, nv), dtype=I32, device=dev) if debug else None
    inv = torch.empty((K, V, nv, 3), dtype=F32, device=dev) if debug else None
    with _Span("spt", 12.0 * K * P + 64.0 * K * V):
        _check(load_library().bx_spt_pnt(_dp(delta, F32, "delta"), K, P, _dp(voxels, F32), V, azi_n, _dp(rot, F32), float(voxel_r), nv,
                                         _dp(w, F32), _dp(b, F32), _dp(feat), _dp(vidx), _dp(inv), _stream()), "bx_spt_pnt")
    return (feat, vidx, inv) if debug else feat


def tf32_split(w: torch.Tensor):
    """hi = round-to-nearest (ties away) TF32 of w (10-bit mantissa), lo = w - hi (exact in fp32)."""
    bits = w.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    hi_bits = ((bits + 0x1000) & 0xFFFFE000) & 0xFFFFFFFF
    hi_bits = torch.where(hi_bits >= 0x80000000, hi_bits - 0x100000000, hi_bits).to(torch.int32)
    hi = hi_bits.view(torch.float32)
    return hi, w - hi


def conv_tc_weights(Wt: torch.Tensor) -> torch.Tensor:
    """[T, Cin, Cout] folded fp32 weights -> the wgmma operand image of ``bx_conv_layer_tc``:
    [chunk(Cin/16)][tap][kstep(2)][split(hi,lo)][kunit(2)][n(NT)][4]."""
    T, Cin, Cout = Wt.shape
    assert Cin % 16 == 0 and Cout <= 128
    NT = 128 if Cout > 64 else (64 if Cout > 32 else 32)          # == bx_conv_tc_ntile(Cout)
    W = torch.zeros((T, Cin, NT), dtype=torch.float32, device=Wt.device)
    W[:, :, :Cout] = Wt
    hi, lo = tf32_split(W)
    both = torch.stack([hi, lo], dim=0)                               # [split, T, Cin, NT]
    both = both.view(2, T, Cin // 16, 2, 2, 4, NT)                    # [split, T, chunk, kstep, kunit, j, NT]
    img = both.permute(2, 1, 3, 0, 4, 6, 5).contiguous()              # [chunk, T, kstep, split, kunit, NT, j]
    return img.view(-1)


def to_blocked(x: torch.Tensor) -> torch.Tensor:
    """[n, C, S...] channel-first -> [n, C/4, S, 4] channel-blocked (activation layout of bx_conv_layer_tc)."""
    n, C = x.shape[0], x.shape[1]
    return x.reshape(n, C // 4, 4, -1).permute(0, 1, 3, 2).contiguous()


def from_blocked(x: torch.Tensor) -> torch.Tensor:
    """[n, C/4, S, 4] channel-blocked -> [n, C, S] channel-first."""
    n, G, S, _ = x.shape
    return x.permute(0, 1, 3, 2).reshape(n, G * 4, S).contiguous()


def conv_layer_tc(geom, x, w_tc, bias, out, n, Cin, Cout, D, H, W, kd, kh, kw, relu, d_n=None, equi_s=None, equi_t=None):
    """x / out are channel-blocked: [n, Cin/4, S_in, 4] / [n, Cout/4, S_out, 4]."""
    ev = None
    if profiler is not None and d_n is None:
        OD, OH, OW = (1, 7, 20) if geom in (GEOM_CYL3D, GEOM_CYL2D) else (D - kd + 1, H - kh + 1, W - kw + 1)
        ev = profiler.span("conv_desc", 2.0 * n * OD * OH * OW * Cout * Cin * kd * kh * kw)
        ev[0].record()
    elif profiler is not None:
        ev = profiler.span("conv_cost", 0.0)
        ev[0].record()
    _check(load_library().bx_conv_layer_tc(geom, _dp(x, F32, "x"), _dp(w_tc, F32, "w_tc"), _dp(bias, F32, "bias"), _dp(out, F32, "out"), int(n),
                                           _dp(d_n, I32, "d_n"), Cin, Cout, D, H, W, kd, kh, kw, int(bool(relu)), _dp(equi_s, F32), _dp(equi_t, F32),
                                           _stream()), "bx_conv_layer_tc")
    if ev:
        ev[1].record()
    return out


def conv_sd_weights(Wt: torch.Tensor) -> torch.Tensor:
    """[T, Cin, Cout] folded fp32 weights (T = 9: 3x3, or 27: 3x3x3 with Cin = 16) -> the fp16 operand image of
    ``bx_conv_layer_sd``: [chunk][tap(9)][kcore(2)][split(hi,lo)][n(NT)][8], w = hi + lo * 2^-11.  Cout <= 32 (NT = 32):
    [chunk][tap][kcore][P | Q][64][8], where in each 16-row group w of P rows 0-7 / 8-15 are hi / lo of channels 8w..8w+7 and
    in Q they are zero / hi (the 64-row A operand of the channels-as-M mainloop; the rows-as-M mainloop reads hi and lo out of
    P with a 256-byte core-matrix stride)."""
    T, Cin, Cout = Wt.shape
    assert T in (9, 27) and Cin % 16 == 0 and Cout <= 128 and (T == 9 or Cin == 16)
    NT = 128 if Cout > 64 else (64 if Cout > 32 else 32)
    W = torch.zeros((T, Cin, NT), dtype=torch.float32, device=Wt.device)
    W[:, :, :Cout] = Wt
    if T == 27:
        W = W.view(3, 9, 16, NT)                                   # chunk = radial slice dz
    else:
        W = W.view(9, Cin // 16, 16, NT).permute(1, 0, 2, 3)          # [chunk, tap, 16, NT]
    hi = W.half()
    lo = ((W - hi.float()) * 2048.0).half()
    nch = W.shape[0]
    if NT == 32:
        grp = lambda x: x.reshape(nch, 9, 2, 8, 4, 8).permute(0, 1, 2, 4, 5, 3)   # [chunk, tap, kcore, w, channel, 8]
        h, l = grp(hi), grp(lo)
        P = torch.stack([h, l], dim=4)                                # [chunk, tap, kcore, w, split, channel, 8]
        Q = torch.stack([torch.zeros_like(h), h], dim=4)
        return torch.stack([P, Q], dim=3).contiguous().view(-1)       # [chunk, tap, kcore, P|Q, w, split, channel, 8]
    both = torch.stack([hi, lo], dim=2)                               # [chunk, tap, split, 16, NT]
    both = both.reshape(nch, 9, 2, 2, 8, NT).permute(0, 1, 3, 2, 5, 4).contiguous()   # [chunk, tap, kcore, split, NT, 8]
    return both.view(-1)


def conv_sd_rows(n: int, rows_per_sample: int = 176) -> int:
    """Rows of a presplit activation image for n samples (cylindrical layers: 176 per sample; whole 128-row tiles + 48 halo rows)."""
    return int(load_library().bx_conv_sd_rows(int(n), int(rows_per_sample)))


def conv_sd_buffer(n: int, C: int, device, rows_per_sample: int = 176):
    """Uninitialised presplit activation image [C/16, 4, rows, 8] fp16 (the producing kernel writes every row that is read
    into a kept result)."""
    return torch.empty((C // 16, 4, conv_sd_rows(n, rows_per_sample), 8), dtype=torch.float16, device=device)


def conv_layer_sd(geom, x, w_sd, bias, out, n, Cin, Cout, relu, flag=None, d_n=None, D=0, W=0, tile_ctr=None):
    """x: fp32 channel-blocked [n, Cin/4, S_in, 4] or presplit fp16 [Cin/16, 4, rows, 8]; out likewise (dtype decides);
    ``flag``: int32[1] fp16-range flag (sticky); ``d_n``: device-side sample count; D, W: input raster of GEOM_VALID3D;
    ``tile_ctr``: int32[2] zeroed device counters -> dynamic tile scheduling (one pair per launch in flight)."""
    ev = None
    if profiler is not None:
        if geom == GEOM_VALID3D:
            ev = profiler.span("conv_cost", 0.0)
        else:
            ev = profiler.span("conv_desc", 2.0 * n * 140 * Cout * Cin * (27 if geom == GEOM_CYL3D else 9))
        ev[0].record()
    in_sd, out_sd = x.dtype == torch.float16, out.dtype == torch.float16
    _check(load_library().bx_conv_layer_sd(geom, _dp(x, None, "x"), int(in_sd), _dp(w_sd, torch.float16, "w_sd"), _dp(bias, F32, "bias"),
                                           _dp(out, None, "out"), int(out_sd), int(n), _dp(d_n, I32, "d_n"), Cin, Cout, int(D), int(W), int(bool(relu)),
                                           _dp(flag, I32, "flag"), _dp(tile_ctr, I32, "tile_ctr"), _stream()), "bx_conv_layer_sd")
    if ev:
        ev[1].record()
    return out


def conv_sd_weights_costab(Wt: torch.Tensor) -> torch.Tensor:
    """Second CostNet layer [27 taps (dn, dk, dl), 32, 64] -> the conv_sd image of the equivalent 96 -> 64, k = (3,1,3) layer:
    chunk = (dk, 16 channels), taps (dn, dl)."""
    assert Wt.shape == (27, 32, 64)
    W = Wt.view(3, 3, 3, 32, 64).permute(1, 0, 2, 3, 4).reshape(3, 9, 32, 64)          # [dk, tap = dn*3+dl, c, co]
    W = W.permute(1, 0, 2, 3).reshape(9, 96, 64).contiguous()                            # channel = dk * 32 + c
    return conv_sd_weights(W)


def conv_layer_sd_costab(fa, fb, w_sd, bias, out, n, relu, flag=None, d_n=None):
    """relu(A - B) regenerated from the factor maps -> 96 -> 64 conv over the 18 x 18 raster (bx_conv_layer_sd_costab)."""
    ev = profiler.span("conv_cost", 0.0) if profiler is not None else None
    if ev:
        ev[0].record()
    _check(load_library().bx_conv_layer_sd_costab(_dp(fa, F32, "fa"), _dp(fb, F32, "fb"), _dp(w_sd, torch.float16, "w_sd"), _dp(bias, F32, "bias"),
                                                  _dp(out, None, "out"), int(out.dtype == torch.float16), int(n), _dp(d_n, I32, "d_n"), int(bool(relu)),
                                                  _dp(flag, I32, "flag"), _stream()), "bx_conv_layer_sd_costab")
    if ev:
        ev[1].record()
    return out


def sd_pack(x: torch.Tensor) -> torch.Tensor:
    """Test helper (torch ops): channel-first [n, C, 7, 20] fp32 -> the presplit padded image [C/16, 4, rows, 8] fp16."""
    n, C = x.shape[0], x.shape[1]
    rows = conv_sd_rows(n)
    xp = torch.zeros((n, C, 8, 22), dtype=torch.float32, device=x.device)
    xp[:, :, 1:, 1:21] = x
    xp[:, :, 1:, 0] = x[:, :, :, 19]
    xp[:, :, 1:, 21] = x[:, :, :, 0]
    flat = torch.zeros((rows, C), dtype=torch.float32, device=x.device)
    flat[: n * 176] = xp.permute(0, 2, 3, 1).reshape(n * 176, C)
    hi = flat.half()
    lo = ((flat - hi.float()) * 2048.0).half()
    img = torch.stack([hi, lo], dim=0).view(2, rows, C // 16, 2, 8).permute(2, 0, 3, 1, 4).contiguous()   # [chunk, split, kcore, rows, 8]
    return img.view(C // 16, 4, rows, 8)


def sd_unpack(img: torch.Tensor, n: int) -> torch.Tensor:
    """Test helper: presplit padded image -> channel-first [n, C, 7, 20] fp32 (hi + lo * 2^-11), plus the padded raster
    [n, C, 8, 22] for checking the zero rows / wrap columns."""
    nch, _, rows, _ = img.shape
    v = img.view(nch, 2, 2, rows, 8).float()
    val = v[:, 0] + v[:, 1] / 2048.0                                  # [chunk, kcore, rows, 8]
    flat = val.permute(2, 0, 1, 3).reshape(rows, nch * 16)
    xp = flat[: n * 176].view(n, 8, 22, nch * 16).permute(0, 3, 1, 2)
    return xp[:, :, 1:, 1:21].contiguous(), xp


def costvol_factor_weights(Wt: torch.Tensor):
    """Folded first CostNet layer [27 taps (dn,dk,dl), 32, 32] -> (wa [32,3,5,32], wb [32,3,3,32]) of bx_costvol_ab:
    wa[c,dk,e,co] = sum of w over (dn,dl) with dl - dn = e - 2, wb[c,dk,dl,co] = sum over dn (fp64 sums, fp32 storage)."""
    W = Wt.detach().double().cpu().view(3, 3, 3, Wt.shape[1], Wt.shape[2])     # [dn, dk, dl, c, co]
    wa = torch.zeros((Wt.shape[1], 3, 5, Wt.shape[2]), dtype=torch.float64)
    for dn in range(3):
        for dl in range(3):
            wa[:, :, dl - dn + 2, :] += W[dn, :, dl].permute(1, 0, 2)
    wb = W.sum(dim=0).permute(2, 0, 1, 3).contiguous()                              # [c, dk, dl, co]
    return wa.float().contiguous().to(Wt.device), wb.float().contiguous().to(Wt.device)


def costvol_ab(equi_s, equi_t, s_mids, t_mids, d_M, maxM, wa, wb, bias, A=None, B=None):
    """Factors of the first CostNet activation: out0 = relu(A[co][k][(l-n) mod 20] - B[co][k][l]); A, B channel-blocked."""
    dev = equi_s.device
    if A is None:
        A = torch.empty((maxM, 8, 60, 4), dtype=F32, device=dev)      # channel-blocked [32/4][3*20][4]
    if B is None:
        B = torch.empty((maxM, 8, 54, 4), dtype=F32, device=dev)      # channel-blocked [32/4][3*18][4]
    with _Span("conv_cost"):
        _check(load_library().bx_costvol_ab(_dp(equi_s, F32, "equi_s"), _dp(equi_t, F32, "equi_t"), _dp(s_mids, I32, "s_mids"),
                                            _dp(t_mids, I32, "t_mids"), _dp(d_M, I32, "d_M"), int(maxM), _dp(wa, F32, "wa"), _dp(wb, F32, "wb"),
                                            _dp(bias, F32, "bias"), _dp(A), _dp(B), _stream()), "bx_costvol_ab")
    return A, B


def pool_desc(x, w1, b1, w2, b2, desc=None, equi=None, channels_last=False, d_K=None):
    """x: [K,32,7,20] (channel-first) or channel-blocked [K,8,140,4] with channels_last=True.  equi is always [K,32,7,20].
    d_K: optional int32[1] CUDA count: rows at or beyond it are not written."""
    K, C = x.shape[0], 32
    S = x.numel() // max(K * C, 1) if K > 0 else 140
    dev = x.device
    if desc is None:
        desc = torch.empty((K, C), dtype=F32, device=dev)
    if equi is None:
        equi = torch.empty((K, C, 7, 20) if S == 140 else (K, C, S), dtype=F32, device=dev)
    _check(load_library().bx_pool_desc_n(_dp(x, F32, "x"), K, C, S, int(bool(channels_last)), _dp(w1, F32), _dp(b1, F32), _dp(w2, F32), _dp(b2, F32),
                                         _dp(desc), _dp(equi), _dp(d_K, I32, "d_K"), _stream()), "bx_pool_desc")
    return desc, equi


def mutual_nn(a, b, want_nn=False, out=None, d_Ka=None, d_Kb=None):
    """out: optional (s_mids [>=Ka], t_mids [>=Ka], dM [1]) int32 buffers to fill (dM must be zero on entry).
    d_Ka / d_Kb: optional int32[1] CUDA counts: only the first rows of a / b take part (0 on either side: *dM = 0)."""
    Ka, Kb, C = a.shape[0], b.shape[0], a.shape[1]
    dev = a.device
    keys = torch.empty(Ka + Kb + 1, dtype=torch.int64, device=dev)
    if out is not None:
        s, t, dM = out
    else:
        s = torch.empty(max(Ka, 1), dtype=I32, device=dev)
        t = torch.empty(max(Ka, 1), dtype=I32, device=dev)
        dM = torch.zeros(1, dtype=I32, device=dev)
    snn = torch.empty(max(Ka, 1), dtype=I32, device=dev) if want_nn else None
    tnn = torch.empty(max(Kb, 1), dtype=I32, device=dev) if want_nn else None
    _check(load_library().bx_mutual_nn_n(_dp(a, F32, "a"), Ka, _dp(b, F32, "b"), Kb, C, _dp(d_Ka, I32, "d_Ka"), _dp(d_Kb, I32, "d_Kb"), _dp(keys),
                                         _dp(s), _dp(t), _dp(dM), _dp(snn), _dp(tnn), _stream()), "bx_mutual_nn")
    return s, t, dM, snn, tnn


def concat_matches(s_lists, t_lists, counts, s_row_off, t_row_off, d_offs):
    """[S,K] per-scale match lists + device counts -> (s_all, t_all) [S*K] in scale order with row offsets added;
    d_offs [S+1] int32 receives the prefix sums."""
    S, K = s_lists.shape
    dev = s_lists.device
    s_all = torch.empty(S * K, dtype=I32, device=dev)
    t_all = torch.empty(S * K, dtype=I32, device=dev)
    so = np.ascontiguousarray(s_row_off, dtype=np.int32)
    to = np.ascontiguousarray(t_row_off, dtype=np.int32)
    _check(load_library().bx_concat_matches(_dp(s_lists, I32, "s_lists"), _dp(t_lists, I32, "t_lists"), _dp(counts, I32, "counts"), S, K,
                                            so.ctypes.data_as(c_void_p), to.ctypes.data_as(c_void_p), _dp(s_all), _dp(t_all),
                                            _dp(d_offs, I32, "d_offs"), _stream()), "bx_concat_matches")
    return s_all, t_all


def hypotheses(logits, azi_n, kpts_s, kpts_t, Rt_s, Rt_t, s_mids, t_mids, d_M, maxM, d_off, d_off_out, ind_out, R_acc, t_acc,
               ss_acc, tt_acc):
    _check(load_library().bx_hypotheses(_dp(logits, F32), azi_n, _dp(kpts_s, F32), _dp(kpts_t, F32), _dp(Rt_s, F32), _dp(Rt_t, F32), _dp(s_mids, I32),
                                        _dp(t_mids, I32), _dp(d_M, I32), int(maxM), _dp(d_off, I32), _dp(d_off_out, I32), _dp(ind_out, F32),
                                        _dp(R_acc, F32), _dp(t_acc, F32), _dp(ss_acc, F32), _dp(tt_acc, F32), _stream()), "bx_hypotheses")


def consensus(ss, tt, R, t, d_Mc, maxMc, azi_n, inlier_th):
    dev = ss.device
    counts = torch.empty(max(maxMc, 1), dtype=I32, device=dev)
    ind = torch.empty(max(maxMc, 1), dtype=I32, device=dev)
    dI = torch.zeros(1, dtype=I32, device=dev)
    dbest = torch.zeros(1, dtype=I32, device=dev)
    _check(load_library().bx_consensus(_dp(ss, F32), _dp(tt, F32), _dp(R, F32), _dp(t, F32), _dp(d_Mc, I32), int(maxMc), azi_n, float(inlier_th),
                                       _dp(counts), _dp(ind), _dp(dI), _dp(dbest), _stream()), "bx_consensus")
    return ind, dI, dbest, counts


def ransac_workspace(max_iter, device):
    n = int(load_library().bx_ransac_workspace_bytes(int(max_iter)))
    return torch.empty((n + 7) // 8, dtype=torch.int64, device=device)


def ransac(ss, tt, inlier_ind, d_I, maxI, dist_th, similar_th, confidence, max_iter, seed, workspace=None, result=None):
    """result: 18-element float64 CUDA tensor = T (16 doubles) + {num_inliers, best_itr, iters_run, 0} as int32 pairs."""
    dev = ss.device
    if workspace is None:
        workspace = ransac_workspace(max_iter, dev)
    if result is None:
        result = torch.empty(18, dtype=torch.float64, device=dev)
    ev = profiler.span("ransac", 0.0) if profiler else None
    if ev:
        ev[0].record()
    _check(load_library().bx_ransac(_dp(ss, F32), _dp(tt, F32), _dp(inlier_ind, I32), _dp(d_I, I32), int(maxI), float(dist_th), float(similar_th),
                                    float(confidence), int(max_iter), int(seed) & 0xFFFFFFFFFFFFFFFF, _dp(workspace), _dp(result), _stream()),
           "bx_ransac")
    if ev:
        ev[1].record()
    return result


def early_exit_gate(result, min_inliers: int, caps, counts, num_scales: int, scales_used=None):
    """Early-exit decision on the device from a RANSAC result block: counts[i] = 0 when result's num_inliers >= min_inliers,
    else caps[i] (host ints); scales_used (float64[1], optional) = 1 or num_scales."""
    cp = np.ascontiguousarray(caps, dtype=np.int32)
    assert counts.numel() >= len(cp)
    _check(load_library().bx_early_exit_gate(_dp(result, torch.float64, "result"), int(min_inliers), len(cp), cp.ctypes.data_as(c_void_p),
                                             _dp(counts, I32, "counts"), int(num_scales), _dp(scales_used, torch.float64, "scales_used"),
                                             _stream()), "bx_early_exit_gate")
    return counts


def decode_ransac_result(result_cpu: torch.Tensor):
    T = result_cpu[:16].reshape(4, 4).numpy().copy()
    ints = result_cpu[16:18].numpy().view(np.int32)
    return T, int(ints[0]), int(ints[1]), int(ints[2])


def refine(ss, tt, d_n, maxn, T_in, dist_th, T_out=None, d_rounds=None):
    dev = ss.device
    if T_out is None:
        T_out = torch.empty(16, dtype=F32, device=dev)
    if d_rounds is None:
        d_rounds = torch.zeros(1, dtype=I32, device=dev)
    _check(load_library().bx_refine(_dp(ss, F32), _dp(tt, F32), _dp(d_n, I32), int(maxn), _dp(T_in, torch.float64, "T_in"), float(dist_th), _dp(T_out),
                                    _dp(d_rounds), _stream()), "bx_refine")
    return T_out, d_rounds


def radius_neighbors(queries, supports, q_batches, s_batches, radius: float):
    """All supports within `radius` of every query, distance-sorted, padded with len(supports) -- the reference's
    ``radius_neighbors.batch_query`` (cpp_wrappers/cpp_neighbors).  Two launches: count, then gather+sort."""
    lib = load_library()
    qb = np.ascontiguousarray(q_batches, dtype=np.int32)
    sb = np.ascontiguousarray(s_batches, dtype=np.int32)
    nq, ns = queries.shape[0], supports.shape[0]
    dmax = torch.zeros(1, dtype=I32, device=queries.device)
    args = (_dp(queries, F32, "queries"), nq, _dp(supports, F32, "supports"), ns, qb.ctypes.data_as(c_void_p), len(qb),
            sb.ctypes.data_as(c_void_p), len(sb), float(radius))
    _check(lib.bx_radius_neighbors(*args, None, 0, _dp(dmax), None, None, _stream()), "bx_radius_neighbors")
    mc = int(dmax.item())
    out = torch.empty((nq, max(mc, 1)), dtype=I32, device=queries.device)
    sd = si = None
    if mc > 4096:      # balls too large for the shared-memory sort: global scratch rows for the rank sort
        if nq * mc * 12 > (8 << 30):
            raise BufferXError(f"bx_radius_neighbors: {nq} queries x {mc} neighbours need more than 8 GB of scratch")
        sd = torch.empty((nq, mc), dtype=torch.float64, device=queries.device)
        si = torch.empty((nq, mc), dtype=I32, device=queries.device)
    if mc > 0:
        _check(lib.bx_radius_neighbors(*args, _dp(out), mc, _dp(dmax), _dp(sd), _dp(si), _stream()), "bx_radius_neighbors")
    return out[:, :mc]


def grid_subsample(points, dl: float):
    """Voxel barycentres (reference ``grid_subsampling.subsample``): returns (keys u64-as-int64 [m], xyz [m,3], counts [m])."""
    lib = load_library()
    n = points.shape[0]
    dev = points.device
    cap = 1
    while cap < 2 * n:
        cap <<= 1
    tkeys = torch.empty(cap, dtype=torch.int64, device=dev)
    tacc = torch.empty((cap, 4), dtype=F32, device=dev)
    mm = torch.empty(6, dtype=F32, device=dev)
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    xyz = torch.empty((n, 3), dtype=F32, device=dev)
    cnt = torch.empty(n, dtype=I32, device=dev)
    dm = torch.zeros(1, dtype=I32, device=dev)
    _check(lib.bx_grid_subsample(_dp(points, F32, "points"), n, float(dl), _dp(tkeys), _dp(tacc), cap, _dp(mm), _dp(keys), _dp(xyz), _dp(cnt),
                                 _dp(dm), _stream()), "bx_grid_subsample")
    m = int(dm.item())
    return keys[:m], xyz[:m], cnt[:m]


F64 = torch.float64


def pca_analysis(points: torch.Tensor, sample_idx: torch.Tensor | None = None):
    """sklearn-PCA of the sampled points (reference utils/tools.py:132-149).  Returns (mean [3], variance [3] desc,
    components [3,3] rows) as float64 CUDA tensors (views of one 15-double block)."""
    n = points.shape[0]
    dev = points.device
    ns = n if sample_idx is None else int(sample_idx.shape[0])
    acc = torch.empty(9, dtype=F64, device=dev)
    out = torch.empty(15, dtype=F64, device=dev)
    _check(load_library().bx_pca_analysis(_dp(points, F32, "points"), n, _dp(sample_idx, I32, "sample_idx"), ns, _dp(acc), _dp(out), _stream()),
           "bx_pca_analysis")
    return out[0:3], out[3:6], out[6:15].view(3, 3)


def project_range(points: torch.Tensor, mean: torch.Tensor, axis: torch.Tensor):
    """(min, max) of (p - mean) . axis over the cloud, float64 CUDA tensor [2]."""
    dev = points.device
    ma = torch.cat([mean.reshape(3), axis.reshape(3)]).to(F64).contiguous()
    work = torch.empty(2, dtype=torch.int64, device=dev)
    out = torch.empty(2, dtype=F64, device=dev)
    _check(load_library().bx_project_range(_dp(points, F32, "points"), points.shape[0], _dp(ma), _dp(work), _dp(out), _stream()), "bx_project_range")
    return out


VOXEL_AXIS_CELLS = 1 << 21          # voxel keys hold 21 bits per axis


def _dec_ordered(e):
    """bx_bootstrap.cu's order-preserving u64 encoding of doubles, decoded on the host: int64 array -> float64 array."""
    u = e.view(np.uint64)
    neg = (u >> np.uint64(63)) == 0
    return np.where(neg, ~u, u & np.uint64(0x7FFFFFFFFFFFFFFF)).view(np.float64)


def voxel_down_sample(points: torch.Tensor, voxel: float):
    """Open3D voxel_down_sample: returns (keys [m] int64 = ix | iy << 21 | iz << 42, xyz [m,3] f32, counts [m]), hash order.
    A cloud spanning 2^21 voxels or more on an axis is refused (its keys would alias); the extent is read from the
    kernel's min / max in the same transfer as the voxel count.  So is a cloud whose extent is not finite (an infinite
    coordinate, or an axis without one finite value): it has no voxel grid.  The min / max skip NaN coordinates."""
    lib = load_library()
    n = points.shape[0]
    dev = points.device
    voxel = float(voxel)
    cap = 1
    while cap < 2 * n:
        cap <<= 1
    tkeys = torch.empty(cap, dtype=torch.int64, device=dev)
    tacc = torch.empty((cap, 4), dtype=F64, device=dev)
    mm_dm = torch.empty(7, dtype=torch.int64, device=dev)         # minmax6, then the voxel count in the low half of [6]
    mm, dm = mm_dm[:6], mm_dm[6:].view(I32)
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    xyz = torch.empty((n, 3), dtype=F32, device=dev)
    cnt = torch.empty(n, dtype=I32, device=dev)
    _check(lib.bx_voxel_down_sample(_dp(points, F32, "points"), n, voxel, _dp(tkeys), _dp(tacc), cap, _dp(mm), _dp(keys), _dp(xyz),
                                    _dp(cnt), _dp(dm), _stream()), "bx_voxel_down_sample")
    h = mm_dm.cpu().numpy()
    m = int(h[6:7].view(np.int32)[0])
    lo, hi = _dec_ordered(h[0:3]), _dec_ordered(h[3:6])
    for c in range(3):
        t = (float(hi[c]) - (float(lo[c]) - voxel * 0.5)) / voxel                    # the kernel's index of the largest point
        if not math.isfinite(t):
            raise BufferXError(f"bx_voxel_down_sample: axis {'xyz'[c]} has no finite extent (min {lo[c]}, max {hi[c]}); "
                               "voxel_down_sample needs finite coordinates")
        top = math.floor(t)
        if top >= VOXEL_AXIS_CELLS:
            raise BufferXError(f"bx_voxel_down_sample: the cloud spans {top + 1} voxels of {voxel} on axis {'xyz'[c]}; "
                               f"voxel keys hold fewer than 2^21 = {VOXEL_AXIS_CELLS} per axis")
    return keys[:m], xyz[:m], cnt[:m]


# --------------------------------------------------------------------------- #
# training stages' validation forward (cfg.stage "Desc" / "Pose", eval mode)
# --------------------------------------------------------------------------- #
def gt_matches(src: torch.Tensor, tgt: torch.Tensor, T: torch.Tensor, voxel: float):
    """Ground-truth correspondences: src [N,3], tgt [M,3], T [4,4] f32 -> (pairs [N,2] int32, count [1] int32 on the device);
    rows >= count are undefined."""
    N, M = src.shape[0], tgt.shape[0]
    dev = src.device
    nn = torch.empty(max(N, 1), dtype=I32, device=dev)
    pairs = torch.empty((max(N, 1), 2), dtype=I32, device=dev)
    cnt = torch.zeros(1, dtype=I32, device=dev)
    _check(load_library().bx_gt_matches(_dp(src, F32, "src"), N, _dp(tgt, F32, "tgt"), M, _dp(T, F32, "T"), float(voxel), _dp(nn), _dp(pairs),
                                        _dp(cnt), _stream()), "bx_gt_matches")
    return pairs, cnt


def so2_augment(delta: torch.Tensor, rand_axis: torch.Tensor, angles: torch.Tensor, aug_R: torch.Tensor | None = None):
    """Rotates delta [K,P,3] and rand_axis [K,3] in place about z by angles [K] (f32); returns aug_R [K,3,3]."""
    K, P, _ = delta.shape
    if aug_R is None:
        aug_R = torch.empty((K, 3, 3), dtype=F32, device=delta.device)
    _check(load_library().bx_so2_augment(_dp(delta, F32, "delta"), K, P, _dp(rand_axis, F32, "rand_axis"), _dp(angles, F32, "angles"), _dp(aug_R),
                                         _stream()), "bx_so2_augment")
    return aug_R


def equi_match(d1: torch.Tensor, d2: torch.Tensor, out: torch.Tensor | None = None):
    """EquiMatch score of two [B,C,K,L] equivariant maps -> [B,L]."""
    B, C, K, L = d1.shape
    if tuple(d2.shape) != (B, C, K, L):
        raise BufferXError(f"equi_match: shapes {tuple(d1.shape)} and {tuple(d2.shape)} differ")
    if out is None:
        out = torch.empty((B, L), dtype=F32, device=d1.device)
    _check(load_library().bx_equi_match(_dp(d1, F32, "d1"), _dp(d2, F32, "d2"), B, C, K, L, _dp(out, F32, "out"), _stream()), "bx_equi_match")
    return out


def so2_gt(s_rand_axis, s_R, t_R, T, azi_n: int, integer: bool, aug_R=None):
    """SO(2) label of every patch: int64 [P] (integer=True) or float32 [P]."""
    P = s_rand_axis.shape[0]
    dev = s_rand_axis.device
    out = torch.empty(P, dtype=torch.int64 if integer else F32, device=dev)
    li, lf = (_dp(out), None) if integer else (None, _dp(out))
    _check(load_library().bx_so2_gt(_dp(s_rand_axis, F32, "s_rand_axis"), _dp(s_R, F32, "s_R"), _dp(t_R, F32, "t_R"), _dp(T, F32, "T"),
                                    _dp(aug_R, F32, "aug_R"), P, int(azi_n), li, lf, _stream()), "bx_so2_gt")
    return out


def icp(src: torch.Tensor, tgt: torch.Tensor, max_correspondence_distance: float, init: torch.Tensor, relative_fitness: float,
        relative_rmse: float, max_iteration: int):
    """Point-to-point ICP (bx_icp): src [Ns,3], tgt [Nt,3], init [4,4] float64 CUDA tensors.  Returns (result float64 [20] =
    T (16) + fitness + inlier_rmse + int32 {num_correspondences, iterations, converged, 0}, corr int32 [Ns]: each source
    point's target index or -1), both on the device; nothing is read back."""
    for t, name in ((src, "src"), (tgt, "tgt")):
        if t.dim() != 2 or t.shape[1] != 3 or t.shape[0] < 1:
            raise BufferXError(f"icp: {name} must be [N,3] with N >= 1, got {tuple(t.shape)}")
    if init.numel() != 16:
        raise BufferXError(f"icp: init must hold a 4x4 matrix (16 doubles), got {tuple(init.shape)}")
    lib = load_library()
    Ns, Nt = src.shape[0], tgt.shape[0]
    dev = src.device
    ws = torch.empty((int(lib.bx_icp_workspace_bytes(Ns, Nt)) + 255) // 8 + 32, dtype=torch.float64, device=dev)
    off = (-ws.data_ptr()) % 256 // 8                                    # the workspace must be 256-byte aligned
    result = torch.empty(20, dtype=F64, device=dev)
    corr = torch.empty(max(Ns, 1), dtype=I32, device=dev)
    with _Span("icp"):
        _check(lib.bx_icp(_dp(src, F64, "src"), Ns, _dp(tgt, F64, "tgt"), Nt, float(max_correspondence_distance),
                          _dp(init, F64, "init"), float(relative_fitness), float(relative_rmse), int(max_iteration), _dp(corr),
                          _dp(result), ws[off:].data_ptr(), _stream()), "bx_icp")
    return result, corr


def decode_icp_result(result_cpu: torch.Tensor):
    """-> (T [4,4] float64, fitness, inlier_rmse, num_correspondences, iterations, converged)."""
    T = result_cpu[:16].reshape(4, 4).numpy().copy()
    ints = result_cpu[18:20].numpy().view(np.int32)
    return T, float(result_cpu[16]), float(result_cpu[17]), int(ints[0]), int(ints[1]), bool(ints[2])


# --------------------------------------------------------------------------- #
# the Pose-stage training step (bx_train_step.cu): activations channel-blocked fp32 [n, C/4, S, 4]
# --------------------------------------------------------------------------- #
F64 = torch.float64


def _splits():
    return int(load_library().bx_ts_splits())


def _ts_shape(what, t, shape, name):
    """Refuse a mis-shaped input of a bx_ts_* kernel before launch (they index by the sizes passed, not the tensor's)."""
    if not isinstance(t, torch.Tensor) or tuple(t.shape) != tuple(shape):
        got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
        raise BufferXError(f"{what}: {name} must be {list(shape)}, got {got}")


def _ts_blocked(what, x, name="x"):
    if not isinstance(x, torch.Tensor) or x.dim() != 4 or x.shape[3] != 4:
        raise BufferXError(f"{what}: {name} must be a blocked image [n, C/4, S, 4], got "
                           f"{tuple(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__}")
    return x.shape[0], x.shape[1], x.shape[2]


def channel_sums(x):
    """-> float64 [2, C] per channel of the blocked x [n, C/4, S, 4] (fp32 or float64): (sum x, sum x^2)."""
    n, G, S = _ts_blocked("channel_sums", x)
    C = 4 * G
    partial = torch.empty(_splits() * 2 * C, dtype=F64, device=x.device)
    out = torch.empty(2 * C, dtype=F64, device=x.device)
    f64 = x.dtype == F64
    fn = load_library().bx_ts_channel_sums_f64 if f64 else load_library().bx_ts_channel_sums
    _check(fn(_dp(x, F64 if f64 else F32, "x"), n, C, S, _dp(partial), _dp(out), _stream()), "bx_ts_channel_sums")
    return out.view(2, C)


def moments3(v):
    """[..., 3] fp32 -> float64 [9]: sums of x, y, z, xx, xy, xz, yy, yz, zz."""
    if not isinstance(v, torch.Tensor) or v.dim() < 1 or v.shape[-1] != 3 or v.numel() == 0:
        raise BufferXError(f"moments3: v must be [..., 3] with at least one vector, got "
                           f"{tuple(v.shape) if isinstance(v, torch.Tensor) else type(v).__name__}")
    R = v.numel() // 3
    partial = torch.empty(_splits() * 9, dtype=F64, device=v.device)
    out = torch.empty(9, dtype=F64, device=v.device)
    _check(load_library().bx_ts_moments3(_dp(v, F32, "v"), R, _dp(partial), _dp(out), _stream()), "bx_ts_moments3")
    return out


def bn_apply(z, scale, shift, relu, out=None):
    """y = z scale + shift per channel (ReLU if relu) on a blocked image, fp32 or float64 (scale / shift of the same dtype)."""
    n, G, S = _ts_blocked("bn_apply", z, "z")
    _ts_shape("bn_apply", scale, (4 * G,), "scale")
    _ts_shape("bn_apply", shift, (4 * G,), "shift")
    if out is not None:
        _ts_shape("bn_apply", out, z.shape, "out")
    y = torch.empty_like(z) if out is None else out
    dt = z.dtype
    fn = load_library().bx_ts_bn_apply_f64 if dt == F64 else load_library().bx_ts_bn_apply
    _check(fn(_dp(z, dt, "z"), _dp(scale, dt, "scale"), _dp(shift, dt, "shift"), n, 4 * G, S, int(bool(relu)), _dp(y, dt, "y"), _stream()),
           "bx_ts_bn_apply")
    return y


def bn_backward(dy, z, y, mean, rstd, gamma):
    """Batch-statistics BatchNorm + ReLU backward, float64 blocked: -> (dz like z, sums [2, C] = (sum dz', sum dz' x^)
    = (dbeta, dgamma)), dz' = dy [y > 0], x^ = (z - mean) rstd.  y is the forward's ReLU output (bn_apply's), so the
    mask is the forward's bit for bit.  A BatchNorm with affine=False passes gamma = 1 and rstd = its scale."""
    n, G, S = _ts_blocked("bn_backward", z, "z")
    _ts_shape("bn_backward", dy, z.shape, "dy")
    _ts_shape("bn_backward", y, z.shape, "y")
    for name, t in (("mean", mean), ("rstd", rstd), ("gamma", gamma)):
        _ts_shape("bn_backward", t, (4 * G,), name)
    C = 4 * G
    partial = torch.empty(_splits() * 2 * C, dtype=F64, device=z.device)
    sums = torch.empty(2 * C, dtype=F64, device=z.device)
    dx = torch.empty_like(z)
    _check(load_library().bx_ts_bn_backward(_dp(dy, F64, "dy"), _dp(z, F64, "z"), _dp(y, F64, "y"), _dp(mean, F64, "mean"),
                                            _dp(rstd, F64, "rstd"), _dp(gamma, F64, "gamma"), n, C, S, _dp(partial), _dp(sums),
                                            _dp(dx), _stream()), "bx_ts_bn_backward")
    return dx, sums.view(2, C)


def conv1x1(x, w, b=None, out=None):
    """1x1 convolution of a blocked image, fp32 or float64 (w, b, out of x's dtype): x [n, Cin/4, S, 4], w [Cin, Cout],
    b [Cout] or None -> [n, Cout/4, S, 4]; with ``out`` the result is added to it.  Cin, Cout <= 32, multiples of 4."""
    n, G, S = _ts_blocked("conv1x1", x)
    if not isinstance(w, torch.Tensor) or w.dim() != 2 or w.shape[0] != 4 * G:
        raise BufferXError(f"conv1x1: w must be [{4 * G}, Cout], got {tuple(w.shape) if isinstance(w, torch.Tensor) else w}")
    Cout = w.shape[1]
    if Cout % 4 or not 4 <= Cout <= 32 or 4 * G > 32:
        raise BufferXError(f"conv1x1: {4 * G} -> {Cout} channels: both must be multiples of 4, at most 32")
    if b is not None:
        _ts_shape("conv1x1", b, (Cout,), "b")
    acc = out is not None
    if acc:
        _ts_shape("conv1x1", out, (n, Cout // 4, S, 4), "out")
    else:
        out = torch.empty((n, Cout // 4, S, 4), dtype=x.dtype, device=x.device)
    dt = F64 if x.dtype == F64 else F32
    fn = load_library().bx_ts_conv1x1_f64 if dt == F64 else load_library().bx_ts_conv1x1
    _check(fn(_dp(x, dt, "x"), _dp(w, dt, "w"), _dp(b, dt, "b"), n, 4 * G, Cout, S, int(acc), _dp(out, dt, "out"), _stream()),
           "bx_ts_conv1x1")
    return out


def costvol(equi_s, equi_t):
    """Full fp32 maps [M,32,7,20] (patch i against patch i) -> the blocked float64 cost volume [M, 8, 2000, 4] of rows 1..5."""
    M = equi_s.shape[0] if isinstance(equi_s, torch.Tensor) and equi_s.dim() == 4 else -1
    _ts_shape("costvol", equi_s, (M, 32, 7, 20), "equi_s")
    _ts_shape("costvol", equi_t, (M, 32, 7, 20), "equi_t")
    cv = torch.empty((M, 8, 2000, 4), dtype=F64, device=equi_s.device)
    _check(load_library().bx_ts_costvol(_dp(equi_s, F32, "equi_s"), _dp(equi_t, F32, "equi_t"), M, _dp(cv), _stream()), "bx_ts_costvol")
    return cv


def softargmax(logits, g=None):
    """float64 logits [M, L] -> ind [M]; with g [M] (dL/d ind, float64) -> dL/dlogits [M, L]."""
    if not isinstance(logits, torch.Tensor) or logits.dim() != 2:
        raise BufferXError(f"softargmax: logits must be [M, L], got {tuple(logits.shape) if isinstance(logits, torch.Tensor) else logits}")
    M, L = logits.shape
    if g is not None:
        _ts_shape("softargmax", g, (M,), "g")
    ind = None if g is not None else torch.empty(M, dtype=F64, device=logits.device)
    dl = torch.empty_like(logits) if g is not None else None
    _check(load_library().bx_ts_softargmax(_dp(logits, F64, "logits"), M, L, _dp(g, F64, "g"), _dp(ind), _dp(dl), _stream()), "bx_ts_softargmax")
    return dl if g is not None else ind


def _conv_shapes(what, x, Wt, D, H, W, kd, kh, kw):
    """x [n, Cin/4, D*H*W, 4] and Wt [kd*kh*kw, Cin, Cout] of one valid 3-D convolution -> (n, Cin, Cout); the kernel
    itself refuses Cin % 32, Cout % 4, a kernel larger than the extent and n = 0."""
    n, G, S = _ts_blocked(what, x)
    if not isinstance(Wt, torch.Tensor) or Wt.dim() != 3:
        raise BufferXError(f"{what}: Wt must be [kd*kh*kw, Cin, Cout], got {tuple(Wt.shape) if isinstance(Wt, torch.Tensor) else Wt}")
    _ts_shape(what, Wt, (kd * kh * kw, 4 * G, Wt.shape[2]), "Wt")
    if S != D * H * W:
        raise BufferXError(f"{what}: x holds {S} positions per channel, the geometry {D}x{H}x{W} has {D * H * W}")
    if Wt.shape[2] % 4:
        raise BufferXError(f"{what}: Cout = {Wt.shape[2]} is not a multiple of 4")
    if not (1 <= kd <= D and 1 <= kh <= H and 1 <= kw <= W):
        raise BufferXError(f"{what}: kernel {kd}x{kh}x{kw} does not fit the extent {D}x{H}x{W}")
    return n, 4 * G, Wt.shape[2]


def conv_forward(x, Wt, b, D, H, W, kd, kh, kw):
    """float64 valid 3-D convolution: x [n, Cin/4, D*H*W, 4], Wt [T, Cin, Cout], b [Cout] -> [n, Cout/4, OD*OH*OW, 4]."""
    n, Cin, Cout = _conv_shapes("conv_forward", x, Wt, D, H, W, kd, kh, kw)
    _ts_shape("conv_forward", b, (Cout,), "b")
    out = torch.empty((n, Cout // 4, (D - kd + 1) * (H - kh + 1) * (W - kw + 1), 4), dtype=F64, device=x.device)
    _check(load_library().bx_ts_conv_forward(_dp(x, F64, "x"), _dp(Wt, F64, "Wt"), _dp(b, F64, "b"), n, Cin, Cout, D, H, W, kd, kh, kw,
                                             _dp(out), _stream()), "bx_ts_conv_forward")
    return out


def conv_backward(x, dy, Wt, D, H, W, kd, kh, kw, want_dx=True):
    """float64 valid 3-D convolution backward: x [n, Cin/4, D*H*W, 4], dy [n, Cout/4, OD*OH*OW, 4], Wt [T, Cin, Cout] ->
    (dx like x or None, dW [T, Cin, Cout])."""
    n, Cin, Cout = _conv_shapes("conv_backward", x, Wt, D, H, W, kd, kh, kw)
    _ts_shape("conv_backward", dy, (n, Cout // 4, (D - kd + 1) * (H - kh + 1) * (W - kw + 1), 4), "dy")
    T = kd * kh * kw
    wpart = torch.empty(_splits() * T * Cin * Cout, dtype=F64, device=x.device)
    dW = torch.empty((T, Cin, Cout), dtype=F64, device=x.device)
    dx = torch.empty_like(x) if want_dx else None
    _check(load_library().bx_ts_conv_backward(_dp(x, F64, "x"), _dp(dy, F64, "dy"), _dp(Wt, F64, "Wt"), n, Cin, Cout, D, H, W, kd, kh, kw,
                                              _dp(dx), _dp(wpart), _dp(dW), _stream()), "bx_ts_conv_backward")
    return dx, dW


# --------------------------------------------------------------------------- #
# the Desc-stage training step (bx_train_desc.cu): float64 activations channel-blocked [n, C/4, S, 4]; a cylindrical
# raster has 140 = 7 x 20 positions per depth slice
# --------------------------------------------------------------------------- #
CYL_S = 140
U8 = torch.uint8


def _cyl_shapes(what, x, Din, C=None):
    n, G, S = _ts_blocked(what, x)
    if x.dtype != F64:
        raise BufferXError(f"{what}: x must be float64, got {x.dtype}")
    if S != Din * CYL_S:
        raise BufferXError(f"{what}: x holds {S} positions per channel, a cylindrical raster of depth {Din} has {Din * CYL_S}")
    if C is not None and 4 * G != C:
        raise BufferXError(f"{what}: x has {4 * G} channels, expected {C}")
    return n, 4 * G


def cyl_forward(x, Wt, b, Din):
    """One Cylindrical_Net convolution on the fp64 tensor cores: x [n, Cin/4, Din*140, 4], Wt [Din*9, Cin, Cout], b [Cout]
    (float64) -> [n, Cout/4, 140, 4].  Circular azimuth / zero elevation padding is applied by the kernel."""
    n, Cin = _cyl_shapes("cyl_forward", x, Din)
    if not isinstance(Wt, torch.Tensor) or Wt.dim() != 3:
        raise BufferXError(f"cyl_forward: Wt must be [Din*9, Cin, Cout], got {tuple(Wt.shape) if isinstance(Wt, torch.Tensor) else Wt}")
    Cout = Wt.shape[2]
    _ts_shape("cyl_forward", Wt, (Din * 9, Cin, Cout), "Wt")
    _ts_shape("cyl_forward", b, (Cout,), "b")
    if Cin % 16 or Cout % 8:
        raise BufferXError(f"cyl_forward: Cin = {Cin} must be a multiple of 16 and Cout = {Cout} of 8")
    out = torch.empty((n, Cout // 4, CYL_S, 4), dtype=F64, device=x.device)
    _check(load_library().bx_td_cyl_forward(_dp(x, F64, "x"), _dp(Wt, F64, "Wt"), _dp(b, F64, "b"), n, Cin, Cout, Din, _dp(out), _stream()),
           "bx_td_cyl_forward")
    return out


def cyl_backward(x, dy, Wt, Din, want_dx=True):
    """Backward of cyl_forward: x [n, Cin/4, Din*140, 4], dy [n, Cout/4, 140, 4], Wt [Din*9, Cin, Cout] -> (dx like x or
    None, dW [Din*9, Cin, Cout]); the bias gradient is channel_sums(dy)[0]."""
    n, Cin = _cyl_shapes("cyl_backward", x, Din)
    if not isinstance(Wt, torch.Tensor) or Wt.dim() != 3:
        raise BufferXError(f"cyl_backward: Wt must be [Din*9, Cin, Cout], got {tuple(Wt.shape) if isinstance(Wt, torch.Tensor) else Wt}")
    Cout = Wt.shape[2]
    _ts_shape("cyl_backward", Wt, (Din * 9, Cin, Cout), "Wt")
    _ts_shape("cyl_backward", dy, (n, Cout // 4, CYL_S, 4), "dy")
    if Cout % 16 or Cin % 8:
        raise BufferXError(f"cyl_backward: Cin = {Cin} must be a multiple of 8 and Cout = {Cout} of 16")
    lib = load_library()
    wpart = torch.empty(_splits() * Din * 9 * Cin * Cout, dtype=F64, device=x.device)
    dW = torch.empty((Din * 9, Cin, Cout), dtype=F64, device=x.device)
    _check(lib.bx_td_cyl_wgrad(_dp(x, F64, "x"), _dp(dy, F64, "dy"), n, Cin, Cout, Din, _dp(wpart), _dp(dW), _stream()), "bx_td_cyl_wgrad")
    dx = None
    if want_dx:
        dx = torch.empty_like(x)
        _check(lib.bx_td_cyl_dgrad(_dp(dy, F64, "dy"), _dp(Wt, F64, "Wt"), n, Cin, Cout, Din, _dp(dx), _stream()), "bx_td_cyl_dgrad")
    return dx, dW


def _pnt_inv(what, inv):
    if not isinstance(inv, torch.Tensor) or inv.dim() != 4 or inv.shape[3] != 3 or inv.numel() == 0 or inv.shape[2] > 255:
        raise BufferXError(f"{what}: inv must be [K, V, nv, 3] with 1 <= nv <= 255, got "
                           f"{tuple(inv.shape) if isinstance(inv, torch.Tensor) else type(inv).__name__}")
    return inv.shape[0], inv.shape[1], inv.shape[2]


def pnt_forward(inv, W, b, scale, shift):
    """The point layer in training mode on the de-rotated samples inv [K, V, nv, 3] fp32: W [16, 3], b, scale, shift [16]
    (float64; x^ = (W inv + b) scale + shift) -> (feat [K, 4, V, 4] float64 = max over the samples of relu(x^), arg [K, 16, V]
    uint8 = the first maximal sample)."""
    K, V, nv = _pnt_inv("pnt_forward", inv)
    _ts_shape("pnt_forward", W, (16, 3), "W")
    for name, t in (("b", b), ("scale", scale), ("shift", shift)):
        _ts_shape("pnt_forward", t, (16,), name)
    feat = torch.empty((K, 4, V, 4), dtype=F64, device=inv.device)
    arg = torch.empty((K, 16, V), dtype=U8, device=inv.device)
    _check(load_library().bx_td_pnt_forward(_dp(inv, F32, "inv"), _dp(W, F64, "W"), _dp(b, F64, "b"), _dp(scale, F64, "scale"),
                                            _dp(shift, F64, "shift"), K, V, nv, _dp(feat), _dp(arg), _stream()), "bx_td_pnt_forward")
    return feat, arg


def pnt_backward(inv, arg, dfeat, W, b, mean, rstd, gamma, scale, shift, mo9):
    """Backward of pnt_forward from dfeat (like feat): -> float64 [16, 6] = dW (3 columns), db, dgamma, dbeta.  mean, rstd:
    the batch statistics; gamma: the BatchNorm weight; mo9: moments3(inv)."""
    K, V, nv = _pnt_inv("pnt_backward", inv)
    _ts_shape("pnt_backward", arg, (K, 16, V), "arg")
    _ts_shape("pnt_backward", dfeat, (K, 4, V, 4), "dfeat")
    _ts_shape("pnt_backward", W, (16, 3), "W")
    for name, t in (("b", b), ("mean", mean), ("rstd", rstd), ("gamma", gamma), ("scale", scale), ("shift", shift)):
        _ts_shape("pnt_backward", t, (16,), name)
    _ts_shape("pnt_backward", mo9, (9,), "mo9")
    partial = torch.empty(_splits() * 80, dtype=F64, device=inv.device)
    out = torch.empty((16, 6), dtype=F64, device=inv.device)
    _check(load_library().bx_td_pnt_backward(_dp(inv, F32, "inv"), _dp(arg, U8, "arg"), _dp(dfeat, F64, "dfeat"), _dp(W, F64, "W"),
                                             _dp(b, F64, "b"), _dp(mean, F64, "mean"), _dp(rstd, F64, "rstd"), _dp(gamma, F64, "gamma"),
                                             _dp(scale, F64, "scale"), _dp(shift, F64, "shift"), _dp(mo9, F64, "mo9"), K, V, nv, _dp(partial),
                                             _dp(out), _stream()), "bx_td_pnt_backward")
    return out


def cross_sums(X, D):
    """X [n, Ca/4, S, 4], D [n, Cb/4, S, 4] float64 -> [Ca, Cb] = sum over samples and positions of X[a] D[b]."""
    n, Ga, S = _ts_blocked("cross_sums", X, "X")
    _ts_blocked("cross_sums", D, "D")
    _ts_shape("cross_sums", D, (n, D.shape[1], S, 4), "D")
    Ca, Cb = 4 * Ga, 4 * D.shape[1]
    partial = torch.empty(_splits() * Ca * Cb, dtype=F64, device=X.device)
    out = torch.empty((Ca, Cb), dtype=F64, device=X.device)
    _check(load_library().bx_td_cross_sums(_dp(X, F64, "X"), _dp(D, F64, "D"), n, Ca, Cb, S, _dp(partial), _dp(out), _stream()),
           "bx_td_cross_sums")
    return out


def pool_forward(x, w):
    """x [K, 8, 140, 4], w [K, 1, 140, 4] (the attention in channel 0), float64 -> (f [K, 32] float64, desc [K, 32],
    equi [K, 32, 7, 20] fp32)."""
    _ts_shape("pool_forward", x, (x.shape[0] if isinstance(x, torch.Tensor) else -1, 8, CYL_S, 4), "x")
    K = x.shape[0]
    _ts_shape("pool_forward", w, (K, 1, CYL_S, 4), "w")
    f = torch.empty((K, 32), dtype=F64, device=x.device)
    desc = torch.empty((K, 32), dtype=F32, device=x.device)
    equi = torch.empty((K, 32, 7, 20), dtype=F32, device=x.device)
    _check(load_library().bx_td_pool_forward(_dp(x, F64, "x"), _dp(w, F64, "w"), K, _dp(f), _dp(desc), _dp(equi), _stream()), "bx_td_pool_forward")
    return f, desc, equi


def pool_backward(x, w, f, ddesc, dequi):
    """Backward of pool_forward from ddesc [K, 32], dequi [K, 32, 7, 20] (fp32) -> (dx like x, dw like w)."""
    _ts_shape("pool_backward", x, (x.shape[0] if isinstance(x, torch.Tensor) else -1, 8, CYL_S, 4), "x")
    K = x.shape[0]
    _ts_shape("pool_backward", w, (K, 1, CYL_S, 4), "w")
    _ts_shape("pool_backward", f, (K, 32), "f")
    _ts_shape("pool_backward", ddesc, (K, 32), "ddesc")
    _ts_shape("pool_backward", dequi, (K, 32, 7, 20), "dequi")
    dx = torch.empty_like(x)
    dw = torch.empty_like(w)
    _check(load_library().bx_td_pool_backward(_dp(x, F64, "x"), _dp(w, F64, "w"), _dp(f, F64, "f"), _dp(ddesc, F32, "ddesc"),
                                              _dp(dequi, F32, "dequi"), K, _dp(dx), _dp(dw), _stream()), "bx_td_pool_backward")
    return dx, dw


def equi_match_backward(d1, d2, dcor):
    """Gradients of equi_match(d1, d2) [B, L] with respect to d1 and d2 ([B, C, K, L] fp32) from dcor [B, L]."""
    if not isinstance(d1, torch.Tensor) or d1.dim() != 4:
        raise BufferXError(f"equi_match_backward: d1 must be [B, C, K, L], got {tuple(d1.shape) if isinstance(d1, torch.Tensor) else d1}")
    B, C, K, L = d1.shape
    _ts_shape("equi_match_backward", d2, (B, C, K, L), "d2")
    _ts_shape("equi_match_backward", dcor, (B, L), "dcor")
    g1, g2 = torch.empty_like(d1), torch.empty_like(d2)
    if B == 0:
        return g1, g2
    _check(load_library().bx_td_equi_match_backward(_dp(d1, F32, "d1"), _dp(d2, F32, "d2"), _dp(dcor, F32, "dcor"), B, C, K, L, _dp(g1),
                                                    _dp(g2), _stream()), "bx_td_equi_match_backward")
    return g1, g2


# --------------------------------------------------------------------------- #
def dp_mean(gathered: torch.Tensor):
    """The cross-rank mean of one sharded training step (driver.train_sharded): ``gathered`` [W, n + 1] fp32 CUDA holds
    one record per rank, n values then the rank's contribution flag.  Returns (out [n] fp32, count [1] int32 on the
    device): out[i] = fl32((sum over the rows with a non-zero flag, in ascending row order, of (double) gathered[r, i]) /
    count); out is left unwritten (torch.empty) when count is 0."""
    if not isinstance(gathered, torch.Tensor) or gathered.dim() != 2 or gathered.shape[0] < 1 or gathered.shape[1] < 1:
        raise BufferXError(f"dp_mean: gathered must be a [W >= 1, n + 1 >= 1] tensor, got "
                           f"{tuple(gathered.shape) if isinstance(gathered, torch.Tensor) else type(gathered).__name__}")
    W, n = gathered.shape[0], gathered.shape[1] - 1
    ptr = _dp(gathered, F32, "gathered")
    out = torch.empty(n, dtype=F32, device=gathered.device)
    count = torch.empty(1, dtype=I32, device=gathered.device)
    # an empty tensor's data_ptr() may be NULL, which the C-ABI refuses: with n = 0 nothing is written through `out`
    _check(load_library().bx_dp_mean(ptr, W, n, _dp(out) if n else _dp(count), _dp(count), _stream()), "bx_dp_mean")
    return out, count
