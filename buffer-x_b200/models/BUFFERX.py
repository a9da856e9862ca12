"""BufferX on H100: the per-pair registration ``forward()``, in eval mode the training stages' validation forward, and in
training mode the Pose stage's step (batch-statistics BatchNorm, ``pred_ind`` differentiable in ``Pose.conv``) and the Desc
stage's step (``src_des``, ``tgt_des`` and ``equi_score`` differentiable in the descriptor network's parameters).

Mirrors ``BufferX`` of /root/reference/models/BUFFERX.py (constructor :72-84, inference branch of
``forward`` :257-467, ``mutual_matching`` :469-496, ``post_refinement`` :522-556): same attribute names
(``Desc``, ``Pose``, ``equi_match``, ``pose_estimator``), same ``state_dict()`` keys, same return tuple
``(pose 4x4, [desc_s, pose_s, pose_optim_s], num_inliers, num_mutual_inliers, num_inlier_ind,
scales_used)``.  Differences that do not change results:
  * FPS runs once per cloud for max(num_points_radius_estimate, num_fps) points -- the reference's
    per-scale calls return the same indices and FPS(k) is a prefix of FPS(k') (SURVEY 8.1 item 8);
  * the radius histogram is built once and serves every scale's bisection, on the device (a larger cloud of more than
    200000 points keeps the reference's per-scale sub-sample: one draw and one histogram per scale);
  * data-dependent sizes stay in device counters, so the whole pair is enqueued without a host round
    trip; the host reads one small result block at the end (early-exit mode in ``forward`` adds one read after scale 0;
    ``forward_async`` decides early exit on the device).

Throughput API on top of the reference surface (CUDA streams + graphs instead of a tracing compiler):
  * ``enable_cuda_graphs(True)``: the enqueue of a pair is captured once per (Ns, Nt, aligned) shape and
    replayed -- one graph launch instead of ~150 kernel launches; with ``size_classes=True`` once per
    (C_src, C_tgt, aligned) capacity, the true point counts read by the N-dependent kernels from the device, so
    a stream of pairs of every size replays a handful of graphs (``large_classes=True`` extends this to clouds of more
    than 200000 points, their radius sub-sample drawn on the host at launch);
  * ``forward_async(data_source) -> handle`` / ``handle.result()``: several pairs in flight on separate
    streams (FPS is a latency-bound 16-SM kernel; a second pair's convolutions fill the other SMs).
    With ``cfg.match.enable_early_exit`` the scale-0 RANSAC result gates the later scales on the device
    (``_enqueue_device_exit``), so early-exit pairs are captured and replayed too.
"""
import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from bufferx_b200 import ops
from . import patchnet as pn
from .patch_embedder import MiniSpinNet
from .pose_estimator import PoseEstimator


def _azimuth_index_list(azi_n):
    init = np.arange(azi_n)
    return np.array([np.concatenate([init[azi_n - i:], init[:azi_n - i]]) for i in range(azi_n)])


class EquiMatch(nn.Module):
    """Training-time SO(2) matching score (reference BUFFERX.py:16-36); kept for API parity, plain torch."""

    def __init__(self, config):
        super().__init__()
        self.azi_n = config.patch.azi_n
        self.index_list = _azimuth_index_list(self.azi_n)

    def forward(self, Des1, Des2):
        B, C, K, L = Des1.shape
        idx = torch.from_numpy(self.index_list).to(Des1.device).reshape(-1)
        d1 = Des1[:, :, :, idx].reshape(B, C, K, self.azi_n, self.azi_n).permute(0, 1, 3, 2, 4).reshape(B, C, -1, K * L)
        return torch.einsum("bfag,bfg->ba", d1, Des2.reshape(B, C, K * L))


class _EquiMatchFn(torch.autograd.Function):
    """EquiMatch score of two equivariant maps on bx_equi_match, differentiable in both (bx_td_equi_match_backward)."""

    @staticmethod
    def forward(ctx, d1, d2):
        ctx.save_for_backward(d1, d2)
        return ops.equi_match(d1, d2)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        d1, d2 = ctx.saved_tensors
        return ops.equi_match_backward(d1, d2, g.float().contiguous())


class CostVolume(nn.Module):
    """SO(2) cost volume + CostNet (reference BUFFERX.py:39-69); state_dict prefix ``conv.``."""

    def __init__(self, config):
        super().__init__()
        self.azi_n = config.patch.azi_n
        self.index_list = _azimuth_index_list(self.azi_n)
        self.conv = pn.CostNet(inchan=32, dim=20)

    def logits(self, equi_s, equi_t, s_mids, t_mids, d_M, maxM):
        """Full-height maps [K,32,7,20] + match lists; rows 1..ele_n-2 are sliced inside the kernel."""
        return self.conv.forward_matches(equi_s, equi_t, s_mids, t_mids, d_M, maxM)


class _Timer:
    def __init__(self, enabled):
        self.enabled = enabled
        self.total = 0.0
        if enabled:
            self.a, self.b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def tic(self):
        if self.enabled:
            self.a.record()

    def toc(self):
        if self.enabled:
            self.b.record()
            self.b.synchronize()
            self.total += self.a.elapsed_time(self.b) / 1000.0


class _PairSlot:
    """Static buffers + (optionally) a captured CUDA graph for one (C_src, C_tgt, aligned, early-exit setting) on its own
    stream.  C_src / C_tgt are the capacities of the cloud buffers.  An exact-shape slot (``counted`` False) serves the pairs
    of exactly that shape and runs the kernels without point counts; a size-class slot (``counted`` True) serves every pair
    whose clouds fit the capacities: the true counts are copied to the device before each replay and the N-dependent
    kernels (FPS, radius histogram, permutation, patch gathering) stop at them, so the padding rows are never read.
    A large-class slot (``subsample`` True: a size-class slot whose larger capacity exceeds MAX_CLASS_POINTS) also holds the
    reference's [S, 200000] radius sub-samples, one per scale, drawn at launch from torch's CPU generator in scale order as
    eager ``forward`` draws them."""

    def __init__(self, model, Cs, Ct, aligned, use_graph, counted=False, subsample=False):
        cfg = model.config
        self.model, self.Cs, self.Ct, self.aligned, self.counted = model, Cs, Ct, aligned, counted
        self.n_s, self.n_t = Cs, Ct
        dev = next(model.parameters()).device
        self.dev = dev
        S = cfg.patch.num_scales
        self.stream = torch.cuda.Stream(device=dev)
        self.xyz = torch.empty((Cs + Ct, 3), dtype=torch.float32, device=dev)      # both clouds back to back: the FPS input
        self.src, self.tgt = self.xyz[:Cs], self.xyz[Cs:]
        self.perm_s = torch.empty((S, Cs), dtype=torch.int32, device=dev)
        self.perm_t = torch.empty((S, Ct), dtype=torch.int32, device=dev)
        self.h_perm_s = torch.empty((S, Cs), dtype=torch.int32).pin_memory()
        self.h_perm_t = torch.empty((S, Ct), dtype=torch.int32).pin_memory()
        self.h_src = torch.empty((Cs, 3), dtype=torch.float32).pin_memory()
        self.h_tgt = torch.empty((Ct, 3), dtype=torch.float32).pin_memory()
        self.counts = torch.tensor([Cs, Ct], dtype=torch.int32, device=dev) if counted else None
        self.h_counts = torch.empty(2, dtype=torch.int32).pin_memory() if counted else None
        # index 0 is valid in any cloud: the warm-up and the capture read it before the first launch draws
        self.sub = torch.zeros((S, ops.RADIUS_SUBSAMPLE), dtype=torch.int32, device=dev) if subsample else None
        self.h_sub = torch.empty((S, ops.RADIUS_SUBSAMPLE), dtype=torch.int32).pin_memory() if subsample else None
        self.h_tail = None
        self.done = torch.cuda.Event()
        self.graph = None
        self.tail = None
        self.busy = False
        if use_graph:
            with torch.cuda.device(dev), torch.cuda.stream(self.stream):
                self.xyz.zero_()
                base = torch.arange(max(Cs, Ct), dtype=torch.int32, device=dev)
                self.perm_s.copy_(base[:Cs].expand(S, Cs)); self.perm_t.copy_(base[:Ct].expand(S, Ct))
                self.src[:, 0] = torch.linspace(1, 2, Cs, device=dev)      # any valid cloud: warm-up sets kernel attributes
                self.tgt[:, 0] = torch.linspace(1, 2, Ct, device=dev)
                self._enqueue()                                            # eager warm-up on this stream
            self.stream.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.device(dev), torch.cuda.graph(self.graph, stream=self.stream):
                self.tail = self._enqueue()
            # the graph replays the device pointers of the folded weights it captured: keep those tensors alive even when
            # a later in-place weight change makes the caches rebuild (load_state_dict / .to() drop the slots themselves)
            self.captured_weights = (model.Desc.prepared(dev), model.Desc.conv_net.folded(), model.Pose.conv.folded())
        # pinned landing buffer for the result block
        n_tail = 18 + (S + 1) + 1 + 1 + 16 + 1   # RANSAC block, scale offsets, consensus count, scales used, refined pose, fp16-range flag
        self.h_tail = torch.empty(n_tail, dtype=torch.float64).pin_memory()

    def _enqueue(self):
        perms = [(self.perm_s[i], self.perm_t[i]) for i in range(self.perm_s.shape[0])]
        return self.model._enqueue(self.src, self.tgt, self.aligned, perms, None, False, device_exit=True, counts=self.counts,
                                   xyz=self.xyz, sub=self.sub)[0]

    def launch(self, data_source, perms):
        """H2D of the inputs (pinned staging when they arrive as host arrays), the pair, D2H of the result."""
        xs, xt = torch.as_tensor(data_source["src_fds_pcd"]).reshape(-1, 3), torch.as_tensor(data_source["tgt_fds_pcd"]).reshape(-1, 3)
        n_s, n_t = xs.shape[0], xt.shape[0]
        if n_s > self.Cs or n_t > self.Ct or (not self.counted and (n_s, n_t) != (self.Cs, self.Ct)):
            raise ops.BufferXError(f"forward_async: a ({n_s}, {n_t})-point pair does not fit a slot of capacity ({self.Cs}, {self.Ct})")
        self.n_s, self.n_t = n_s, n_t
        # CUDA inputs may still be in flight on the caller's stream (`.cuda(non_blocking=True)`, a voxel_down_sample
        # kernel): the slot stream starts after everything the caller has enqueued so far, and the caching allocator is
        # told that the slot stream reads them (so the memory is not handed out again before the copy has run).
        self.stream.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.device(self.dev), torch.cuda.stream(self.stream):
            # only the first n rows are written: the padding of a size-class buffer keeps whatever the last pair left there
            for dst, hbuf, x in ((self.src[:n_s], self.h_src[:n_s], xs), (self.tgt[:n_t], self.h_tgt[:n_t], xt)):
                if x.is_cuda:
                    x.record_stream(self.stream)
                    dst.copy_(x, non_blocking=True)
                else:
                    if x.is_pinned():
                        dst.copy_(x, non_blocking=True)
                    else:
                        hbuf.copy_(x)
                        dst.copy_(hbuf, non_blocking=True)
            S = self.perm_s.shape[0]
            on_device = perms is not None and isinstance(perms[0][0], torch.Tensor) and perms[0][0].is_cuda
            for i in range(S):
                if perms is None:   # the reference's host draws, in its order (src then tgt, per scale)
                    self.h_perm_s[i, :n_s].copy_(torch.from_numpy(np.random.choice(n_s, n_s, replace=False).astype(np.int32)))
                    self.h_perm_t[i, :n_t].copy_(torch.from_numpy(np.random.choice(n_t, n_t, replace=False).astype(np.int32)))
                else:
                    ps, pt = perms[i]
                    if on_device:
                        ps.record_stream(self.stream); pt.record_stream(self.stream)
                        self.perm_s[i, :n_s].copy_(ps, non_blocking=True); self.perm_t[i, :n_t].copy_(pt, non_blocking=True)
                        continue
                    self.h_perm_s[i, :n_s].copy_(torch.as_tensor(ps, dtype=torch.int32)); self.h_perm_t[i, :n_t].copy_(torch.as_tensor(pt, dtype=torch.int32))
            if not on_device:
                if (n_s, n_t) == (self.Cs, self.Ct):
                    self.perm_s.copy_(self.h_perm_s, non_blocking=True)
                    self.perm_t.copy_(self.h_perm_t, non_blocking=True)
                else:           # rows of a capacity buffer: the first n entries of each
                    for i in range(S):
                        self.perm_s[i, :n_s].copy_(self.h_perm_s[i, :n_s], non_blocking=True)
                        self.perm_t[i, :n_t].copy_(self.h_perm_t[i, :n_t], non_blocking=True)
            if self.counted:
                self.h_counts[0], self.h_counts[1] = n_s, n_t
                self.counts.copy_(self.h_counts, non_blocking=True)
            if self.sub is not None and max(n_s, n_t) > ops.RADIUS_SUBSAMPLE:
                # eager forward's draws (reference BUFFERX.py:664-665, one per scale) on the cloud it picks: the source iff
                # n_s > n_t.  All S are drawn, also when the device then exits after scale 0 (the reference draws one)
                for i in range(S):
                    self.h_sub[i].copy_(torch.randint(0, n_s if n_s > n_t else n_t, (ops.RADIUS_SUBSAMPLE,)))
                self.sub.copy_(self.h_sub, non_blocking=True)
            if self.graph is not None:
                self.graph.replay()
                tail = self.tail
            else:
                tail = self._enqueue()
            self.h_tail.copy_(tail, non_blocking=True)
            self.done.record(self.stream)
        self.busy = True
        return self

    def result(self):
        self.done.synchronize()
        self.busy = False
        out = self.model._decode(self.h_tail.clone(), [0.0, 0.0, 0.0])
        if self.model._overflow:            # an activation left fp16 range: this pair is recomputed on the TF32 kernel
            n_s, n_t = self.n_s, self.n_t   # the exact clouds and permutations, not the capacity buffers
            return self.model._rerun_tf32(dict(src_fds_pcd=self.src[:n_s].clone(), tgt_fds_pcd=self.tgt[:n_t].clone(), is_aligned_to_global_z=self.aligned),
                                          [(self.perm_s[i, :n_s].clone(), self.perm_t[i, :n_t].clone()) for i in range(self.perm_s.shape[0])], None)
        return out


class BufferX(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.config.stage = config.stage
        self.Desc = MiniSpinNet(config)
        self.Pose = CostVolume(config)
        self.equi_match = EquiMatch(config)
        self.Pose.conv.flag_source = self.Desc.conv_net.overflow_flag      # one sticky fp16-range flag per model
        if config.stage == "test":
            self.pose_estimator = PoseEstimator(config)
        self._use_graphs = False
        self._slots = {}
        self._slots_per_shape = 2
        self._size_classes = False
        self._large_classes = False
        self._rr = {}

    def get_parameter(self):
        return list(self.parameters())

    # Captured graphs bake in the device pointers of the folded weights (and live on one device): anything that can
    # replace the parameters -- load_state_dict(), .to()/.cuda()/.half()/.float() -- drops the captured slots and the
    # per-stream RANSAC workspaces, so the next forward re-captures against the new buffers.
    def _drop_captured_state(self):
        for slots in self._slots.values():
            for sl in slots:
                if sl.busy:
                    sl.done.synchronize()
        self._slots.clear()
        self._rr.clear()
        pe = getattr(self, "pose_estimator", None)
        if pe is not None and hasattr(pe, "_ws"):
            pe._ws.clear()

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        if hasattr(self, "_slots"):
            self._drop_captured_state()
        return out

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        self._drop_captured_state()
        for m in self.modules():
            if hasattr(m, "invalidate"):
                m.invalidate()
        return out

    # ------------------------------------------------------------------------------------------------
    def mutual_matching(self, src_des, tgt_des):
        """[M,C],[N,C] -> (s_mids, t_mids) int64, like the reference (one device->host read for M)."""
        s, t, dM, _, _ = ops.mutual_nn(src_des.contiguous(), tgt_des.contiguous())
        M = int(dM.item())
        return s[:M].long(), t[:M].long()

    def post_refinement(self, initial_trans, src_keypts, tgt_keypts, weights=None):
        """[1,4,4], [1,n,3], [1,n,3] -> [1,4,4] (reference BUFFERX.py:522-556)."""
        assert initial_trans.shape[0] == 1
        ss, tt = src_keypts[0].contiguous(), tgt_keypts[0].contiguous()
        n = ss.shape[0]
        d_n = torch.tensor([n], dtype=torch.int32, device=ss.device)
        T_in = initial_trans[0].to(torch.float64).reshape(16).contiguous()
        T, _ = ops.refine(ss, tt, d_n, n, T_in, self.config.match.dist_th)
        return T.view(1, 4, 4)

    # ------------------------------------------------------------------------------------------------
    def enable_cuda_graphs(self, flag=True, slots_per_shape=2, size_classes=False, large_classes=False):
        """Capture the per-pair enqueue once per slot key and replay it (no effect on results, except for a pair whose larger
        cloud has more than 200000 points on an exact-shape slot: the capture draws its radius sub-sample on the device, not
        from torch's CPU generator as eager ``forward`` and the reference do); ``forward`` then runs through the same slots as
        ``forward_async`` (unless early exit, timing or debug is on).

        ``size_classes=False``: slots are keyed by the exact (Ns, Nt, aligned) shape (plus the early-exit setting), so a stream
        whose pairs all differ in size captures a graph for almost every pair.  ``size_classes=True``: each cloud is given a
        capacity, its size class (``ops.fps_size_class``: the largest point count with the same FPS launch configuration),
        slots are keyed by (C_src, C_tgt, aligned) and every pair whose clouds fit replays the class graph with its true
        point counts on the device -- results bit-identical to the exact-shape route.  A pair whose larger cloud has more
        than 200000 points keeps an exact-shape slot (the reference sub-samples such a cloud with a draw sized by N), unless
        ``large_classes=True``: such pairs then get size-class slots too (``ops.fps_large_size_class``: above 524288 points,
        capacities at most 1.25x the cloud, up to 1638400 points), and each launch draws the 200000-index sub-sample on the
        host from torch's CPU generator (one draw per scale, in scale order, as the reference draws them) and uploads them
        with the counts -- results byte-identical to eager ``forward`` with the same ``perms`` and the same generator state,
        graphs on or off.  With early exit the device decides after the launch, so a launch always makes all S draws: after
        a pair that exits at scale 0 the generator is S - 1 draws ahead of the reference's (as the NumPy permutations are,
        see ``_graphable``); the scales that run use the reference's draws.
        ``slots_per_shape`` slots (pairs in flight) are kept per key.  These options also apply to ``forward_async``
        without graphs."""
        if large_classes and not size_classes:
            raise ValueError("enable_cuda_graphs: large_classes=True extends size_classes=True; set both")
        self._use_graphs = bool(flag)
        self._slots_per_shape = int(slots_per_shape)
        self._size_classes = bool(size_classes)
        self._large_classes = bool(large_classes)
        self._slots.clear()
        self._rr.clear()
        return self

    def _graphable(self):
        """Whether ``forward`` may route through the slots.  Early exit stays on the host decision in ``forward``: only that
        reproduces the reference's NumPy draw order (scales 1..S-1 draw their permutations only when the pair does not exit),
        the drop-in contract of ``forward``; likewise torch's CPU generator, which ``forward`` rewinds to after scale 0's radius
        sub-sample when a pair above 200000 points exits.  ``forward_async`` draws all 2*S permutations (and S sub-samples) at
        launch and decides on the device."""
        cfg = self.config
        return not cfg.match.get("enable_early_exit", True) and not cfg.test.get("enable_timing", False)

    def _exit_key(self):
        m = self.config.match
        return (True, int(m.get("early_exit_min_inliers", 15))) if m.get("enable_early_exit", True) else (False, None)

    MAX_GRAPH_SHAPES = 8      # graphs are per slot key; least recently used keys are dropped beyond this
    # larger clouds are sub-sampled by a draw sized by N (reference BUFFERX.py:664-665): exact slots, unless large_classes
    MAX_CLASS_POINTS = 200000

    def _slot_key(self, Ns, Nt, aligned):
        """(slot key, capacities, counted) of a pair.  The early-exit threshold is baked into a captured gate launch: a
        graph is never replayed under another setting."""
        if self._size_classes and self._large_classes:
            Cs, Ct = ops.fps_large_size_class(Ns), ops.fps_large_size_class(Nt)
            return (Cs, Ct, bool(aligned)) + self._exit_key(), Cs, Ct, True
        if self._size_classes and max(Ns, Nt) <= self.MAX_CLASS_POINTS:
            Cs, Ct = ops.fps_size_class(Ns), ops.fps_size_class(Nt)
            return (Cs, Ct, bool(aligned)) + self._exit_key(), Cs, Ct, True
        return (Ns, Nt, bool(aligned)) + self._exit_key(), Ns, Nt, False

    def _evict(self, key):
        pe = getattr(self, "pose_estimator", None)
        for sl in self._slots[key]:
            if pe is not None and hasattr(pe, "_ws"):
                pe._ws.pop((str(sl.dev), sl.stream.cuda_stream), None)
        del self._slots[key]
        self._rr.pop(key, None)

    def _slot(self, Ns, Nt, aligned):
        key, Cs, Ct, counted = self._slot_key(Ns, Nt, aligned)
        if key in self._slots and any(sl.counted != counted for sl in self._slots[key]):
            # an exact shape above MAX_CLASS_POINTS that equals a size class: the two kinds of slot never share a key
            if any(sl.busy for sl in self._slots[key]):
                raise ops.BufferXError("forward_async: collect the pending results before launching this pair")
            self._evict(key)
        if key not in self._slots and len(self._slots) >= self.MAX_GRAPH_SHAPES:
            # datasets with a different size for every pair would otherwise pin one set of graph pools per pair; for
            # those, use size classes (`enable_cuda_graphs(True, size_classes=True)`)
            for old in list(self._slots):
                if all(not sl.busy for sl in self._slots[old]):
                    self._evict(old)
                    break
        else:
            if key in self._slots:          # keep insertion order = recency order
                self._slots[key] = self._slots.pop(key)
        lst = self._slots.setdefault(key, [])
        i = self._rr.get(key, 0)
        if len(lst) < self._slots_per_shape:
            subsample = counted and self._large_classes and max(Cs, Ct) > self.MAX_CLASS_POINTS
            lst.append(_PairSlot(self, Cs, Ct, aligned, self._use_graphs, counted, subsample))
            slot = lst[-1]
        else:
            slot = lst[i % len(lst)]
            if slot.busy:
                raise ops.BufferXError("forward_async: collect the oldest handle's result() before launching more pairs")
        self._rr[key] = i + 1
        return slot

    @staticmethod
    def _cloud_sizes(data_source):
        """(Ns, Nt) of a pair; refuses, before anything is launched, a cloud larger than the patch gatherer's shared-memory
        bitmap holds (ops.FPS_LARGE_MAX_POINTS points)."""
        sizes = tuple(int(np.prod(np.shape(data_source[k])[:-1])) for k in ("src_fds_pcd", "tgt_fds_pcd"))
        for name, n in zip(("source", "target"), sizes):
            if n > ops.FPS_LARGE_MAX_POINTS:
                raise ops.BufferXError(f"BufferX: the {name} cloud has {n} points; clouds of up to {ops.FPS_LARGE_MAX_POINTS} "
                                       "points are supported (the patch gatherer's shared-memory bitmap holds one bit per point)")
        return sizes

    def forward_async(self, data_source, perms=None):
        """Enqueue one pair on a slot stream; returns a handle whose ``result()`` is the forward tuple.  Without ``perms`` the
        2*S permutations are drawn from NumPy's global RNG at launch, also when early exit stops the pair after scale 0.
        The slot is chosen by the pair's shape, or by its clouds' size classes after
        ``enable_cuda_graphs(..., size_classes=True)``; either way the result is that of eager ``forward`` with the same
        ``perms``, except on a captured exact-shape slot for a pair whose larger cloud has more than 200000 points, whose
        radius sub-sample the capture draws on the device.  A large-class slot (``large_classes=True``) draws it at launch
        from torch's CPU generator, as eager ``forward`` does."""
        if self.config.test.get("enable_timing", False):
            raise ops.BufferXError("forward_async needs timing disabled (the per-stage timers require host round trips)")
        Ns, Nt = self._cloud_sizes(data_source)
        return self._slot(Ns, Nt, bool(data_source["is_aligned_to_global_z"])).launch(data_source, perms)

    # ------------------------------------------------------------------------------------------------
    def _enqueue(self, src, tgt, aligned, perms, ransac_seed, debug, timers=None, device_exit=False, counts=None, xyz=None, sub=None):
        """Everything of one pair on the current stream, no host synchronisation unless early exit is on and the decision is
        the host's (``device_exit`` False: ``forward``).  Returns (tail block on the device, debug dict).
        ``counts`` (size-class slots): [2] int32 CUDA point counts; src / tgt are then capacity buffers whose first counts
        rows are the clouds, and ``perms`` rows likewise.  ``sub`` (large-class slots, with ``counts``): [S, 200000] int32 CUDA
        radius sub-samples, row i read by scale i when the larger cloud has more than 200000 points; without it the counted
        clouds have at most MAX_CLASS_POINTS points.  ``xyz``: src and tgt back to back, when the caller holds them so (saves the concatenation
        before FPS)."""
        cfg = self.config
        dev = src.device
        Ns, Nt = src.shape[0], tgt.shape[0]
        Kr, K = cfg.patch.num_points_radius_estimate, cfg.patch.num_fps
        S = cfg.patch.num_scales
        thresholds = cfg.patch.search_radius_thresholds
        assert S == len(thresholds), f"num_scales {S} != num_thresholds {len(thresholds)}"
        enable_early_exit = cfg.match.get("enable_early_exit", True)
        azi_n = cfg.patch.azi_n
        desc_t, pose_t, opt_t = timers if timers is not None else (_Timer(False), _Timer(False), _Timer(False))

        assert counts is None or not debug
        npts = None if counts is None else [counts[0:1], counts[1:2]] * S      # per descriptor job: (src, tgt) per scale

        desc_t.tic()
        # ---- key-points: one FPS per cloud, both clouds in one launch --------------------------------
        if xyz is None:
            xyz = torch.cat([src, tgt], dim=0)
        nfps = max(Kr, K)
        if max(Ns, Nt) <= ops.FPS_MAX_POINTS:
            fidx, fk = ops.fps(xyz, [0, Ns, Ns + Nt], nfps, d_counts=counts)
        else:   # beyond one cluster's registers: that cloud on the grid-wide kernel (a capacity above it holds such a cloud)
            per = [ops.fps_large(c, nfps, d_count=None if counts is None else counts[j:j + 1]) if c.shape[0] > ops.FPS_MAX_POINTS
                   else ops.fps(c, [0, c.shape[0]], nfps, d_counts=None if counts is None else counts[j:j + 1])
                   for j, c in enumerate((src, tgt))]
            fidx = torch.stack([i.reshape(nfps) for i, _ in per])
            fk = torch.stack([k.reshape(nfps, 3) for _, k in per])
        kpts1, kpts2 = fk[0, :Kr].contiguous(), fk[1, :Kr].contiguous()
        src_kpts, tgt_kpts = fk[0, :K].contiguous(), fk[1, :K].contiguous()
        # ---- density-aware radii of every scale: one histogram, or one per scale for a cloud above 200000 points ------
        rng_after_first = None      # torch's CPU generator after scale 0's draw: where the reference leaves it on an exit
        if counts is not None:      # the device picks the larger cloud from the counts (and sub-samples it through ``sub``)
            r_dev, m_dev, _ = ops.radius_estimate_pair(kpts1, src, kpts2, tgt, thresholds, counts, d_sub=sub)
        else:
            pts_r, kpts_r = (src, kpts1) if Ns > Nt else (tgt, kpts2)
            N = pts_r.shape[0]
            if N > ops.RADIUS_SUBSAMPLE:
                # reference BUFFERX.py:320-329 + 664-665: each scale estimates its radius on its own 200000-index draw,
                # the denominator keeping N.  Eager: the reference's draws from the CPU generator in scale order (the same
                # indices under torch.manual_seed); under CUDA-graph capture a host draw would be frozen into the graph, so
                # the capture draws on the device (DESIGN.md section 2)
                on_dev = {"device": dev} if torch.cuda.is_current_stream_capturing() else {}
                subs = []
                for i in range(S):
                    subs.append(torch.randint(0, N, (ops.RADIUS_SUBSAMPLE,), **on_dev).to(dev, non_blocking=True))
                    if i == 0 and not on_dev:
                        rng_after_first = torch.get_rng_state()
                est = [ops.radius_estimate(kpts_r, pts_r[subs[i]].contiguous(), thresholds[i:i + 1], denom=N * Kr) for i in range(S)]
                r_dev, m_dev = torch.cat([e[0] for e in est]), torch.cat([e[1] for e in est])
            else:
                r_dev, m_dev, _ = ops.radius_estimate(kpts_r, pts_r, thresholds, denom=N * Kr)
        desc_t.toc()

        maxMc = S * K
        R_acc = torch.empty((maxMc, 3, 3), dtype=torch.float32, device=dev)
        t_acc = torch.empty((maxMc, 3), dtype=torch.float32, device=dev)
        ss_acc = torch.empty((maxMc, 3), dtype=torch.float32, device=dev)
        tt_acc = torch.empty((maxMc, 3), dtype=torch.float32, device=dev)
        offs = torch.zeros(S + 1, dtype=torch.int32, device=dev)
        dbg = dict(scales=[]) if debug else None
        if enable_early_exit and device_exit and not debug:
            tail = self._enqueue_device_exit(src, tgt, aligned, perms, ransac_seed, src_kpts, tgt_kpts, r_dev, R_acc, t_acc, ss_acc, tt_acc, offs,
                                             npts)
            return tail, None

        scales_used = 0
        should_exit = False
        res_block = None
        inl = dI = None
        # Without early exit every scale runs anyway: describe all 2*S (cloud, scale) key-point sets in one batched
        # pass (one SPT / conv-stack / pooling launch sequence instead of 2*S).  The host permutation draws keep the
        # reference's order (src then tgt, scale by scale).
        batched = None
        if not enable_early_exit and not debug:
            desc_t.tic()
            jobs = []
            for i in range(S):
                for pts_c, k_c, j in ((src, src_kpts, 0), (tgt, tgt_kpts, 1)):
                    pm = None if perms is None else perms[i][j]
                    if pm is None:
                        pm = np.random.choice(pts_c.shape[0], pts_c.shape[0], replace=False)
                    if not isinstance(pm, torch.Tensor):
                        pm = torch.from_numpy(np.ascontiguousarray(pm, dtype=np.int32))
                    if not pm.is_cuda or pm.dtype != torch.int32:
                        pm = pm.to(dev, dtype=torch.int32, non_blocking=True)
                    jobs.append((pts_c, k_c, r_dev[i:i + 1], pm))
            batched = self.Desc.forward_multi(jobs, aligned, radii=r_dev, npts=npts)
            desc_t.toc()
        if batched is not None and S <= 8:
            # all scales at once: per-scale mutual matching into rows of one [S,K] buffer, one concatenation kernel
            # (device-side prefix sums = the `offs` of the sequential flow), then CostNet, the hypothesis build and the
            # consensus over the concatenated list -- the order of the reference's per-scale torch.cat.
            pose_t.tic()
            multi = self.Desc.last_multi
            s_lists = torch.empty((S, K), dtype=torch.int32, device=dev)
            t_lists = torch.empty((S, K), dtype=torch.int32, device=dev)
            cnts = torch.zeros(S, dtype=torch.int32, device=dev)
            for i in range(S):
                ops.mutual_nn(batched[2 * i]["desc"], batched[2 * i + 1]["desc"], out=(s_lists[i], t_lists[i], cnts[i:i + 1]))
            s_all, t_all = ops.concat_matches(s_lists, t_lists, cnts, [2 * i * K for i in range(S)],
                                              [(2 * i + 1) * K for i in range(S)], offs)
            d_Mall = offs[S:S + 1]
            logits = self.Pose.logits(multi["equi"], multi["equi"], s_all, t_all, d_Mall, S * K)
            kp_all = torch.cat([src_kpts, tgt_kpts] * S, dim=0)
            zero_off = torch.zeros(2, dtype=torch.int32, device=dev)
            ops.hypotheses(logits, azi_n, kp_all, kp_all, multi["R"], multi["R"], s_all, t_all, d_Mall, S * K,
                           zero_off[0:1], zero_off[1:2], None, R_acc, t_acc, ss_acc, tt_acc)
            scales_used = S
            inl, dI, dbest, counts = ops.consensus(ss_acc, tt_acc, R_acc, t_acc, d_Mall, S * K, azi_n, cfg.match.inlier_th)
            pose_t.toc()
        for i in range(S if (batched is None or S > 8) else 0):
            desc_t.tic()
            des_r = r_dev[i:i + 1]
            ps = None if perms is None else perms[i][0]
            pt = None if perms is None else perms[i][1]
            if batched is not None:         # only with more than 8 scales (the batched tail above handles S <= 8)
                sd, td = batched[2 * i], batched[2 * i + 1]
            else:
                sd = self.Desc(src[None], src_kpts[None], des_r, aligned, perm=ps, debug=debug)
                td = self.Desc(tgt[None], tgt_kpts[None], des_r, aligned, perm=pt, debug=debug)
            s_mids, t_mids, dM, snn, tnn = ops.mutual_nn(sd["desc"], td["desc"], want_nn=debug)
            desc_t.toc()

            pose_t.tic()
            logits = self.Pose.logits(sd["equi"], td["equi"], s_mids, t_mids, dM, K)
            ind = torch.empty(K, dtype=torch.float32, device=dev) if debug else None
            ops.hypotheses(logits, azi_n, src_kpts, tgt_kpts, sd["R"], td["R"], s_mids, t_mids, dM, K,
                           offs[i:i + 1], offs[i + 1:i + 2], ind, R_acc, t_acc, ss_acc, tt_acc)
            scales_used = i + 1
            need_consensus = (i == S - 1) or (enable_early_exit and i == 0) or debug
            if need_consensus:
                inl, dI, dbest, counts = ops.consensus(ss_acc, tt_acc, R_acc, t_acc, offs[i + 1:i + 2], (i + 1) * K, azi_n,
                                                       cfg.match.inlier_th)
            pose_t.toc()
            if debug:
                dbg["scales"].append(dict(s=sd, t=td, s_mids=s_mids, t_mids=t_mids, dM=dM, snn=snn, tnn=tnn, logits=logits,
                                          ind=ind, inlier_ind=inl.clone(), dI=dI.clone(), best=dbest.clone()))
            if enable_early_exit and i == 0:
                opt_t.tic()
                res_block = self.pose_estimator.enqueue(ss_acc, tt_acc, inl, dI, (i + 1) * K, ransac_seed)
                _, num_inliers, _, _ = ops.decode_ransac_result(res_block.cpu())   # one host read
                opt_t.toc()
                should_exit = self.pose_estimator.compute_confidence_score(num_inliers)
                if should_exit:
                    if rng_after_first is not None:     # the reference made only scale 0's sub-sample draw
                        torch.set_rng_state(rng_after_first)
                    break

        opt_t.tic()
        if (not enable_early_exit) or (enable_early_exit and not should_exit):
            res_block = self.pose_estimator.enqueue(ss_acc, tt_acc, inl, dI, scales_used * K, ransac_seed)
        d_Mc = offs[scales_used:scales_used + 1]
        if cfg.test.pose_refine is True:
            refined, _ = ops.refine(ss_acc, tt_acc, d_Mc, scales_used * K, res_block[:16], cfg.match.dist_th)
            refined = refined.double()
        else:
            refined = torch.zeros(16, dtype=torch.float64, device=dev)
        # ---- one small block holds everything the caller needs ---------------------------------------
        su = torch.full((1,), float(scales_used), dtype=torch.float64, device=dev)
        # last element: the sticky fp16-range flag of the shifted-descriptor conv kernel (0 unless an activation overflowed)
        tail = torch.cat([res_block, offs.double(), dI.double(), su, refined, self.Desc.conv_net.overflow_flag(dev).double()])
        if debug:
            dbg.update(fps_idx=fidx, kpts=fk, des_r=r_dev, des_m=m_dev, ss=ss_acc, tt=tt_acc, R=R_acc, t=t_acc)
        return tail, dbg

    def _enqueue_device_exit(self, src, tgt, aligned, perms, ransac_seed, src_kpts, tgt_kpts, r_dev, R_acc, t_acc, ss_acc, tt_acc, offs,
                             npts=None):
        """Early exit decided on the device (forward_async / graphs): scale 0 on the batched route up to its RANSAC,
        bx_early_exit_gate turns the result into the key-point counts of scales 1..S-1 (K to continue, 0 to exit), and those
        scales' descriptors, matches, CostNet rows and hypotheses are sized by the counts and appended behind scale 0's.  On
        exit offs[S] == offs[1], so the final consensus and RANSAC see exactly scale 0's inputs with the same seed and
        reproduce its result; they are kept rather than skipped so that one captured graph serves both outcomes."""
        cfg = self.config
        dev = src.device
        K, S, azi_n = cfg.patch.num_fps, cfg.patch.num_scales, cfg.patch.azi_n
        G = S - 1
        jobs = []
        for i in range(S):
            for pts_c, k_c, j in ((src, src_kpts, 0), (tgt, tgt_kpts, 1)):
                pm = None if perms is None else perms[i][j]
                if pm is None:
                    pm = np.random.choice(pts_c.shape[0], pts_c.shape[0], replace=False)
                if not isinstance(pm, torch.Tensor):
                    pm = torch.from_numpy(np.ascontiguousarray(pm, dtype=np.int32))
                if not pm.is_cuda or pm.dtype != torch.int32:
                    pm = pm.to(dev, dtype=torch.int32, non_blocking=True)
                jobs.append((pts_c, k_c, r_dev[i:i + 1], pm))
        s_lists = torch.empty((S, K), dtype=torch.int32, device=dev)
        t_lists = torch.empty((S, K), dtype=torch.int32, device=dev)
        cnts = torch.zeros(S, dtype=torch.int32, device=dev)
        # ---- scale 0: descriptors, matches, CostNet, hypotheses, consensus, RANSAC -------------------------------------
        d0 = self.Desc.forward_multi(jobs[:2], aligned, radii=r_dev[0:1], npts=None if npts is None else npts[:2])
        m0 = self.Desc.last_multi
        ops.mutual_nn(d0[0]["desc"], d0[1]["desc"], out=(s_lists[0], t_lists[0], cnts[0:1]))
        s0, t0 = ops.concat_matches(s_lists[:1], t_lists[:1], cnts[:1], [0], [K], offs[0:2])
        logits = self.Pose.logits(m0["equi"], m0["equi"], s0, t0, cnts[0:1], K)
        kp0 = torch.cat([src_kpts, tgt_kpts], dim=0)
        ops.hypotheses(logits, azi_n, kp0, kp0, m0["R"], m0["R"], s0, t0, cnts[0:1], K, offs[0:1], offs[1:2], None,
                       R_acc, t_acc, ss_acc, tt_acc)
        inl, dI, _, _ = ops.consensus(ss_acc, tt_acc, R_acc, t_acc, offs[1:2], K, azi_n, cfg.match.inlier_th)
        res0 = self.pose_estimator.enqueue(ss_acc, tt_acc, inl, dI, K, ransac_seed)
        # ---- the decision: counts [key-points per job, patches per radius group (G), patches of the batch] -----------
        counts = torch.empty(2 + G, dtype=torch.int32, device=dev)
        su = torch.empty(1, dtype=torch.float64, device=dev)
        ops.early_exit_gate(res0, cfg.match.get("early_exit_min_inliers", 15), [K] + [2 * K] * G + [2 * G * K], counts, S, su)
        if G > 0:
            # ---- scales 1..S-1, sized by the counts (nothing is computed on exit) ---------------------------------
            d1 = self.Desc.forward_multi(jobs[2:], aligned, radii=r_dev[1:],
                                         counts=dict(job=counts[0:1], group=counts[1:1 + G], total=counts[1 + G:2 + G]),
                                         npts=None if npts is None else npts[2:])
            m1 = self.Desc.last_multi
            for i in range(1, S):
                ops.mutual_nn(d1[2 * i - 2]["desc"], d1[2 * i - 1]["desc"], out=(s_lists[i], t_lists[i], cnts[i:i + 1]),
                              d_Ka=counts[0:1], d_Kb=counts[0:1])
            offs_new = torch.empty(S, dtype=torch.int32, device=dev)
            s1, t1 = ops.concat_matches(s_lists[1:], t_lists[1:], cnts[1:], [2 * j * K for j in range(G)],
                                        [(2 * j + 1) * K for j in range(G)], offs_new)
            torch.add(offs_new[1:], offs[1:2], out=offs[2:])          # offs[1 + i] = scale-0 matches + the new prefix sums
            logits = self.Pose.logits(m1["equi"], m1["equi"], s1, t1, offs_new[G:G + 1], G * K)
            kp1 = torch.cat([src_kpts, tgt_kpts] * G, dim=0)
            ops.hypotheses(logits, azi_n, kp1, kp1, m1["R"], m1["R"], s1, t1, offs_new[G:G + 1], G * K, offs[1:2], offs[S:S + 1], None,
                           R_acc, t_acc, ss_acc, tt_acc)
        # ---- consensus over all appended rows, final RANSAC and refinement ------------------------------------------
        d_Mc = offs[S:S + 1]
        inl, dI, _, _ = ops.consensus(ss_acc, tt_acc, R_acc, t_acc, d_Mc, S * K, azi_n, cfg.match.inlier_th)
        res_block = self.pose_estimator.enqueue(ss_acc, tt_acc, inl, dI, S * K, ransac_seed)
        if cfg.test.pose_refine is True:
            refined, _ = ops.refine(ss_acc, tt_acc, d_Mc, S * K, res_block[:16], cfg.match.dist_th)
            refined = refined.double()
        else:
            refined = torch.zeros(16, dtype=torch.float64, device=dev)
        return torch.cat([res_block, offs.double(), dI.double(), su, refined, self.Desc.conv_net.overflow_flag(dev).double()])

    def _decode(self, tail, times):
        cfg = self.config
        S = cfg.patch.num_scales
        init_pose, num_inliers, best_itr, iters = ops.decode_ransac_result(tail[:18])
        offs_h = tail[18:18 + S + 1].numpy().astype(np.int64)
        num_inlier_ind = int(tail[18 + S + 1].item())
        scales_used = int(tail[18 + S + 2].item())
        num_mutual_inliers = int(offs_h[scales_used])
        self._overflow = bool(tail[-1].item() != 0)
        if cfg.test.pose_refine is True:
            pose = tail[18 + S + 3:18 + S + 3 + 16].numpy().astype(np.float32).reshape(4, 4)
        else:
            pose = init_pose
        self._last_ransac = dict(init_pose=init_pose, best_itr=best_itr, iters=iters, offs=offs_h)
        return pose, times, num_inliers, num_mutual_inliers, num_inlier_ind, scales_used

    def _rerun_tf32(self, data_source, perms, ransac_seed, debug=False):
        """The shifted-descriptor kernel splits values into two fp16 operands; an activation >= 65000 (never seen with
        BatchNorm-ed stacks, but possible in principle) raises its sticky flag.  From then on the descriptor stack of this
        model runs on the TF32 kernel (bx_conv_tc.cu): drop the captured graphs, clear the flag, recompute this pair."""
        net = self.Desc.conv_net
        if not net.force_tf32:
            print("bufferx_b200: activation outside fp16 range -- convolution stacks switched to the TF32 tensor-core kernel")
        net.force_tf32 = True
        self.Pose.conv.force_tf32 = True
        self._drop_captured_state()
        net.overflow_flag(next(self.parameters()).device).zero_()
        return self.forward(data_source, perms=perms, ransac_seed=ransac_seed, debug=debug)

    # ------------------------------------------------------------------------------------------------
    def _draw_des_r(self):
        """Descriptor radius of the training branch (reference BUFFERX.py:175-198), drawn from NumPy's global RNG."""
        cfg = self.config
        name, center = cfg.data.dataset, cfg.patch.des_r
        if name == "3DMatch":
            lo, hi = center * 0.5, center * 1.5
            return np.round(np.clip(np.random.normal(center, (hi - lo) / 6, 1), lo, hi), 2)[0]
        if name == "KITTI":
            values = {3.0: [2.0, 2.5, 3.0, 3.5, 4.0], 0.3: [0.2, 0.25, 0.3, 0.35, 0.4]}.get(center)
            if values is None:
                raise ValueError(f"KITTI training radii are defined for des_r 3.0 and 0.3, not {center}")
            return np.random.choice(values, p=[0.2, 0.2, 0.2, 0.2, 0.2])
        return center

    def _train_forward(self, data_source, perms=None, aug_angles=None, match_choice=None):
        """Validation forward of cfg.stage "Desc" / "Pose" in eval mode (reference BUFFERX.py:148-255), or with the model in
        training mode the forward of the stage's training step (every BatchNorm on batch statistics, its running
        statistics updated: the descriptor network's twice, source then target; "Pose": ``pred_ind`` carries a grad_fn into
        ``Pose.conv``'s weights and biases, "Desc": ``src_des``, ``tgt_des`` and ``equi_score`` into the descriptor
        network's parameters; the batch statistics land in ``self.last_train_stats``): ground-truth
        correspondences on the second-level clouds, descriptors of the (sub-sampled) matched key-points, then EquiMatch
        score + integer SO(2) label ("Desc") or CostNet soft arg-max + float SO(2) label of the augmented target ("Pose").
        NumPy's global RNG is consumed like the reference: match sub-sampling (only beyond cfg.train.pos_num), des_r,
        source permutation, target permutation, augmentation angles.  ``perms`` = (src, tgt) permutations, ``aug_angles``
        [K] and ``match_choice`` (rows of the match list) replace the respective draws.  Device->host reads: the number of
        ground-truth matches (it sizes the draw), and at the end the fp16-range flag of the convolution kernels."""
        cfg = self.config
        stage = cfg.stage
        dev = next(self.parameters()).device
        azi_n = cfg.patch.azi_n

        def _pts(x, shape=(-1, 3)):
            return torch.as_tensor(x).to(dev, dtype=torch.float32, non_blocking=True).reshape(*shape).contiguous()

        train = self.training
        rng_state = np.random.get_state()     # replayed if the pair has to be recomputed on the TF32 kernels
        if train:
            # the step moves every running statistic and optimizer.step() the weights: captured graphs hold the old folded ones
            self._drop_captured_state()
            stats = dict(src=[], tgt=[], pose=[]) if stage == "Pose" else dict(src=[], tgt=[])
        with torch.cuda.device(dev):
            src, tgt = _pts(data_source["src_fds_pcd"]), _pts(data_source["tgt_fds_pcd"])
            src_sds, tgt_sds = _pts(data_source["src_sds_pcd"]), _pts(data_source["tgt_sds_pcd"])
            T = _pts(data_source["relt_pose"], (4, 4))
            vs = data_source["voxel_sizes"]
            voxel = float(vs.reshape(-1)[0].item() if isinstance(vs, torch.Tensor) else np.asarray(vs, dtype=np.float32).reshape(-1)[0])
            pairs, d_cnt = ops.gt_matches(src_sds, tgt_sds, T, voxel)
            n_match = int(d_cnt.item())
            match = pairs[:n_match]
            if match_choice is not None:
                match = match[torch.as_tensor(np.asarray(match_choice), dtype=torch.long).to(dev)]
            elif n_match > cfg.train.pos_num:
                rand_ind = np.random.choice(range(n_match), cfg.train.pos_num, replace=False)
                match = match[torch.from_numpy(rand_ind).to(dev)]
            if match.shape[0] == 0:
                print(f"{data_source.get('src_id')} {data_source.get('tgt_id')} has no keypts")
                return None
            match = match.long()
            src_kpt, tgt_kpt = src_sds[match[:, 0]].contiguous(), tgt_sds[match[:, 1]].contiguous()
            des_r = self._draw_des_r()
            aligned = bool(data_source["is_aligned_to_global_z"])
            ps, pt = (None, None) if perms is None else perms
            if train and stage == "Desc":
                src_d = self.Desc.forward_desc_train(src[None], src_kpt[None], des_r, aligned, perm=ps, stats=stats["src"])
                tgt_d = self.Desc.forward_desc_train(tgt[None], tgt_kpt[None], des_r, aligned, perm=pt, stats=stats["tgt"])
            elif train:
                src_d = self.Desc.forward_train(src[None], src_kpt[None], des_r, aligned, perm=ps, stats=stats["src"])
                tgt_d = self.Desc.forward_train(tgt[None], tgt_kpt[None], des_r, aligned, True, perm=pt, aug_angles=aug_angles,
                                                stats=stats["tgt"])
            else:
                src_d = self.Desc(src[None], src_kpt[None], des_r, aligned, perm=ps)
                tgt_d = self.Desc(tgt[None], tgt_kpt[None], des_r, aligned, None, stage == "Pose", perm=pt, aug_angles=aug_angles)
            K = src_kpt.shape[0]
            if K < 2:
                print(f"{data_source.get('src_id')} {data_source.get('tgt_id')} don't have enough patches")
                return None
            if stage == "Desc":
                out = {"src_kpt": src_kpt, "tgt_kpt": tgt_kpt, "src_des": src_d["desc"], "tgt_des": tgt_d["desc"],
                       "equi_score": _EquiMatchFn.apply(src_d["equi"], tgt_d["equi"]) if train
                       else ops.equi_match(src_d["equi"], tgt_d["equi"]),
                       "gt_label": ops.so2_gt(src_d["rand_axis"], src_d["R"], tgt_d["R"], T, azi_n, True)}
                if train:
                    self.last_train_stats = stats
            elif train:
                out = {"pred_ind": self.Pose.conv.forward_train(src_d["equi"], tgt_d["equi"], stats["pose"]),
                       "gt_ind": ops.so2_gt(src_d["rand_axis"], src_d["R"], tgt_d["R"], T, azi_n, False, aug_R=tgt_d["aug_rotation"])}
                self.last_train_stats = stats
            else:
                # patch i of the source against patch i of the target: identity match lists through CostNet, the soft
                # arg-max from the hypothesis kernel (its pose outputs land in scratch buffers)
                ids = torch.arange(K, dtype=torch.int32, device=dev)
                d_K = torch.full((1,), K, dtype=torch.int32, device=dev)
                logits = self.Pose.logits(src_d["equi"], tgt_d["equi"], ids, ids, d_K, K)
                pred = torch.empty(K, dtype=torch.float32, device=dev)
                offs = torch.zeros(2, dtype=torch.int32, device=dev)
                scratch = [torch.empty((K, 3, 3), dtype=torch.float32, device=dev)] + \
                          [torch.empty((K, 3), dtype=torch.float32, device=dev) for _ in range(3)]
                ops.hypotheses(logits, azi_n, src_kpt, tgt_kpt, src_d["R"], tgt_d["R"], ids, ids, d_K, K, offs[0:1], offs[1:2], pred,
                               *scratch)
                out = {"pred_ind": pred,
                       "gt_ind": ops.so2_gt(src_d["rand_axis"], src_d["R"], tgt_d["R"], T, azi_n, False, aug_R=tgt_d["aug_rotation"])}
            # the training step runs every convolution on the TF32 kernel, which has no fp16-range limit: nothing to recompute
            overflow = not train and self.Desc.conv_net.overflow_flag(dev).item() != 0
        if overflow:      # an activation left fp16 range: recompute the pair with the TF32 kernels and the same draws
            np.random.set_state(rng_state)
            net = self.Desc.conv_net
            net.force_tf32 = True
            self.Pose.conv.force_tf32 = True
            self._drop_captured_state()
            net.overflow_flag(dev).zero_()
            return self._train_forward(data_source, perms, aug_angles, match_choice)
        return out

    def forward(self, data_source, perms=None, ransac_seed=None, debug=False, aug_angles=None, match_choice=None):
        cfg = self.config
        if cfg.stage != "test":
            if cfg.stage not in ("Desc", "Pose"):
                raise NotImplementedError(
                    "bufferx_b200 runs cfg.stage 'test', and for the training stages 'Desc' / 'Pose' their validation forward "
                    "(eval mode) and their training step (train mode)")
            if self.training and cfg.stage == "Desc" and any(p.requires_grad for p in self.Pose.parameters()):
                raise NotImplementedError(
                    "the Desc training step (training-mode BatchNorm and the backward pass through Desc) needs CostNet frozen "
                    "(requires_grad=False on every Pose parameter, as train.py does for this stage)")
            if self.training and cfg.stage == "Pose" and any(p.requires_grad for p in self.Desc.parameters()):
                raise NotImplementedError(
                    "the Pose training step needs the descriptor network frozen (requires_grad=False on every Desc parameter, "
                    "as train.py does for this stage): the backward pass through Desc is not built")
            if next(self.parameters()).device.type != "cuda":
                raise ops.BufferXError("BufferX.forward needs the model on a CUDA device: there is no CPU path")
            return self._train_forward(data_source, perms, aug_angles, match_choice)
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise ops.BufferXError("BufferX.forward needs the model on a CUDA device: there is no CPU path")
        sizes = self._cloud_sizes(data_source)
        if self._use_graphs and not debug and ransac_seed is None and self._graphable():
            return self.forward_async(data_source, perms).result()

        def _cloud(x):
            x = torch.as_tensor(x)
            return x.to(dev, dtype=torch.float32, non_blocking=True).reshape(-1, 3).contiguous()

        aligned = bool(data_source["is_aligned_to_global_z"])
        enable_timing = cfg.test.get("enable_timing", False)
        rng_state = np.random.get_state() if perms is None else None     # replayed if the pair has to be recomputed
        # ... and torch's CPU generator, when the pair draws its radius sub-samples from it
        torch_rng = torch.get_rng_state() if max(sizes) > ops.RADIUS_SUBSAMPLE else None
        with torch.cuda.device(dev):        # kernels launch on the model's device, whatever the caller's current device
            src, tgt = _cloud(data_source["src_fds_pcd"]), _cloud(data_source["tgt_fds_pcd"])
            timers = (_Timer(enable_timing), _Timer(enable_timing), _Timer(enable_timing))
            tail, dbg = self._enqueue(src, tgt, aligned, perms, ransac_seed, debug, timers)
        tail_h = tail.cpu()                 # the one device->host read of the pair
        timers[2].toc()                     # pairs with the tic before RANSAC / refinement in _enqueue (pose_optim time)
        out = self._decode(tail_h, [timers[0].total, timers[1].total, timers[2].total])
        if self._overflow:
            if rng_state is not None:
                np.random.set_state(rng_state)
            if torch_rng is not None:
                torch.set_rng_state(torch_rng)
            return self._rerun_tf32(data_source, perms, ransac_seed, debug)
        if debug:
            dbg.update(self._last_ransac)
            self.last_debug = dbg
        return out
