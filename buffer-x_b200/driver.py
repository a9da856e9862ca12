"""Pair sharding across GPUs: one process per GPU, pairs round-robin, ONE all-gather of records.

Evaluation (``evaluate_sharded``) and training (``train_sharded``, DESIGN.md §8) both run one process per GPU.

The reference is single-process / single-GPU (``nn.DataParallel(model, [gpu])``,
/root/reference/test.py:105) and processes pairs in a serial loop with no cross-pair state
(test.py:132-146), so the path shards embarrassingly: pair i -> rank i mod world.  The only collective
is the final gather of a fixed 32-float record per pair (4x4 pose, 3 timings, 4 counters, rte, rre,
success, pair id + padding).  Works with ``nccl`` (GPU tensors) and ``gloo`` (CPU tests).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

from . import ops

RECORD = 32  # floats per pair


def shard_indices(n_pairs: int, rank: int, world: int):
    """Round-robin assignment (BASELINE.json config 4): pair i -> rank i mod world."""
    return list(range(rank, n_pairs, world))


def pack_record(pair_id, pose, times, num_inliers, num_mutual, num_inlier_ind, scales_used, rte=np.nan, rre=np.nan, success=0.0):
    r = np.zeros(RECORD, dtype=np.float32)
    r[:16] = np.asarray(pose, dtype=np.float64).reshape(16)
    r[16:19] = np.asarray(times, dtype=np.float64)[:3]
    r[19:23] = [num_inliers, num_mutual, num_inlier_ind, scales_used]
    r[23], r[24], r[25], r[26] = rte, rre, success, pair_id
    return r


def unpack_record(r):
    r = np.asarray(r)
    return dict(pair_id=int(round(float(r[26]))), pose=r[:16].reshape(4, 4).astype(np.float64), times=r[16:19].tolist(),
                num_inliers=int(r[19]), num_mutual=int(r[20]), num_inlier_ind=int(r[21]), scales_used=int(r[22]),
                rte=float(r[23]), rre=float(r[24]), success=bool(r[25] > 0.5))


def gather_records(local: np.ndarray, n_pairs: int, device=None):
    """local: [n_local, RECORD] records of this rank -> [n_pairs, RECORD] on every rank, ordered by pair id.
    Uses a single all_gather of equally padded blocks (ranks may own ceil or floor(n_pairs/world) pairs)."""
    local = np.asarray(local, dtype=np.float32).reshape(-1, RECORD)
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        out = local
    else:
        world = dist.get_world_size()
        per = (n_pairs + world - 1) // world
        blk = torch.full((per, RECORD), float("nan"), dtype=torch.float32)
        blk[: local.shape[0]] = torch.from_numpy(local)
        if device is not None:
            blk = blk.to(device)
        bufs = [torch.empty_like(blk) for _ in range(world)]
        dist.all_gather(bufs, blk)
        out = torch.cat(bufs).cpu().numpy()
        out = out[~np.isnan(out[:, 26])]
    order = np.argsort(out[:, 26], kind="stable")
    return out[order]


def evaluate_sharded(forward_fn, pairs, cfg, out_dir=None, experiment_id="bufferx_b200", timestr="run", dataset="synthetic", device=None,
                     write_logs=False):
    """The reference's test loop (test.py:132-338) over a LIST of pairs, sharded round-robin over the ranks of the default
    process group: rank r calls ``forward_fn(data_source)`` (``BufferX.forward`` signature and return tuple) for the pairs
    r, r + world, ..., evaluates each against ``data_source["relt_pose"]`` (test.py:168-172), packs one record per pair, ONE
    all-gather collects them, and rank 0 writes the reference's artefacts from the gathered records: the per-sample CSV
    (utils/result_io.py:7-49), the summary CSV (:80-124) and -- ``write_logs`` -- the 3DMatch ``.log`` entries
    (test.py:151-166).  Returns (summary dict, states [n_pairs, 12]) on every rank."""
    import os
    import time
    from . import evaluation as E
    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    rte_th, rre_th = cfg.test.rte_thresh, cfg.test.rre_thresh
    recs = []
    for i in shard_indices(len(pairs), rank, world):
        d = pairs[i]
        t0 = time.perf_counter()
        pose, times, ninl, nmut, nind, su = forward_fn(d)
        wall = time.perf_counter() - t0
        gt = np.asarray(d["relt_pose"].cpu() if isinstance(d["relt_pose"], torch.Tensor) else d["relt_pose"])
        st = E.pair_state(pose, gt, ninl, nmut, nind, su, times if any(times) else [wall, 0.0, 0.0], rte_th, rre_th)
        recs.append(pack_record(i, pose if pose is not None else np.eye(4), st[9:12], ninl, nmut, nind, su, rte=st[1], rre=st[2], success=float(st[0])))
    local = np.stack(recs) if recs else np.zeros((0, RECORD), np.float32)
    allrec = gather_records(local, len(pairs), device=device)
    states = E.states_from_records(allrec)
    summary = E.summarize_states(states, dataset)
    if rank == 0 and out_dir is not None:
        exp = experiment_id.rsplit("/", 1)[-1]
        pose_method = str(cfg.match.pose_estimator).upper()
        early = "ON" if cfg.match.get("enable_early_exit", True) else "OFF"
        E.save_per_sample_results(states, os.path.join(out_dir, "per_sample_results", exp,
                                                       f"{exp}_{dataset}_{cfg.patch.num_points_per_patch}_{cfg.patch.num_scales}_{cfg.patch.num_fps}_{timestr}.csv"),
                                  pose_method, early)
        E.save_full_results_csv([summary], experiment_id, timestr, cfg.patch.num_points_per_patch, cfg.patch.num_scales, cfg.patch.num_fps,
                                full_results_dir=os.path.join(out_dir, "full_results"))
        if write_logs:
            for r in allrec:
                u = unpack_record(r)
                d = pairs[u["pair_id"]]
                scene = str(d.get("scene_name", "scene"))
                E.append_trajectory_entry(os.path.join(out_dir, "logs", scene, f"{timestr}.log"), str(d.get("src_id", u["pair_id"])).split("_")[-1],
                                          str(d.get("tgt_id", u["pair_id"])).split("_")[-1], u["pose"])
    return summary, states


# --------------------------------------------------------------------------- #
# Sharded training (DESIGN.md §8): one pair per rank per step, ONE all-gather of a fixed-size record per step, and the
# rank-order float64 mean of the contributors' gradients and BatchNorm buffers (ops.dp_mean) on every rank.
METERS = ("desc_loss", "desc_acc", "eqv_loss", "eqv_acc", "match_loss")      # the trainer's meter list (trainer.py:33)
BEST_KEY = {"Desc": "desc_loss", "Pose": "match_loss"}                         # the best-snapshot criterion (trainer.py:70-77)
_NBT_EXACT = 1 << 24      # num_batches_tracked travels in the fp32 record: exact below 2^24


def _world(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


def _gather_rows(t, group=None):
    """t [k] on the model's device -> [W, k] on the same device, row r = rank r's t: ONE all_gather.  NCCL gathers
    device tensors; gloo gathers host copies (PyTorch documents gloo's all_gather for host tensors only)."""
    world, _ = _world(group)
    if world == 1:
        return t[None]
    src = t if dist.get_backend(group) == "nccl" else t.cpu()
    out = torch.empty((world, t.numel()), dtype=t.dtype, device=src.device)
    dist.all_gather(list(out.unbind(0)), src, group=group)
    return out.to(t.device)


def _bn_buffers(model):
    """running_mean, running_var and num_batches_tracked of every BatchNorm, in named_buffers() order."""
    ids = {id(b) for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm) for b in m.buffers(recurse=False)}
    return [b for _, b in model.named_buffers() if id(b) in ids]


def epoch_shard(n: int, rank: int, world: int, epoch: int, seed: int, max_iter: int):
    """The pair indices rank ``rank`` trains on in epoch ``epoch``, one per step: positions rank, rank + world, ... of a
    permutation of range(n) drawn from ``seed + epoch`` (the same on every rank; NumPy's global RNG is left alone), for
    min(max_iter, ceil(n / world)) steps.  None marks a step in which this rank has no pair left: it still takes part in
    the step's collective, contributing nothing."""
    perm = np.random.RandomState(seed + epoch).permutation(n)
    steps = min(int(max_iter), -(-n // world))
    return [int(perm[s * world + rank]) if s * world + rank < n else None for s in range(steps)]


def train_step(model, optimizer, data, train_loss, group=None, mean_fn=None):
    """One sharded training step on this rank: ``optimizer.zero_grad()``, ``model(data)`` (skipped when ``data`` is None),
    ``train_loss(out) -> (loss, stats)`` and ``loss.backward()``, then ONE all-gather of the rank's record (the trainable
    parameters' gradients in named_parameters() order, zeros for a None grad or a rank without output; the BatchNorm
    buffers; the contribution flag) and ``mean_fn`` (ops.dp_mean) over the gathered matrix.  A rank whose forward returned
    None (or that had no pair) restores the BatchNorm buffers it held before the forward.  When at least one rank
    contributed, every rank takes the mean as its gradients and BatchNorm buffers and calls ``optimizer.step()`` unless a
    mean gradient is non-finite (trainer.py:145-152, on the averaged gradient, so every rank decides alike); when none
    did, the step changes nothing.  Returns (contributors, stepped, this rank's stats or None)."""
    mean_fn = mean_fn or ops.dp_mean
    params = [p for _, p in model.named_parameters() if p.requires_grad]
    bufs = _bn_buffers(model)
    for t in params + [b for b in bufs if b.is_floating_point()]:
        if t.dtype != torch.float32:
            raise TypeError(f"train_step: parameters and BatchNorm statistics must be float32, got {t.dtype}")
    snap = [b.detach().clone() for b in bufs]
    optimizer.zero_grad()
    out = model(data) if data is not None else None
    stats = None
    if out is not None:
        loss, stats = train_loss(out)
        loss.backward()
    else:
        with torch.no_grad():
            for b, s in zip(bufs, snap):
                b.copy_(s)
    sizes = [p.numel() for p in params] + [b.numel() for b in bufs]
    n_grad, n = sum(sizes[:len(params)]), sum(sizes)
    dev = params[0].device if params else bufs[0].device
    rec = torch.zeros(n + 1, dtype=torch.float32, device=dev)
    with torch.no_grad():
        parts = rec[:n].split(sizes)
        for part, p in zip(parts, params):
            if out is not None and p.grad is not None:
                part.copy_(p.grad.reshape(-1))
        for part, b in zip(parts[len(params):], bufs):
            if not b.is_floating_point() and int(b.max()) >= _NBT_EXACT:
                raise OverflowError("train_step: num_batches_tracked has reached 2^24, beyond the fp32 record's exact range")
            part.copy_(b.reshape(-1))
        rec[n] = 1.0 if out is not None else 0.0
        with ops._Span("dp_exchange"):        # the all-gather, the mean and the write-back (tools/train_sharded_bench.py)
            gathered = _gather_rows(rec, group)
            mean, count = mean_fn(gathered)
            count = int(count.item())
            if count:
                parts = mean.split(sizes)
                for part, p in zip(parts, params):
                    p.grad = part.view_as(p)
                for part, b in zip(parts[len(params):], bufs):
                    b.copy_((part if b.is_floating_point() else part.round()).view_as(b))
        if count == 0:
            return 0, False, stats
        finite = bool(torch.isfinite(mean[:n_grad]).all())
    if finite:
        optimizer.step()
    return count, finite, stats


def _loader(dataset, indices, collate, num_workers):
    from torch.utils.data import DataLoader, Subset
    return DataLoader(Subset(dataset, indices), batch_size=1, shuffle=False, num_workers=num_workers,
                      collate_fn=collate if collate is not None else (lambda b: b[0]))


def validate_sharded(model, val_set, eval_stats, collate=None, group=None, num_workers=0):
    """The trainer's validation pass (trainer.py:171-220) with the pairs split round-robin: each rank runs the eval-mode
    forward under no_grad on its pairs and ``eval_stats(out) -> stats`` on each output, ONE all-gather of fixed-size
    float64 records [pair id, has output, key present x len(METERS), value x len(METERS)] collects them, and every rank
    averages each meter over the pairs in pair order.  Returns (means {key: avg} -- 0 for a key no pair reported, as
    AverageMeter -- and the gathered records ordered by pair id, numpy [n_val, 2 + 2 len(METERS)])."""
    world, rank = _world(group)
    M = len(METERS)
    mine = shard_indices(len(val_set), rank, world)
    rec = torch.full((-(-len(val_set) // world), 2 + 2 * M), float("nan"), dtype=torch.float64)
    was_training = model.training
    model.eval()
    with torch.no_grad():
        for j, d in enumerate(_loader(val_set, mine, collate, num_workers)):
            out = model(d)
            rec[j, :2 + M] = 0.0
            rec[j, 0] = mine[j]
            if out is None:
                continue
            rec[j, 1] = 1.0
            st = eval_stats(out)
            for i, k in enumerate(METERS):
                if st.get(k) is not None:
                    rec[j, 2 + i], rec[j, 2 + M + i] = 1.0, float(st[k])
    model.train(was_training)
    dev = next(model.parameters()).device
    allrec = _gather_rows(rec.reshape(-1).to(dev), group).reshape(-1, 2 + 2 * M).cpu().numpy()
    allrec = allrec[~np.isnan(allrec[:, 0])]
    allrec = allrec[np.argsort(allrec[:, 0], kind="stable")]
    res = {}
    for i, k in enumerate(METERS):
        total, cnt = 0.0, 0
        for r in allrec:
            if r[1] == 1.0 and r[2 + i] == 1.0:
                total += float(r[2 + M + i])
                cnt += 1
        res[k] = total / cnt if cnt else 0
    return res, allrec


def _broadcast_state(model, group=None):
    """Every rank takes rank 0's state_dict."""
    world, _ = _world(group)
    if world == 1:
        return
    src = 0 if group is None else dist.get_global_rank(group, 0)
    nccl = dist.get_backend(group) == "nccl"
    with torch.no_grad():
        for v in model.state_dict().values():
            t = v if nccl else v.cpu()
            dist.broadcast(t, src, group=group)
            if t is not v:
                v.copy_(t)


def train_sharded(model, optimizer, scheduler, train_set, val_set, cfg, train_loss, eval_stats, collate=None, seed=0,
                  snapshot_root=None, num_workers=0, group=None, log=None):
    """``Trainer.train`` (trainer.py:56-220) for stage ``cfg.stage`` over every rank of the process group (or alone, without
    one), with the semantics of DESIGN.md §8: rank 0's state_dict broadcast at start, NumPy's global RNG and torch's CPU
    generator seeded with ``seed + rank``; per epoch ``epoch_shard`` steps of ``train_step`` (one pair per rank, batch of
    one, ``collate`` over a list of one sample; default: the sample itself), rank 0 writes
    ``{snapshot_root}/{stage}/{epoch}.pth``, ``validate_sharded`` on ``val_set``, rank 0 writes ``best.pth`` when the
    stage's validation loss improves, a barrier, and ``scheduler.step()`` every cfg.optim.scheduler_interval[stage]
    epochs.  ``train_loss(out) -> (loss, stats)``, ``eval_stats(out) -> stats`` mirror the trainer's two loss paths.
    Returns the per-epoch validation means."""
    import gc
    import os
    world, rank = _world(group)
    stage = cfg.stage
    net = getattr(model, "module", model)
    _broadcast_state(net, group)
    np.random.seed(seed + rank)
    torch.manual_seed(seed + rank)
    interval = cfg.optim.scheduler_interval[stage]
    best, history = 1000000000, []

    def save(name):
        if rank == 0 and snapshot_root is not None:
            d = os.path.join(snapshot_root, stage)
            os.makedirs(d, exist_ok=True)
            torch.save(net.state_dict(), os.path.join(d, f"{name}.pth"))

    for epoch in range(cfg.train.epoch):
        gc.collect()
        shard = epoch_shard(len(train_set), rank, world, epoch, seed, cfg.train.max_iter)
        pairs = iter(_loader(train_set, [i for i in shard if i is not None], collate, num_workers))
        model.train()
        stepped = 0
        for i in shard:
            _, did, _ = train_step(model, optimizer, next(pairs) if i is not None else None, train_loss, group)
            stepped += did
        save(f"{epoch}")
        res, _ = validate_sharded(model, val_set, eval_stats, collate, group, num_workers)
        if res[BEST_KEY[stage]] < best:
            best = res[BEST_KEY[stage]]
            save("best")
        if world > 1:
            dist.barrier(group)
        if log is not None and rank == 0:
            log(f"Epoch {epoch}: {len(shard)} steps x {world} ranks, {stepped} optimizer steps; evaluation {res}")
        if (epoch + 1) % interval == 0:
            scheduler.step()
        history.append(res)
    return history
