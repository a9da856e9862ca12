"""CPU ORACLE of the Pose stage's training step (``cfg.stage`` "Pose", ``model.train()``), in float64.

TEST INFRASTRUCTURE ONLY.  File:line are relative to the reference checkout:
    training step      trainer.py:93-167 (model.train(), forward, HuberLoss(pred_ind, gt_ind), backward, optimizer.step())
    frozen Desc        train.py:36-48 (requires_grad=False on every module but the stage being trained)
    Desc forward       models/patch_embedder.py:44-90 with every BatchNorm in training mode
    Pose forward       models/BUFFERX.py:39-69 (CostVolume) and models/patchnet.py:192-210 (CostNet)
``model.train()`` switches the frozen descriptor network to batch statistics too: ``requires_grad=False`` does not change
a BatchNorm's mode.  So every BatchNorm below normalises with the biased batch variance and moves its running statistics
(momentum 0.1, unbiased variance in the running update), the descriptor network's twice per step: the source call, then
the target call.  The integer decisions (match list, patches, frames, SPT selection) and the fp32 de-rotated point-layer
inputs are those of oracle/oracle.py and oracle/train_stages.py; everything from the point layer on is float64 torch on
the CPU, and the gradients are float64 autograd.  Pinned against the reference's own modules in training mode by
tests/golden/train_pose_step.npz (tests/tools/gen_train_pose_golden.py).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import oracle as O
from oracle import train_stages as TS

CYL_CONVS = [0, 3, 6, 9, 12, 15, 18, 21]
COST_CONVS = [0, 3, 6, 9, 12, 15, 18, 21, 24, 27]


def state64(sd):
    """float64 copies of a state_dict's floating tensors (integers kept): the running statistics this oracle updates."""
    return {k: (v.detach().double().clone() if v.is_floating_point() else v.detach().clone()) for k, v in sd.items()}


def bn_hparams(model):
    """{state_dict prefix: (momentum, eps)} of every BatchNorm of ``model`` (read from the modules, as torch's BatchNorm
    reads them in training mode)."""
    from torch.nn.modules.batchnorm import _BatchNorm
    return {name: (m.momentum, m.eps) for name, m in model.named_modules() if isinstance(m, _BatchNorm)}


def bn_train(x, st, key, affine, stats, hp):
    """BatchNorm in training mode on x (channel axis 1) with (momentum, eps) = hp[key]: normalise with the batch mean and
    biased variance, update st[key.running_*] in place and num_batches_tracked; (batch mean, batch variance) are appended
    to ``stats``."""
    momentum, eps = hp[key]
    if momentum is None:                      # cumulative moving average, as torch's BatchNorm with momentum=None
        momentum = 1.0 / float(st[key + ".num_batches_tracked"] + 1)
    dims = [d for d in range(x.dim()) if d != 1]
    stats.append((x.detach().mean(dims), x.detach().var(dims, unbiased=False)))
    st[key + ".num_batches_tracked"] = st[key + ".num_batches_tracked"] + 1
    return F.batch_norm(x, st[key + ".running_mean"], st[key + ".running_var"], st[key + ".weight"] if affine else None,
                        st[key + ".bias"] if affine else None, training=True, momentum=momentum, eps=eps)


def pad_cyl(x):
    return O._pad_cyl(x)


def desc_train(inv, st, stats, hp, rad_n=3, ele_n=7, azi_n=20, pfx="Desc."):
    """Point layer + Cylindrical_Net + pool layer of MiniSpinNet in training mode, float64, on the de-rotated samples
    inv [K,V,nv,3] -> (x [K,32,7,20], equi, desc).  ``hp``: bn_hparams of the model."""
    x = torch.as_tensor(np.asarray(inv)).double().permute(0, 3, 1, 2)
    x = F.conv2d(x, st[pfx + "pnt_layer.0.weight"], st[pfx + "pnt_layer.0.bias"])
    x = F.relu(bn_train(x, st, pfx + "pnt_layer.1", True, stats, hp)).amax(dim=3)
    K = x.shape[0]
    x = x.view(K, 16, rad_n, ele_n, azi_n)
    c = pfx + "conv_net.ops."
    x = F.conv3d(pad_cyl(x), st[c + "0.weight"], st[c + "0.bias"])
    x = F.relu(bn_train(x, st, c + "1", False, stats, hp)).squeeze(2)
    for i in CYL_CONVS[1:]:
        x = F.conv2d(pad_cyl(x), st[c + f"{i}.weight"], st[c + f"{i}.bias"])
        if i != 21:
            x = F.relu(bn_train(x, st, c + f"{i + 1}", False, stats, hp))
    w = F.conv2d(x, st[pfx + "pool_layer.0.weight"], st[pfx + "pool_layer.0.bias"])
    w = F.relu(bn_train(w, st, pfx + "pool_layer.1", True, stats, hp))
    w = F.conv2d(w, st[pfx + "pool_layer.3.weight"], st[pfx + "pool_layer.3.bias"])
    w = F.relu(bn_train(w, st, pfx + "pool_layer.4", True, stats, hp))
    f = F.avg_pool2d(x * w, kernel_size=(x.shape[2], x.shape[3])).view(K, -1)
    return x, F.normalize(x, p=2, dim=1), F.normalize(f, p=2, dim=1)


def cost_volume(d1, d2, azi_n=20):
    """CostVolume.forward's volume (BUFFERX.py:52-64): [M,C,n,k,l] = d1[c,k,(l-n) mod azi_n] - d2[c,k,l]."""
    M = d1.shape[0]
    l = torch.arange(azi_n)
    idx = (l[None, :] - l[:, None]) % azi_n
    x = d1[:, :, :, idx.reshape(-1)].reshape(M, d1.shape[1], d1.shape[2], azi_n, azi_n)
    return x.permute(0, 1, 3, 2, 4) - d2.unsqueeze(2)


def costnet_train(d1, d2, params, st, stats, hp, keep=None, azi_n=20, pfx="Pose.conv."):
    """CostNet in training mode, float64: d1, d2 [M,32,5,20] (no gradient), params = {"ops.i.weight"/"ops.i.bias": leaf
    tensors} -> pred_ind [M] differentiable in params.  ``keep`` (a dict): each convolution's input and output (the output
    with retain_grad) under "x{i}" / "z{i}", for the error bounds of the gradients."""
    x = cost_volume(d1.double(), d2.double(), azi_n)
    for i in COST_CONVS:
        if keep is not None:
            keep[f"x{i}"] = x.detach()
        z = F.conv3d(x, params[f"ops.{i}.weight"], params[f"ops.{i}.bias"])
        if keep is not None and z.requires_grad:
            z.retain_grad()
            keep[f"z{i}"] = z
        x = z if i == 27 else F.relu(bn_train(z, st, pfx + f"ops.{i + 1}", False, stats, hp))
    cost = x.reshape(x.shape[0], azi_n)
    if keep is not None:
        keep["logits"] = cost.detach()
    prob = F.softmax(cost, dim=-1)
    return torch.sum(prob * torch.arange(azi_n, dtype=torch.float64)[None], dim=-1)


def pose_params(sd, pfx="Pose.conv."):
    """CostNet's weights and biases as float64 leaf tensors requiring grad, keyed "ops.i.weight" / "ops.i.bias"."""
    return {k[len(pfx):]: sd[k].detach().double().clone().requires_grad_(True) for k in sd
            if k.startswith(pfx) and k.split(".")[-1] in ("weight", "bias") and int(k.split(".")[-2]) in COST_CONVS}


def _describe_train(st, stats, hp, cfg, pts, kpts, des_r, aligned, perm, angles, z_axis=None):
    P = cfg.patch.num_points_per_patch
    rad_n, azi_n, ele_n = cfg.patch.rad_n, cfg.patch.azi_n, cfg.patch.ele_n
    _, patches = O.select_patches(pts, perm, kpts, des_r, P)
    delta, Rt, rand_axis = O.lrf(patches, des_r, aligned, z_axis=z_axis)
    aug_R = None
    if angles is not None:
        delta, rand_axis, aug_R = TS.so2_augment(delta, rand_axis, angles)
    inv, _ = O.spt(delta, rad_n, azi_n, ele_n, cfg.patch.delta / rad_n, cfg.patch.voxel_sample)
    with torch.no_grad():
        _, equi, desc = desc_train(inv, st, stats, hp, rad_n, ele_n, azi_n)
    return dict(equi=equi, desc=desc, R=Rt, rand_axis=rand_axis, aug_rotation=aug_R, inv=inv)


def train_step(sd, hp, cfg, data, rng=None, perms=None, aug_angles=None, match_choice=None, keep=None):
    """The Pose stage's training forward (BufferX.forward under model.train(), BUFFERX.py:148-255), NumPy draws in the
    reference's order (match sub-sampling, des_r, source permutation, target permutation, augmentation angles) from ``rng``
    (default the global RNG) unless given.  ``hp``: bn_hparams of the model.  -> None (no matches / fewer than two patches) or dict(pred_ind (float64,
    differentiable in ``params``), gt_ind (fp32 labels), params, state (the float64 state after the running updates),
    stats (dict src / tgt / pose: (batch mean, batch variance) of every BatchNorm in module order), K)."""
    rng = np.random if rng is None else rng
    src, tgt = TS._f32(data["src_fds_pcd"]), TS._f32(data["tgt_fds_pcd"])
    src_sds, tgt_sds = TS._f32(data["src_sds_pcd"]), TS._f32(data["tgt_sds_pcd"])
    T = TS._f32(data["relt_pose"])
    aligned = bool(data["is_aligned_to_global_z"])
    match = TS.matching_indices(src_sds, tgt_sds, T, np.asarray(data["voxel_sizes"]).reshape(-1)[0])
    n_all = match.shape[0]
    if match_choice is not None:
        match = match[np.asarray(match_choice)]
    elif n_all > cfg.train.pos_num:
        match = match[rng.choice(range(n_all), cfg.train.pos_num, replace=False)]
    if match.shape[0] == 0:
        return None
    src_kpt, tgt_kpt = src_sds[match[:, 0]], tgt_sds[match[:, 1]]
    des_r = TS.draw_des_r(cfg, rng)
    K = src_kpt.shape[0]
    st = state64(sd)
    stats = dict(src=[], tgt=[], pose=[])
    ps = perms[0] if perms is not None else rng.choice(src.shape[0], src.shape[0], replace=False)
    s = _describe_train(st, stats["src"], hp, cfg, src, src_kpt, des_r, aligned, ps, None)
    pt = perms[1] if perms is not None else rng.choice(tgt.shape[0], tgt.shape[0], replace=False)
    angles = TS._f32(aug_angles) if aug_angles is not None else TS.draw_aug_angles(rng, K)
    t = _describe_train(st, stats["tgt"], hp, cfg, tgt, tgt_kpt, des_r, aligned, pt, angles)
    if K < 2:
        return None
    e = cfg.patch.ele_n
    params = pose_params(sd)
    pred = costnet_train(s["equi"][:, :, 1:e - 1], t["equi"][:, :, 1:e - 1], params, st, stats["pose"], hp, keep, cfg.patch.azi_n)
    gt = TS.so2_gt(s["rand_axis"], s["R"], t["R"], T, cfg.patch.azi_n, False, aug_R=t["aug_rotation"])
    return dict(pred_ind=pred, gt_ind=torch.from_numpy(gt), params=params, state=st, stats=stats, K=K, src=s, tgt=t,
                aug_angles=angles, match=match)


def grad_abs_bounds(keep, params):
    """Per CostNet parameter the contraction of its gradient evaluated on absolute values, from the float64 activations and
    output gradients kept by ``costnet_train``: |dz|^T |x| for weights, sum |dz| for biases."""
    out = {}
    for i in COST_CONVS:
        dz = keep[f"z{i}"].grad.abs()
        w = params[f"ops.{i}.weight"]
        out[f"ops.{i}.weight"] = torch.nn.grad.conv3d_weight(keep[f"x{i}"].abs(), w.shape, dz)
        out[f"ops.{i}.bias"] = dz.sum(dim=(0, 2, 3, 4))
    return out
