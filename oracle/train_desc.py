"""CPU ORACLE of the Desc stage's training step (``cfg.stage`` "Desc", ``model.train()``), in float64.

TEST INFRASTRUCTURE ONLY.  File:line are relative to the reference checkout:
    training step      trainer.py:93-167 (forward, 4 ContrastiveLoss(src_des, tgt_des, cdist(tgt_kpt, tgt_kpt)) +
                       CrossEntropy(equi_score, gt_label), backward, optimizer.step())
    frozen Pose        train.py:36-48 (requires_grad=False on every module but Desc)
    Desc forward       models/patch_embedder.py:44-90, models/patchnet.py:68-84, every BatchNorm in training mode
    EquiMatch          models/BUFFERX.py:16-36
The integer decisions (match list, patches, frames, SPT selection) and the fp32 de-rotated point-layer inputs are those of
oracle/oracle.py and oracle/train_stages.py; from the point layer on everything is float64 torch on the CPU with the
descriptor network's parameters as autograd leaves.  The max over a voxel's samples is F.max_pool2d, as in the reference:
its gradient goes to the first maximal sample.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import oracle as O
from oracle import train_stages as TS
from oracle.train_step import CYL_CONVS, state64

AFFINE_BN = ("pnt_layer.1", "pool_layer.1", "pool_layer.4")


def desc_params(sd, pfx="Desc."):
    """MiniSpinNet's parameters as float64 leaves requiring grad, keyed without the prefix ("pnt_layer.0.weight", ...)."""
    from oracle.train_step_cases import DESC_BN
    bn_affine = {k[len(pfx):] for k in DESC_BN if not k.startswith(pfx + "conv_net")}
    out = {}
    for k in sd:
        if not k.startswith(pfx) or k.split(".")[-1] not in ("weight", "bias"):
            continue
        mod = k[len(pfx):].rsplit(".", 1)[0]
        if mod.startswith("conv_net.ops.") and int(mod.split(".")[-1]) not in CYL_CONVS:
            continue                                   # (non-affine BatchNorms have no parameters anyway)
        if mod in bn_affine or mod.startswith("conv_net") or mod in ("pnt_layer.0", "pool_layer.0", "pool_layer.3"):
            out[k[len(pfx):]] = sd[k].detach().double().clone().requires_grad_(True)
    return out


def _bn(x, st, key, stats, hp, w=None, b=None, keep=None, kname=None):
    """Training-mode BatchNorm (momentum, eps from hp[key]) as x^ = batch_norm(x) without affine, then x^ gamma + beta:
    the same value and running update as torch's affine BatchNorm; keeps x^ and the output (retain_grad) for the bounds."""
    momentum, eps = hp[key]
    if momentum is None:
        momentum = 1.0 / float(st[key + ".num_batches_tracked"] + 1)
    dims = [d for d in range(x.dim()) if d != 1]
    stats.append((x.detach().mean(dims), x.detach().var(dims, unbiased=False)))
    st[key + ".num_batches_tracked"] = st[key + ".num_batches_tracked"] + 1
    xh = F.batch_norm(x, st[key + ".running_mean"], st[key + ".running_var"], None, None, training=True, momentum=momentum, eps=eps)
    if w is None:
        return xh
    shape = [1, -1] + [1] * (x.dim() - 2)
    y = xh * w.view(shape) + b.view(shape)
    if keep is not None and y.requires_grad:
        y.retain_grad()
        keep[kname + ".xh"] = xh.detach()
        keep[kname + ".y"] = y
    return y


def _conv(fn, x, params, name, keep):
    z = fn(x, params[name + ".weight"], params[name + ".bias"])
    if keep is not None:
        keep[name + ".x"] = x.detach()
        if z.requires_grad:
            z.retain_grad()
            keep[name + ".z"] = z
    return z


def desc_train(inv, params, st, stats, hp, keep=None, rad_n=3, ele_n=7, azi_n=20, pfx="Desc."):
    """MiniSpinNet in training mode, float64, from the de-rotated samples inv [K, V, nv, 3] -> (desc [K, 32],
    equi [K, 32, ele_n, azi_n]) differentiable in ``params`` (desc_params).  ``st``: the float64 state whose running
    statistics are updated; ``stats`` receives (batch mean, batch variance) of every BatchNorm in module order; ``keep``
    (a dict, shared by several calls only if each call gets its own) records each convolution's input and output."""
    x = torch.as_tensor(np.asarray(inv)).double().permute(0, 3, 1, 2)
    nv = x.shape[3]
    z = _conv(F.conv2d, x, params, "pnt_layer.0", keep)
    y = _bn(z, st, pfx + "pnt_layer.1", stats, hp, params["pnt_layer.1.weight"], params["pnt_layer.1.bias"], keep, "pnt_layer.1")
    x = F.max_pool2d(F.relu(y), kernel_size=(1, nv)).squeeze(3)
    K = x.shape[0]
    x = x.reshape(K, 16, rad_n, ele_n, azi_n)
    c = pfx + "conv_net.ops."
    for i in CYL_CONVS:
        name = f"conv_net.ops.{i}"
        z = _conv(F.conv3d if i == 0 else F.conv2d, O._pad_cyl(x), params, name, keep)
        x = z if i == 21 else F.relu(_bn(z, st, c + f"{i + 1}", stats, hp))
        if i == 0:
            x = x.squeeze(2)
    z = _conv(F.conv2d, x, params, "pool_layer.0", keep)
    w = F.relu(_bn(z, st, pfx + "pool_layer.1", stats, hp, params["pool_layer.1.weight"], params["pool_layer.1.bias"], keep, "pool_layer.1"))
    z = _conv(F.conv2d, w, params, "pool_layer.3", keep)
    w = F.relu(_bn(z, st, pfx + "pool_layer.4", stats, hp, params["pool_layer.4.weight"], params["pool_layer.4.bias"], keep, "pool_layer.4"))
    f = F.avg_pool2d(x * w, kernel_size=(x.shape[2], x.shape[3])).view(K, -1)
    return F.normalize(f, p=2, dim=1), F.normalize(x, p=2, dim=1)


def equi_match(s, t):
    """EquiMatch (BUFFERX.py:16-36): cor[k, a] = sum_{c, e, l} s[k, c, e, (l - a) mod L] t[k, c, e, l]."""
    L = s.shape[-1]
    l = torch.arange(L)
    idx = (l[None, :] - l[:, None]) % L                         # [a, l]
    return torch.einsum("kceal,kcel->ka", s[..., idx], t)


def desc_loss(src_des, tgt_des, tgt_kpt, equi_score, gt_label):
    """Trainer.train_epoch's Desc loss: 4 ContrastiveLoss(src_des, tgt_des, cdist(tgt_kpt, tgt_kpt)) + CE(equi_score, gt)."""
    dl, _ = TS._contrastive(src_des, tgt_des, torch.as_tensor(np.asarray(tgt_kpt)).double())
    return 4 * dl + F.cross_entropy(equi_score, torch.as_tensor(np.asarray(gt_label)).long())


def grad_abs_bounds(keep, params):
    """Per parameter the contraction of its gradient on absolute values, from the activations and output gradients kept
    by ``desc_train`` (one dict per call; pass a list to add the calls): |dz|^T |x| for convolution weights, sum |dz| for
    their biases, sum |dy| |x^| and sum |dy| for the affine BatchNorms' weight and bias."""
    keeps = keep if isinstance(keep, list) else [keep]
    out = {k: torch.zeros_like(v, dtype=torch.float64) for k, v in params.items()}
    for kp in keeps:
        for k in params:
            mod, kind = k.rsplit(".", 1)
            if mod in AFFINE_BN:
                dy = kp[mod + ".y"].grad.abs()
                dims = [d for d in range(dy.dim()) if d != 1]
                out[k] += (dy * kp[mod + ".xh"].abs()).sum(dims) if kind == "weight" else dy.sum(dims)
                continue
            dz = kp[mod + ".z"].grad.abs()
            if kind == "bias":
                out[k] += dz.sum(dim=[d for d in range(dz.dim()) if d != 1])
            else:
                fn = torch.nn.grad.conv3d_weight if dz.dim() == 5 else torch.nn.grad.conv2d_weight
                out[k] += fn(kp[mod + ".x"].abs(), params[k].shape, dz)
    return out


def check_grads(desc, params64, absb, what):
    """Every MiniSpinNet gradient elementwise within G_ELEM of the contraction on absolute values and within G_NORM of the
    float64 gradient's norm (a norm ~0, e.g. the biases of BatchNorm'd convolutions, only elementwise) -> ratios."""
    from oracle.train_step_cases import G_ELEM, G_NORM
    bad, ratios = [], {}
    named = dict(desc.named_parameters())
    for k, p64 in params64.items():
        p = named[k]
        assert p.grad is not None, k
        g, g64 = p.grad.detach().cpu().double(), p64.grad
        lim = G_ELEM * absb[k] + 1e-30
        e = float(((g - g64).abs() / lim).max())
        ratios[k] = e
        if e > 1.0:
            bad.append(f"{k}: elementwise err {e:.3g} x bound")
        if float(g64.norm()) > 10 * G_ELEM * float(absb[k].norm()):
            n = float((g - g64).norm()) / float(g64.norm())
            ratios[k + "/norm"] = n / G_NORM
            if n > G_NORM:
                bad.append(f"{k}: norm err {n:.3g}")
    print(what, "gradient error / bound:", {k: round(v, 3) for k, v in ratios.items()})
    assert not bad, f"{what}: " + "; ".join(bad)
    return ratios


def _describe(cfg, pts, kpts, des_r, aligned, perm):
    P = cfg.patch.num_points_per_patch
    _, patches = O.select_patches(pts, perm, kpts, des_r, P)
    delta, Rt, rand_axis = O.lrf(patches, des_r, aligned)
    inv, _ = O.spt(delta, cfg.patch.rad_n, cfg.patch.azi_n, cfg.patch.ele_n, cfg.patch.delta / cfg.patch.rad_n, cfg.patch.voxel_sample)
    return inv, Rt, rand_axis


def train_step(sd, hp, cfg, data, rng=None):
    """The Desc stage's training forward (BufferX.forward under model.train(), BUFFERX.py:148-255), NumPy draws in the
    reference's order (match sub-sampling, des_r, source permutation, target permutation) from ``rng`` (default the global
    RNG).  -> None (no matches / fewer than two patches) or dict(src_des, tgt_des, equi_score (float64, differentiable in
    ``params``), src_equi, tgt_equi, gt_label, tgt_kpt, params, state, stats (src / tgt), inv (src, tgt), K)."""
    rng = np.random if rng is None else rng
    src, tgt = TS._f32(data["src_fds_pcd"]), TS._f32(data["tgt_fds_pcd"])
    src_sds, tgt_sds = TS._f32(data["src_sds_pcd"]), TS._f32(data["tgt_sds_pcd"])
    T = TS._f32(data["relt_pose"])
    aligned = bool(data["is_aligned_to_global_z"])
    match = TS.matching_indices(src_sds, tgt_sds, T, np.asarray(data["voxel_sizes"]).reshape(-1)[0])
    n_all = match.shape[0]
    if n_all > cfg.train.pos_num:
        match = match[rng.choice(range(n_all), cfg.train.pos_num, replace=False)]
    if match.shape[0] == 0:
        return None
    src_kpt, tgt_kpt = src_sds[match[:, 0]], tgt_sds[match[:, 1]]
    des_r = TS.draw_des_r(cfg, rng)
    K = src_kpt.shape[0]
    ps = rng.choice(src.shape[0], src.shape[0], replace=False)
    inv_s, R_s, ra_s = _describe(cfg, src, src_kpt, des_r, aligned, ps)
    pt = rng.choice(tgt.shape[0], tgt.shape[0], replace=False)
    inv_t, R_t, _ = _describe(cfg, tgt, tgt_kpt, des_r, aligned, pt)
    if K < 2:
        return None
    st, params, stats = state64(sd), desc_params(sd), dict(src=[], tgt=[])
    d_s, e_s = desc_train(inv_s, params, st, stats["src"], hp)
    d_t, e_t = desc_train(inv_t, params, st, stats["tgt"], hp)
    gt = TS.so2_gt(ra_s, R_s, R_t, T, cfg.patch.azi_n, True)
    return dict(src_des=d_s, tgt_des=d_t, src_equi=e_s, tgt_equi=e_t, equi_score=equi_match(e_s, e_t), gt_label=torch.from_numpy(np.asarray(gt)),
                tgt_kpt=tgt_kpt, params=params, state=st, stats=stats, inv=(inv_s, inv_t), K=K)
