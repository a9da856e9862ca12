"""CPU ORACLE of the training stages' validation forward (``cfg.stage`` "Desc" / "Pose", eval mode).

TEST INFRASTRUCTURE ONLY, like ``oracle/oracle.py`` whose stages it composes.  File:line are relative to the
reference checkout:
    matching_indices   models/BUFFERX.py:498-520 (utils/SE3.transform + knn_cuda k = 1)
    so2_augment        models/patch_embedder.py:54-67 (kornia axis-angle rotation about z)
    equi_match         models/BUFFERX.py:16-36
    so2_gt             models/BUFFERX.py:86-126 (cal_so2_gt)
    train_forward      models/BUFFERX.py:148-255 (the training-stage branch of BufferX.forward)
    trainer_losses     trainer.py:187-207 (the statistics Trainer.evaluate computes from the returned dict)
The correspondence search and the augmentation use the frozen fp32 evaluation order (no FMA) of the CUDA kernels
in buffer-x_b200/csrc/bx_train.cu; EquiMatch and the SO(2) label are the reference's torch formulae on CPU.  Pinned against the reference's own forward by tests/golden/train_stages.npz
(tests/tools/gen_train_golden.py).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import oracle as O

F32 = np.float32


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=F32))


def transform(pts, T):
    """utils/SE3.transform in fp32: each row ((r0*x + r1*y) + r2*z) + t."""
    p, T = _f32(pts), _f32(T)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([(((T[j, 0] * x) + (T[j, 1] * y)) + (T[j, 2] * z)) + T[j, 3] for j in range(3)], axis=1)


def matching_indices(src, tgt, T, voxel, chunk=512):
    """[C,2] int64 ([i, nn(i)] in source order): nearest target point of every transformed source point (first minimum
    in target order wins), kept where sqrt(((dx*dx) + (dy*dy)) + (dz*dz)) < voxel."""
    q = transform(src, T)
    t = _f32(tgt)
    v = F32(voxel)
    N = q.shape[0]
    nn = np.zeros(N, dtype=np.int64)
    keep = np.zeros(N, dtype=bool)
    if t.shape[0] == 0:
        return np.zeros((0, 2), dtype=np.int64)
    for a in range(0, N, chunk):
        b = min(N, a + chunk)
        dx = q[a:b, 0, None] - t[None, :, 0]
        dy = q[a:b, 1, None] - t[None, :, 1]
        dz = q[a:b, 2, None] - t[None, :, 2]
        d2 = ((dx * dx) + (dy * dy)) + (dz * dz)
        j = np.argmin(d2, axis=1)
        nn[a:b] = j
        keep[a:b] = np.sqrt(d2[np.arange(b - a), j]) < v
    i = np.flatnonzero(keep)
    return np.stack([i, nn[i]], axis=1).astype(np.int64)


def _rotate_rows(v, R):
    """v [..,3] @ R^T per row: v'_j = (v0*R[j,0] + v1*R[j,1]) + v2*R[j,2]."""
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    return np.stack([((x * R[..., j, 0]) + (y * R[..., j, 1])) + (z * R[..., j, 2]) for j in range(3)], axis=-1)


def aug_rotations(angles):
    """[K] fp32 angles -> [K,3,3] fp32 (kornia axis_angle_to_rotation_matrix of (0, 0, angle))."""
    return O.azimuth_rotation(torch.from_numpy(_f32(angles))).numpy()


def so2_augment(delta, rand_axis, angles):
    """-> (delta [K,P,3], rand_axis [K,3], aug_R [K,3,3]) rotated patch by patch."""
    R = aug_rotations(angles)
    return _rotate_rows(_f32(delta), R[:, None]).astype(F32), _rotate_rows(_f32(rand_axis), R).astype(F32), R


def draw_aug_angles(rng, K):
    """The reference's draw (patch_embedder.py:56-59): fp64 angles r * 2 * pi, then the cast to fp32."""
    return (rng.random([K, 1]) * 2 * np.pi)[:, 0].astype(F32)


def equi_match(d1: torch.Tensor, d2: torch.Tensor) -> torch.Tensor:
    """cor[b,a] = sum_{c,k,l} d1[b,c,k,(l-a) mod L] * d2[b,c,k,l] in the reference's einsum form."""
    B, C, K, L = d1.shape
    l = torch.arange(L)
    idx = (l[None, :] - l[:, None]) % L
    x = d1[:, :, :, idx.reshape(-1)].reshape(B, C, K, L, L).permute(0, 1, 3, 2, 4).reshape(B, C, L, K * L)
    return torch.einsum("bfag,bfg->ba", x, d2.reshape(B, C, K * L))


def so2_gt(s_rand_axis, s_R, t_R, T, azi_n, integer=True, aug_R=None):
    """cal_so2_gt in torch CPU fp32, literally: the rand axis through both LRFs (and the augmentation), projection onto the
    xy plane, acos of the cosine similarity, sign from the cross product, 2 pi - angle.  int64 labels (rounded half to
    even, azi_n -> 0) or fp32 labels."""
    s = torch.from_numpy(_f32(s_rand_axis))[:, None]
    G = torch.from_numpy(_f32(T)[:3, :3])
    t = torch.matmul(s, G.transpose(-1, -2))
    s = torch.matmul(s, torch.from_numpy(_f32(s_R)))
    t = torch.matmul(t, torch.from_numpy(_f32(t_R)))
    if aug_R is not None:
        t = t @ torch.from_numpy(_f32(aug_R)).transpose(-1, -2)
    z = torch.zeros_like(t)
    z[:, :, -1] = 1
    proj = F.normalize(t - torch.sum(t * z, dim=-1, keepdim=True) * z, p=2, dim=-1)
    s, proj, z = s[:, 0], proj[:, 0], z[:, 0]
    ang = torch.acos(F.cosine_similarity(s, proj).clamp(min=-1, max=1))
    neg = torch.sum(torch.linalg.cross(s, proj, dim=-1) * z, dim=-1) < 0
    ang[neg] = 2 * np.pi - ang[neg]
    lab = ang * azi_n / (2 * np.pi)
    if integer:
        lab = torch.round(lab)
        lab[lab == azi_n] = 0
        return lab.to(torch.int64).numpy()
    lab[lab == azi_n] = 0
    return lab.numpy()


def draw_des_r(cfg, rng):
    """The per-dataset descriptor radius of the training branch (BUFFERX.py:175-198)."""
    name, center = cfg.data.dataset, cfg.patch.des_r
    if name == "3DMatch":
        lo, hi = center * 0.5, center * 1.5
        return np.round(np.clip(rng.normal(center, (hi - lo) / 6, 1), lo, hi), 2)[0]
    if name == "KITTI":
        vals = {3.0: [2.0, 2.5, 3.0, 3.5, 4.0], 0.3: [0.2, 0.25, 0.3, 0.35, 0.4]}[center]
        return rng.choice(vals, p=[0.2, 0.2, 0.2, 0.2, 0.2])
    return center


def train_forward(stage, sd, cfg, data, rng=None, perms=None, aug_angles=None, match_choice=None, z_axes=None, keep=False):
    """The training-stage branch of ``BufferX.forward`` in eval mode.  NumPy draws come from ``rng`` (default: the
    global RNG, consumed in the reference's order: match subsampling, des_r, source permutation, target permutation,
    augmentation angles); ``perms`` (src, tgt), ``aug_angles`` and ``match_choice`` replace the respective draws.
    ``z_axes`` (src, tgt): impose these LRF z axes (replaying a reference run).  Returns the reference's dict or None;
    with keep=True the dict also carries ``aux`` (intermediate results)."""
    assert stage in ("Desc", "Pose")
    rng = np.random if rng is None else rng
    src, tgt = _f32(data["src_fds_pcd"]), _f32(data["tgt_fds_pcd"])
    src_sds, tgt_sds = _f32(data["src_sds_pcd"]), _f32(data["tgt_sds_pcd"])
    T = _f32(data["relt_pose"])
    aligned = bool(data["is_aligned_to_global_z"])
    match = matching_indices(src_sds, tgt_sds, T, np.asarray(data["voxel_sizes"]).reshape(-1)[0])
    n_all = match.shape[0]
    if match_choice is not None:
        match = match[np.asarray(match_choice)]
    elif n_all > cfg.train.pos_num:
        match = match[rng.choice(range(n_all), cfg.train.pos_num, replace=False)]
    if match.shape[0] == 0:
        print(f"{data.get('src_id')} {data.get('tgt_id')} has no keypts")
        return None
    src_kpt, tgt_kpt = src_sds[match[:, 0]], tgt_sds[match[:, 1]]
    des_r = draw_des_r(cfg, rng)
    K = src_kpt.shape[0]
    ps = perms[0] if perms is not None else rng.choice(src.shape[0], src.shape[0], replace=False)
    zs, zt = (None, None) if z_axes is None else z_axes
    s = O.describe(sd, cfg, src, src_kpt, des_r, aligned, ps, keep=keep, z_axis=zs)
    pt = perms[1] if perms is not None else rng.choice(tgt.shape[0], tgt.shape[0], replace=False)
    angles = None
    if stage == "Pose":
        angles = _f32(aug_angles) if aug_angles is not None else draw_aug_angles(rng, K)
    t = _describe_aug(sd, cfg, tgt, tgt_kpt, des_r, aligned, pt, angles, keep, zt)
    azi_n = cfg.patch.azi_n
    aux = dict(match_all=n_all, match=match, des_r=des_r, src=s, tgt=t, aug_angles=angles)
    if K < 2:
        print(f"{data.get('src_id')} {data.get('tgt_id')} don't have enough patches")
        return None
    if stage == "Desc":
        with torch.no_grad():
            score = equi_match(s["equi"], t["equi"])
        out = dict(src_kpt=torch.from_numpy(src_kpt), tgt_kpt=torch.from_numpy(tgt_kpt), src_des=s["desc"], tgt_des=t["desc"],
                   equi_score=score,
                   gt_label=torch.from_numpy(so2_gt(s["rand_axis"].numpy(), s["R"].numpy(), t["R"].numpy(), T, azi_n, True)))
    else:
        e = cfg.patch.ele_n
        with torch.no_grad():
            pred = O.cost_volume(s["equi"][:, :, 1:e - 1], t["equi"][:, :, 1:e - 1], sd, azi_n)
        gt = so2_gt(s["rand_axis"].numpy(), s["R"].numpy(), t["R"].numpy(), T, azi_n, False, aug_R=t["aug_rotation"].numpy())
        out = dict(pred_ind=pred, gt_ind=torch.from_numpy(gt))
    if keep:
        out["aux"] = aux
    return out


def _describe_aug(sd, cfg, pts, kpts, des_r, aligned, perm, angles, keep, z_axis):
    """``describe`` with the SO(2) augmentation between the normalisation and SPT (patch_embedder.py:54-70)."""
    if angles is None:
        return O.describe(sd, cfg, pts, kpts, des_r, aligned, perm, keep=keep, z_axis=z_axis)
    P = cfg.patch.num_points_per_patch
    rad_n, azi_n, ele_n = cfg.patch.rad_n, cfg.patch.azi_n, cfg.patch.ele_n
    idx, patches = O.select_patches(pts, perm, kpts, des_r, P)
    delta, Rt, rand_axis, z_used = O.lrf(patches, des_r, aligned, z_axis=z_axis, want_z=True)
    delta, rand_axis, aug_R = so2_augment(delta, rand_axis, angles)
    inv, vidx = O.spt(delta, rad_n, azi_n, ele_n, cfg.patch.delta / rad_n, cfg.patch.voxel_sample)
    with torch.no_grad():
        feat = O.pnt_max(torch.from_numpy(inv), sd)
        x = O.cyl_net(feat.view(feat.shape[0], feat.shape[1], rad_n, ele_n, azi_n), sd)
        desc, equi = O.pool_desc(x, sd)
    out = dict(desc=desc, equi=equi, R=torch.from_numpy(Rt), rand_axis=torch.from_numpy(rand_axis),
               aug_rotation=torch.from_numpy(aug_R))
    if keep:
        out.update(idx=idx, patches=patches, delta=delta, inv=inv, vidx=vidx, feat=feat, x=x, z=z_used)
    return out


# --------------------------------------------------------------------------- #
# the statistics Trainer.evaluate computes from the returned dict
# --------------------------------------------------------------------------- #
def _contrastive(anchor, positive, kpts, pos_margin=0.1, neg_margin=1.4, safe_radius=0.10):
    """Batch-hard contrastive loss (loss/desc_loss.py ContrastiveLoss, euclidean metric) -> (loss, accuracy %)."""
    def cdist(a, b):
        return torch.sqrt(torch.sum((a[:, None] - b[None]) ** 2, dim=-1) + 1e-12)
    dist = cdist(anchor, positive)
    dk = np.eye(kpts.shape[0]) * 10 + cdist(kpts, kpts).numpy()
    add = torch.zeros_like(dist)
    add[np.where(dk < safe_radius)] += 10
    dist = dist + add
    same = torch.eye(dist.shape[0], dtype=torch.bool).float()
    furthest_pos = torch.max(dist * same, dim=1).values
    closest_neg = torch.min(dist + 1e5 * same, dim=1).values
    diff = furthest_pos - closest_neg
    acc = (diff < 0).sum() * 100.0 / diff.shape[0]
    loss = torch.clamp(furthest_pos - pos_margin, min=0) + torch.clamp(neg_margin - closest_neg, min=0)
    return torch.mean(loss), acc


def trainer_losses(stage, out):
    """desc_loss / desc_acc / eqv_loss / eqv_acc (stage "Desc") or match_loss (stage "Pose") of one output dict, on CPU."""
    o = {k: (v.detach().cpu() if torch.is_tensor(v) else v) for k, v in out.items()}
    if stage == "Desc":
        dl, acc = _contrastive(o["src_des"].float(), o["tgt_des"].float(), o["src_kpt"].float())
        eqv = F.cross_entropy(o["equi_score"].float(), o["gt_label"].long())
        pre = torch.argmax(o["equi_score"], dim=1)
        return dict(desc_loss=float(dl), desc_acc=float(acc), eqv_loss=float(eqv),
                    eqv_acc=float((pre == o["gt_label"]).sum() / pre.shape[0]))
    return dict(match_loss=float(F.huber_loss(o["pred_ind"].float(), o["gt_ind"].float())))


# --------------------------------------------------------------------------- #
# the synthetic cases of tests/golden/train_stages.npz
# --------------------------------------------------------------------------- #
GOLDEN_CASES = ("c1_draw", "c1_isolated")


def golden_case(name, stage):
    """-> (cfg, state_dict, data, seed) of a stored case.  "c1_draw": the C1 pair with second-level clouds at the config's
    voxel size and pos_num 128, so the match subsampling draw runs.  "c1_isolated": a 1000-point C1 pair, second-level
    clouds at 0.2 m plus one isolated correspondence (an empty ball query), z-aligned, no subsampling."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C1")
    cfg.stage = stage
    if name == "c1_draw":
        seed = 0
        cfg.train.pos_num = 128
        data = add_training_clouds(make_pair("C1", seed), cfg)
    elif name == "c1_isolated":
        seed = 1
        cfg.train.pos_num = 100000
        data = add_training_clouds(make_pair("C1", seed, 1000, 1000), cfg, voxel=0.2, isolated=True)
        data["is_aligned_to_global_z"] = True
    else:
        raise ValueError(name)
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    return cfg, sd, data, seed
