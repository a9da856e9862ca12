"""Seeded synthetic registration pairs shaped like the reference's datasets.

There is no dataset (and no network) in this environment, so every test and
benchmark runs on synthetic pairs that reproduce the *input contract* of the hot
path: the dict produced by ``collate_fn_descriptor``
(``/root/reference/dataset/dataloader.py:108-122``) of which inference reads
``src_fds_pcd`` / ``tgt_fds_pcd`` (float32 [N,3], already down-sampled and
shuffled), ``is_aligned_to_global_z`` and ``relt_pose``
(``/root/reference/models/BUFFERX.py:268,295``).

Each pair is *two sensor-frame views of one world scene* (every cloud has its own
sensor at the origin, ground truth = relative pose): the reference's local
reference frame disambiguates its z-axis sign with the vector towards the sensor
origin (``/root/reference/utils/common.py:718``), so "a cloud and a rigidly moved
copy" would flip LRF signs for a reason the real pipeline never sees
(SURVEY.md section 8.1 item 14).

Workloads (BASELINE.json ``configs``):
    C1  2x5000 pts, surface-like, indoor cfg, 256 key-points, 1 scale, 1000 RANSAC iters
    C2  2x20000 pts, 6x6x3 m room, ~60 % overlap, 1500 key-points, 3 scales, 50000 iters
    C3  2x120000 pts, LiDAR-shaped outdoor, 2048 key-points, 3 scales, 50000 iters
    C5  60000 vs 30000 pts heterogeneous outdoor pair
"""
from __future__ import annotations

import math
import os

import numpy as np

from .config import make_cfg

__all__ = ["make_pair", "workload_cfg", "add_training_clouds", "WORKLOADS"]

WORKLOADS = ("C1", "C2", "C3", "C5")


# --------------------------------------------------------------------------- #
# geometry helpers
# --------------------------------------------------------------------------- #
def _rot_z(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _rot_x(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])


def _se3(R, t):
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = t
    return T


class _Scene:
    """A set of parallelograms / cylinders sampled uniformly by area."""

    def __init__(self):
        self.prims = []  # (area, kind, params)

    def add_rect(self, o, e1, e2):
        o, e1, e2 = (np.asarray(v, dtype=np.float64) for v in (o, e1, e2))
        self.prims.append((float(np.linalg.norm(np.cross(e1, e2))), "rect", (o, e1, e2)))

    def add_box(self, lo, hi, bottom=False):
        lo, hi = np.asarray(lo, float), np.asarray(hi, float)
        d = hi - lo
        ex, ey, ez = np.array([d[0], 0, 0]), np.array([0, d[1], 0]), np.array([0, 0, d[2]])
        self.add_rect(lo, ex, ez)
        self.add_rect(lo + ey, ex, ez)
        self.add_rect(lo, ey, ez)
        self.add_rect(lo + ex, ey, ez)
        self.add_rect(lo + ez, ex, ey)
        if bottom:
            self.add_rect(lo, ex, ey)

    def add_cylinder(self, c, r, h):
        self.prims.append((2 * math.pi * r * h, "cyl", (np.asarray(c, float), float(r), float(h))))

    def add_ground_annulus(self, r0, r1, z):
        # density ~ 1/r (ring pattern of a spinning LiDAR): sample r uniformly
        self.prims.append((0.35 * math.pi * (r1 * r1 - r0 * r0) / max(r1, 1.0), "ann", (float(r0), float(r1), float(z))))

    def sample(self, rng, n):
        areas = np.array([p[0] for p in self.prims])
        which = rng.choice(len(self.prims), size=n, p=areas / areas.sum())
        out = np.empty((n, 3))
        u = rng.random(n)
        v = rng.random(n)
        for i, (_, kind, prm) in enumerate(self.prims):
            m = which == i
            if not m.any():
                continue
            if kind == "rect":
                o, e1, e2 = prm
                out[m] = o + u[m, None] * e1 + v[m, None] * e2
            elif kind == "cyl":
                c, r, h = prm
                a = 2 * math.pi * u[m]
                out[m] = c + np.stack([r * np.cos(a), r * np.sin(a), h * v[m]], 1)
            else:
                r0, r1, z = prm
                rr = r0 + (r1 - r0) * u[m]
                a = 2 * math.pi * v[m]
                out[m] = np.stack([rr * np.cos(a), rr * np.sin(a), np.full(m.sum(), z)], 1)
        return out


def _room(rng, sx, sy, sz, n_boxes):
    s = _Scene()
    s.add_rect([0, 0, 0], [sx, 0, 0], [0, sy, 0])          # floor
    s.add_rect([0, 0, sz], [sx, 0, 0], [0, sy, 0])         # ceiling
    s.add_rect([0, 0, 0], [sx, 0, 0], [0, 0, sz])
    s.add_rect([0, sy, 0], [sx, 0, 0], [0, 0, sz])
    s.add_rect([0, 0, 0], [0, sy, 0], [0, 0, sz])
    s.add_rect([sx, 0, 0], [0, sy, 0], [0, 0, sz])
    for _ in range(n_boxes):                               # furniture
        d = rng.uniform([0.3, 0.3, 0.3], [min(1.4, sx / 3), min(1.4, sy / 3), min(1.6, sz * 0.6)])
        lo = np.array([rng.uniform(0.1, sx - d[0] - 0.1), rng.uniform(0.1, sy - d[1] - 0.1), 0.0])
        s.add_box(lo, lo + d)
    for _ in range(max(1, n_boxes // 2)):                  # slanted panels (break the Manhattan symmetry)
        o = rng.uniform([0.3, 0.3, 0.3], [sx - 1.2, sy - 1.2, sz - 1.0])
        e1 = rng.normal(size=3)
        e1 *= rng.uniform(0.5, 1.2) / np.linalg.norm(e1)
        e2 = np.cross(e1, rng.normal(size=3))
        e2 *= rng.uniform(0.4, 1.0) / np.linalg.norm(e2)
        s.add_rect(o, e1, e2)
    return s


def _street(rng):
    s = _Scene()
    s.add_ground_annulus(2.5, 80.0, 0.0)
    for _ in range(14):                                    # building facades
        a = rng.uniform(0, 2 * math.pi)
        d = rng.uniform(10, 60)
        c = np.array([d * math.cos(a), d * math.sin(a), 0.0])
        tang = np.array([-math.sin(a + rng.uniform(-0.6, 0.6)), math.cos(a + rng.uniform(-0.6, 0.6)), 0.0])
        w, h = rng.uniform(8, 30), rng.uniform(4, 15)
        s.add_rect(c - 0.5 * w * tang, w * tang, [0, 0, h])
    for _ in range(30):                                    # poles / trunks
        a = rng.uniform(0, 2 * math.pi)
        d = rng.uniform(4, 50)
        s.add_cylinder([d * math.cos(a), d * math.sin(a), 0.0], rng.uniform(0.1, 0.4), rng.uniform(2, 8))
    for _ in range(12):                                    # parked cars
        a = rng.uniform(0, 2 * math.pi)
        d = rng.uniform(5, 40)
        lo = np.array([d * math.cos(a), d * math.sin(a), 0.0])
        s.add_box(lo, lo + rng.uniform([1.6, 1.6, 1.3], [4.5, 4.5, 1.8]))
    return s


def _view(scene, rng, n, T_ws, fov_cos, rng_max, sigma, min_range):
    """n points of the scene seen from sensor pose T_ws (sensor->world), in the sensor frame."""
    R, c = T_ws[:3, :3], T_ws[:3, 3]
    fwd = R[:, 0]
    got = []
    have = 0
    for _ in range(64):
        p = scene.sample(rng, 4 * n)
        d = p - c
        r = np.linalg.norm(d, axis=1)
        keep = (r > min_range) & (r < rng_max) & ((d @ fwd) > fov_cos * r)
        p = p[keep]
        got.append(p)
        have += len(p)
        if have >= n:
            break
    p = np.concatenate(got, 0)[:n]
    if len(p) < n:
        raise RuntimeError("synthetic scene too small for the requested view")
    p = p + rng.normal(scale=sigma, size=p.shape)
    return ((p - c) @ R).astype(np.float32)  # R^T (p - c)


# --------------------------------------------------------------------------- #
# public API
# --------------------------------------------------------------------------- #
def workload_cfg(name: str):
    """The reference-style cfg tree for a BASELINE.json workload (``cfg.stage == 'test'``)."""
    if name in ("C1", "C2"):
        cfg = make_cfg("3DMatch")
    elif name == "C3":
        cfg = make_cfg("KITTI")
    elif name == "C5":
        cfg = make_cfg("TIERS_hetero")
    else:
        raise ValueError(f"unknown workload {name}")
    cfg.stage = "test"
    if name == "C1":
        cfg.patch.num_fps = 256
        cfg.patch.num_scales = 1
        cfg.patch.search_radius_thresholds = [5]
        cfg.match.iter_n = 1000
    if name == "C3":
        cfg.patch.num_fps = 2048
    return cfg


def make_pair(name: str = "C2", seed: int = 0, n_src: int | None = None, n_tgt: int | None = None):
    """Return the reference's ``data_source`` dict (numpy float32 arrays) for one synthetic pair."""
    rng = np.random.default_rng(1000003 * (WORKLOADS.index(name) + 1) + seed)
    if name == "C1":
        ns, nt = n_src or 5000, n_tgt or 5000
        scene = _room(rng, 3.0, 3.0, 3.0, n_boxes=2)
        c_s = np.array([1.2, 1.3, 1.4]) + rng.uniform(-0.1, 0.1, 3)
        T_s = _se3(_rot_z(rng.uniform(0, 2 * math.pi)), c_s)
        T_rel = _se3(_rot_z(math.radians(30)) @ _rot_x(math.radians(10)), np.array([0.3, -0.2, 0.1]))
        fov, rmax, sigma, rmin = -1.0, 10.0, 0.002, 0.3
        aligned = False
    elif name == "C2":
        ns, nt = n_src or 20000, n_tgt or 20000
        scene = _room(rng, 6.0, 6.0, 3.0, n_boxes=7)
        c_s = np.array([2.4, 2.6, 1.5]) + rng.uniform(-0.3, 0.3, 3)
        T_s = _se3(_rot_z(rng.uniform(0, 2 * math.pi)) @ _rot_x(rng.uniform(-0.15, 0.15)), c_s)
        T_rel = _se3(_rot_z(math.radians(rng.uniform(25, 45))) @ _rot_x(math.radians(rng.uniform(-8, 8))),
                     rng.uniform([0.4, -0.6, -0.1], [0.9, 0.6, 0.1]))
        fov, rmax, sigma, rmin = math.cos(math.radians(75)), 12.0, 0.002, 0.3   # 150 deg cone -> ~60 % overlap
        aligned = False
    elif name in ("C3", "C5"):
        ns, nt = (n_src or 120000, n_tgt or 120000) if name == "C3" else (n_src or 60000, n_tgt or 30000)
        scene = _street(rng)
        T_s = _se3(_rot_z(rng.uniform(0, 2 * math.pi)), np.array([0.0, 0.0, 1.73]))
        base = 10.0 if name == "C3" else 2.0
        T_rel = _se3(_rot_z(math.radians(5.0)), np.array([base, 0.3, 0.0]))
        fov, rmax, sigma, rmin = -1.0, 80.0, 0.01, 2.0
        aligned = True
    else:
        raise ValueError(f"unknown workload {name}")
    # target sensor pose: T_t = T_s @ T_rel^-1  =>  relt_pose (src->tgt) = T_t^-1 T_s = T_rel
    T_t = T_s @ np.linalg.inv(T_rel)
    src = _view(scene, rng, ns, T_s, fov, rmax, sigma, rmin)
    tgt = _view(scene, rng, nt, T_t, fov, rmax, sigma, rmin)
    return {
        "src_fds_pcd": src,
        "tgt_fds_pcd": tgt,
        "relt_pose": T_rel.astype(np.float32),
        "src_id": f"{name}_{seed}_src",
        "tgt_id": f"{name}_{seed}_tgt",
        "scene_name": f"synthetic_{name}",
        "sensor": "synthetic",
        "voxel_sizes": np.array([0.035 if not aligned else 0.3], dtype=np.float32),
        "dataset_names": ["synthetic"],
        "sphericity": np.array([0.0], dtype=np.float32),
        "is_aligned_to_global_z": aligned,
    }


def _voxel_means(pts, voxel):
    """Voxel grid down-sample (Open3D's voxel_down_sample rule: cells of ``voxel`` from min - voxel/2, fp64 mean of the
    points of a cell), cells in ascending (ix, iy, iz) key order, fp32 out."""
    P = np.asarray(pts, dtype=np.float64)
    iv = np.floor((P - (P.min(axis=0) - voxel * 0.5)) / voxel).astype(np.int64)
    keys = iv[:, 0] | (iv[:, 1] << 21) | (iv[:, 2] << 42)
    uk, inv, cnt = np.unique(keys, return_inverse=True, return_counts=True)
    sums = np.zeros((len(uk), 3))
    np.add.at(sums, inv, P)
    return (sums / cnt[:, None]).astype(np.float32)


def add_training_clouds(data, cfg, voxel=None, isolated=False):
    """Make a synthetic pair look like the training loader's collate dict: ``src_sds_pcd`` / ``tgt_sds_pcd`` (second-level
    clouds, voxel down-sample of the first-level clouds at ``cfg.data.voxel_size_0`` unless ``voxel`` is given) and
    ``voxel_sizes`` = [voxel].  ``isolated=True`` appends one corresponding point pair (p and relt_pose p) at least 2 m
    away from both first-level clouds: a key-point whose ball query comes back empty."""
    v = float(cfg.data.voxel_size_0 if voxel is None else voxel)
    out = dict(data)
    src_sds, tgt_sds = _voxel_means(data["src_fds_pcd"], v), _voxel_means(data["tgt_fds_pcd"], v)
    if isolated:
        T = np.asarray(data["relt_pose"], dtype=np.float64)
        p = np.asarray(data["src_fds_pcd"], dtype=np.float64).max(axis=0) + 3.0
        q = T[:3, :3] @ p + T[:3, 3]
        for cloud, x in ((data["src_fds_pcd"], p), (data["tgt_fds_pcd"], q)):
            if np.sqrt(((np.asarray(cloud, dtype=np.float64) - x) ** 2).sum(1)).min() < 2.0:
                raise RuntimeError("isolated point is not isolated")
        src_sds = np.concatenate([src_sds, p[None].astype(np.float32)])
        tgt_sds = np.concatenate([tgt_sds, q[None].astype(np.float32)])
    out["src_sds_pcd"], out["tgt_sds_pcd"] = src_sds, tgt_sds
    out["voxel_sizes"] = np.array([v], dtype=np.float32)
    return out


POSE_TRAINED = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "pose_synth_trained.npz")


def init_synthetic_weights(model, seed: int = 123, logit_gain: float = 4.0, trained_pose: bool = False):
    """Deterministic stand-in for the (unavailable offline) trained checkpoint.

    Seeded He-uniform initialisation of every Conv layer (variance preserving through the ReLU stacks:
    with torch's default init the signal decays below the biases after a few layers and every patch gets
    the same descriptor), non-trivial BatchNorm running statistics (mean ~ N(0, 0.1), var ~ U(0.5, 1.5),
    affine weight ~ U(0.5, 1.5), bias ~ N(0, 0.1)) so that BN folding is exercised, and a gain on
    CostNet's last layer so that the soft arg-max is not degenerate (SURVEY 8.1.13).
    """
    import torch

    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mod in model.modules():
            if isinstance(mod, (torch.nn.Conv2d, torch.nn.Conv3d)):
                fan_in = mod.in_channels * int(np.prod(mod.kernel_size))
                bound = math.sqrt(6.0 / fan_in)
                mod.weight.copy_((torch.rand(mod.weight.shape, generator=g) * 2 - 1) * bound)
                mod.bias.copy_((torch.rand(mod.bias.shape, generator=g) * 2 - 1) * 0.05)
            elif isinstance(mod, (torch.nn.BatchNorm2d, torch.nn.BatchNorm3d)):
                mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
                if mod.affine:
                    mod.weight.copy_(torch.rand(mod.weight.shape, generator=g) + 0.5)
                    mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.1)
        last = model.Pose.conv.ops[27]
        last.weight.mul_(logit_gain)
        last.bias.mul_(logit_gain)
        # trained_pose=True: CostNet fitted on synthetic pairs for exactly this seeded descriptor network
        # (tests/tools/train_costnet.py, pairs disjoint from the bench / test pairs): with it the synthetic C2 pairs
        # actually register (RRE ~1.7 deg, RTE ~5 cm against the ground truth, ~40 consensus inliers instead of ~6),
        # so the consensus / RANSAC / refinement stages see a meaningful problem.  Only valid for the default seed.
        if trained_pose and seed == 123 and os.path.exists(POSE_TRAINED):
            z = np.load(POSE_TRAINED)
            sd = model.state_dict()
            for k in z.files:
                sd[k].copy_(torch.from_numpy(z[k]))
    model.eval()
    for m in model.modules():
        if hasattr(m, "invalidate"):
            m.invalidate()
    return model
