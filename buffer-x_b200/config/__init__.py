"""Configuration surface of the registration hot path.

Mirrors the *semantics* of the reference's ``config`` package
(``/root/reference/config/__init__.py:18-56`` ``make_cfg``;
``indoor_config.py:4-80`` / ``outdoor_config.py:4-82`` base trees and the 14
per-dataset subclasses): the same dataset names, the same field names and
defaults, attribute *and* item access.  The reference writes one class per
dataset; here the whole surface is one table (two base profiles + a per-dataset
override list), which is all the hot path needs.

When this package is used as a drop-in inside the reference checkout the
reference's own ``config`` package is used instead (see INTEGRATION.md); this
module exists so that the H100 path, its tests and ``bench.py`` run without the
reference tree and without the ``easydict`` dependency.
"""
from pathlib import Path

try:  # real easydict if the environment has it (same semantics)
    from easydict import EasyDict as _ED  # type: ignore
except Exception:  # pragma: no cover - exercised in this image
    from ..easydict import EasyDict as _ED

__all__ = ["make_cfg", "DATASETS"]


def _base(indoor: bool) -> _ED:
    c = _ED()
    c.data = _ED(
        dataset="",
        root="",
        downsample=0.02 if indoor else 0.05,
        voxel_size_0=0.035 if indoor else 0.30,
        max_numPts=30000,
        manual_seed=123,
    )
    c.data.voxel_size_1 = c.data.voxel_size_0
    c.train = _ED(
        epoch=10 if indoor else 50,
        max_iter=50000,
        batch_size=1,
        num_workers=0,
        pos_num=512,
        augmentation_noise=0.001 if indoor else 0.01,
        pretrain_model="",
        all_stage=["Desc", "Pose"],
    )
    c.test = _ED(
        experiment_id="threedmatch",
        pose_refine=False,
        enable_timing=False,
        rte_thresh=0.3 if indoor else 2.0,
        rre_thresh=15.0 if indoor else 5.0,
    )
    c.optim = _ED(
        lr={"Desc": 0.001, "Pose": 0.001},
        lr_decay=0.50,
        weight_decay=1e-6,
        scheduler_interval={"Desc": 2, "Pose": 1} if indoor else {"Desc": 10, "Pose": 5},
    )
    c.patch = _ED(
        des_r=0.3 if indoor else 3.0,
        num_points_per_patch=512,
        num_fps=1500,
        rad_n=3,
        azi_n=20,
        ele_n=7,
        delta=0.8,
        voxel_sample=10,
        num_scales=3,
        is_aligned_to_global_z=not indoor,
        search_radius_thresholds=[5, 2, 0.5],
        num_points_radius_estimate=2000,
    )
    c.match = _ED(
        pose_estimator="ransac",
        dist_th=0.10 if indoor else 0.30,
        inlier_th=1 / 3 if indoor else 2.0,
        similar_th=0.8 if indoor else 0.9,
        confidence=0.999 if indoor else 1.0,
        iter_n=50000,
        kiss_resolution=0.3,
        enable_early_exit=False,
        early_exit_min_inliers=50,
    )
    return c


# name -> (indoor?, root sub-path, [(dotted key, value), ...])
DATASETS = {
    "3DMatch": (True, ("ThreeDMatch",), [("data.dataset", "3DMatch"), ("data.benchmark", "3DMatch"),
                                         ("test.pose_refine", True)]),
    "3DLoMatch": (True, ("ThreeDMatch",), [("data.dataset", "3DMatch"), ("data.benchmark", "3DLoMatch"),
                                           ("test.pose_refine", True)]),
    "Scannetpp_iphone": (True, ("Scannetpp_iphone",), []),
    "Scannetpp_faro": (True, ("scannetpp", "scannet-plusplus"), []),
    "ModelNet40": (True, ("processed_modelnet40",), [("test.pose_refine", False), ("test.rte_thresh", 0.1)]),
    "TIERS": (False, ("tiers_indoor",), [("test.pdist", 2)]),
    "TIERS_hetero": (False, ("tiers_indoor",), [("data.src_sensor", "os0_128"), ("data.tgt_sensor", "os1_64"),
                                                ("test.overlap_voxel_size", 0.1), ("test.overlap_thresh", 0.3),
                                                ("test.pdist", 2)]),
    "KITTI": (False, ("kitti",), [("test.pdist", 10)]),
    "WOD": (False, ("WOD",), [("test.pdist", 10)]),
    "MIT": (False, ("kimera-multi",), [("test.pdist", 5)]),
    "KAIST": (False, ("helipr_kaist05",), [("test.pdist", 10)]),
    "KAIST_hetero": (False, ("helipr_kaist05",), [("data.src_sensor", "Avia"), ("data.tgt_sensor", "Ouster"),
                                                  ("test.pdist", 10)]),
    "ETH": (False, ("ETH",), [("match.dist_th", 0.20), ("match.inlier_th", 1.5), ("match.similar_th", 0.9),
                              ("match.confidence", 1.0), ("match.iter_n", 50000),
                              ("test.rte_thresh", 0.3), ("test.rre_thresh", 2.0)]),
    "Oxford": (False, ("newer-college",), [("test.pdist", 5)]),
}


def _set(cfg, dotted, value):
    node = cfg
    parts = dotted.split(".")
    for p in parts[:-1]:
        node = node[p]
    node[parts[-1]] = value


def make_cfg(dataset_name, root_dir=None):
    """Same contract as ``/root/reference/config/__init__.py:18-56``."""
    if root_dir is None:
        root_dir = Path("../datasets")
    elif not isinstance(root_dir, Path):
        root_dir = Path(root_dir)
    if dataset_name not in DATASETS:
        raise ValueError(f"Unknown dataset: {dataset_name}")
    indoor, sub, overrides = DATASETS[dataset_name]
    cfg = _base(indoor)
    cfg.data.dataset = dataset_name
    cfg.data.root = root_dir.joinpath(*sub)
    for k, v in overrides:
        _set(cfg, k, v)
    return cfg
