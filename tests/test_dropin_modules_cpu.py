"""Module resolution of the drop-in packages under dropin/ (pointnet2_ops, knn_cuda, torch_batch_svd), CPU only.

With ``<repo>/dropin`` and the repository root on PYTHONPATH and a reference checkout as the working directory (how
``python test.py`` / ``python train.py`` run there), the three CUDA-extension names resolve to dropin/ while ``models``,
``utils``, ``dataset`` and ``config`` stay the reference's.  Where a reference checkout is present, its own
``utils.common``, ``dataset.kitti``, ``models.BUFFERX`` and ``models.patch_embedder`` import against the drop-ins;
packages outside the drop-ins' scope (open3d, matplotlib, kornia, nibabel) are replaced by empty stand-in modules where
they are not installed.  The checkout is ``$BUFFERX_REFERENCE``, by default the one ``oracle/ref_check.py`` pins the
oracle against; those tests skip without it.
"""
import json
import os
import subprocess
import sys
import textwrap

import pytest

from oracle.ref_check import REF
from test_dropin import _fake_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "dropin")
REFERENCE = os.environ.get("BUFFERX_REFERENCE", REF)


def _run(code, cwd):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([DROPIN, ROOT])
    out = subprocess.run([sys.executable, "-c", textwrap.dedent(code)], cwd=str(cwd), env=env, capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_dropin_names_resolve_to_dropin_and_reference_names_to_the_checkout(tmp_path):
    ref = _fake_reference(tmp_path)
    res = _run("""
        import importlib.util as u, json, os
        names = ["pointnet2_ops", "pointnet2_ops.pointnet2_utils", "knn_cuda", "torch_batch_svd", "utils.common", "utils.timer",
                 "dataset.dataloader", "models.BUFFERX", "models.patch_embedder", "config"]
        out = {}
        for n in names:
            s = u.find_spec(n)
            out[n] = None if s is None else os.path.realpath(s.origin)
        print(json.dumps(out))
    """, ref)
    for n in ("pointnet2_ops", "pointnet2_ops.pointnet2_utils", "knn_cuda", "torch_batch_svd"):
        assert res[n] is not None and res[n].startswith(os.path.realpath(DROPIN)), f"{n} must resolve to dropin/, got {res[n]}"
    for n in ("utils.common", "utils.timer", "dataset.dataloader", "models.BUFFERX", "models.patch_embedder", "config"):
        assert res[n] is not None and res[n].startswith(os.path.realpath(str(ref))), f"{n} must come from the reference checkout, got {res[n]}"


_STANDINS = textwrap.dedent("""
    import importlib.util, json, os, sys, types
    names = ("open3d", "matplotlib", "matplotlib.colors", "matplotlib.cm", "matplotlib.pyplot", "kornia", "kornia.geometry",
             "kornia.geometry.conversions", "nibabel", "nibabel.quaternions")
    missing = {n for n in names if "." not in n and importlib.util.find_spec(n) is None}
    for name in names:
        if name.split(".")[0] in missing:
            sys.modules[name] = types.ModuleType(name)
            if "." in name:
                parent, child = name.rsplit(".", 1)
                setattr(sys.modules[parent], child, sys.modules[name])
""")


@pytest.mark.skipif(not os.path.isdir(REFERENCE), reason="needs the reference checkout")
def test_reference_utils_and_dataset_import_against_the_dropins():
    res = _run(_STANDINS + textwrap.dedent("""
        import utils.common, dataset.kitti, pointnet2_ops.pointnet2_utils, torch_batch_svd
        print(json.dumps({"common": os.path.realpath(utils.common.__file__), "kitti": os.path.realpath(dataset.kitti.__file__),
                          "pnt2": utils.common.pnt2 is pointnet2_ops.pointnet2_utils, "svd": utils.common.svd is torch_batch_svd.svd,
                          "pnt2_file": os.path.realpath(utils.common.pnt2.__file__)}))
    """), REFERENCE)
    assert res["common"].startswith(REFERENCE) and res["kitti"].startswith(REFERENCE)
    assert res["pnt2"] and res["svd"] and res["pnt2_file"].startswith(os.path.realpath(DROPIN))


@pytest.mark.skipif(not os.path.isdir(REFERENCE), reason="needs the reference checkout")
def test_reference_models_import_against_the_dropins():
    res = _run(_STANDINS + textwrap.dedent("""
        import models.BUFFERX, models.patch_embedder, knn_cuda, pointnet2_ops.pointnet2_utils
        print(json.dumps({"buf": os.path.realpath(models.BUFFERX.__file__), "pe": os.path.realpath(models.patch_embedder.__file__),
                          "knn": models.BUFFERX.KNN is knn_cuda.KNN and models.patch_embedder.KNN is knn_cuda.KNN,
                          "pnt2": models.BUFFERX.pnt2 is pointnet2_ops.pointnet2_utils and models.patch_embedder.pnt2 is pointnet2_ops.pointnet2_utils,
                          "knn_file": os.path.realpath(knn_cuda.__file__)}))
    """), REFERENCE)
    assert res["buf"].startswith(REFERENCE) and res["pe"].startswith(REFERENCE)
    assert res["knn"] and res["pnt2"] and res["knn_file"].startswith(os.path.realpath(DROPIN))
