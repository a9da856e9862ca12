"""bufferx-b200: the BUFFER-X per-pair registration hot path, hand-written for H100 (sm_90a).

Package layout (only what the path needs):
    csrc/      CUDA kernels + the C-ABI shared library (include/bufferx_b200.h)
    ops.py     torch-tensor wrappers over the C-ABI (ctypes; no torch types cross the boundary)
    models/    host-side mirror of the reference's models/BUFFERX.py API (BufferX, MiniSpinNet, ...)
    config/    make_cfg mirror (reference config/ semantics)
    synth.py   seeded synthetic pairs shaped like the reference's datasets
    driver.py  one-process-per-GPU pair sharding + one all-gather of result records

The directory name contains a hyphen (fixed by the task), so the importable name is ``bufferx_b200``
(see the shim ``bufferx_b200.py`` at the repository root); both names map to the same module objects.
"""
import sys as _sys

_REAL, _ALIAS = __name__, "bufferx_b200"


def _alias():
    for name, mod in list(_sys.modules.items()):
        if name == _REAL or name.startswith(_REAL + "."):
            _sys.modules[_ALIAS + name[len(_REAL):]] = mod


if _REAL != _ALIAS:
    _alias()  # make ``import bufferx_b200`` resolve to this package while it is still initialising

from . import easydict, se3, config, synth  # noqa: E402,F401
from .config import make_cfg  # noqa: E402,F401
from . import ops  # noqa: E402,F401
_alias()
from . import models  # noqa: E402,F401
from .models import patchnet, patch_embedder, pose_estimator, BUFFERX  # noqa: E402,F401
from .models.BUFFERX import BufferX  # noqa: E402,F401
from . import driver, bootstrap, evaluation  # noqa: E402,F401
_alias()

__version__ = "0.2.0"
