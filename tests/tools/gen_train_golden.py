"""Regenerate tests/golden/train_stages.npz: the reference's own training-stage forward on the synthetic golden cases.

    python tests/tools/gen_train_golden.py /path/to/reference/checkout

Runs the unmodified reference ``BufferX.forward`` with ``cfg.stage = "Desc"`` and ``"Pose"`` in eval mode on CPU, with
the third-party stubs of oracle/ref_check.py, on every case of ``oracle.train_stages.GOLDEN_CASES`` after
``np.random.seed(seed)``, and stores what it returned: the full ground-truth match list, the key-points, descriptors,
EquiMatch scores and integer labels (Desc), the soft arg-max and float labels (Pose), the LRF z axes the reference
used (so the oracle can be replayed with them) and the next value of NumPy's global RNG (which pins the draw order).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_check  # noqa: E402
from oracle import train_stages as TS  # noqa: E402


def run_reference(ref_root, name, stage):
    ref_check.install_stubs(0)
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    for m in [k for k in sys.modules if k in ("models", "utils") or k.startswith(("models.", "utils."))]:
        del sys.modules[m]
    import models.BUFFERX as RB
    import utils.common as RC

    cfg, sd, data, seed = TS.golden_case(name, stage)
    ref = RB.BufferX(cfg)
    ref.load_state_dict(sd, strict=True)
    ref.eval()
    tdata = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in data.items()}
    cap = dict(z=[], match=[])
    orig_rods = RC.RodsRotatFormula
    RC.RodsRotatFormula = lambda a, b: (cap["z"].append(a.detach().clone().numpy()), orig_rods(a, b))[1]
    orig_gm = ref.get_matching_indices
    ref.get_matching_indices = lambda *a: (lambda r: (cap["match"].append(r.clone()), r)[1])(orig_gm(*a))
    np.random.seed(seed)
    try:
        with torch.no_grad():
            out = ref(tdata)
    finally:
        RC.RodsRotatFormula = orig_rods
    rec = {"rng_next": np.array([np.random.random()]), "match_all": cap["match"][0].numpy().astype(np.int64)}
    if cap["z"]:
        rec["src_z"], rec["tgt_z"] = cap["z"][0], cap["z"][1]
    for k, v in out.items():
        rec[k] = v.numpy()
    return rec


def main(ref_root):
    gold = {}
    for name in TS.GOLDEN_CASES:
        for stage in ("Desc", "Pose"):
            rec = run_reference(ref_root, name, stage)
            for k, v in rec.items():
                gold[f"{name}_{stage}_{k}"] = v
            print(name, stage, {k: getattr(v, "shape", v) for k, v in rec.items()})
    path = os.path.join(ROOT, "tests", "golden", "train_stages.npz")
    np.savez_compressed(path, **gold)
    print("wrote", path)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "../reference")
