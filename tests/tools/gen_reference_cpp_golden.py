"""Fixture generator (needs the reference checkout): builds the reference's own cpp_wrappers C++ into oracle/_ref/libbxref.so
(oracle/ref_build/build_ref.py) and writes what it returns for the seeded inputs of the a17 / a18 tests in
tests/test_oracle_cpu.py (batch radius neighbours, grid subsampling) into tests/golden/reference_cpp.npz.
    python tests/tools/gen_reference_cpp_golden.py"""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle  # noqa: E402

# the inputs of test_radius_neighbors_restatement_equals_reference_cpp / test_grid_subsample_restatement_equals_reference_cpp
NEIGHBOR_CASES = [(0.35, [300, 200], [3500, 2500]), (0.2, [500], [6000]), (0.6, [100, 150, 250], [3000, 3000])]
SUBSAMPLE_DL = (0.2, 0.05, 1.7)


def main():
    spec = importlib.util.spec_from_file_location("_bx_ref_build", os.path.join(ROOT, "oracle", "ref_build", "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build()
    out = {}
    for radius, qb, sb in NEIGHBOR_CASES:
        rng = np.random.default_rng(int(radius * 100))
        s = rng.uniform(-2, 2, (sum(sb), 3)).astype(np.float32)
        q = (s[rng.choice(len(s), sum(qb), replace=False)] + rng.normal(scale=0.01, size=(sum(qb), 3))).astype(np.float32)
        out[f"neighbors_{radius}"] = oracle.ref_radius_neighbors(q, s, qb, sb, radius)
    rng = np.random.default_rng(3)
    pts = (rng.uniform(-3, 3, (20000, 3)) * [1, 1, 0.4]).astype(np.float32)
    for dl in SUBSAMPLE_DL:
        out[f"subsample_{dl}"] = oracle.ref_grid_subsampling(pts, dl)
    path = os.path.join(ROOT, "tests", "golden", "reference_cpp.npz")
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
