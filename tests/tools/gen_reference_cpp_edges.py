"""Fixture generator (needs the reference checkout): builds the reference's own cpp_wrappers C++ into oracle/_ref/libbxref.so
(oracle/ref_build/build_ref.py) and writes what it returns on the a17 / a18 edge inputs of oracle/bootstrap_cases.py
(lattice ties, balls beyond 4096 entries, points on the strict radius boundary, empty balls, 1-8 query batches, offset
clouds, grid origins rounded above the minimum) into tests/golden/reference_cpp_edges.npz, with the inputs.
    python tests/tools/gen_reference_cpp_edges.py"""
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import bootstrap_cases as B  # noqa: E402
from oracle import oracle  # noqa: E402


def main():
    spec = importlib.util.spec_from_file_location("_bx_ref_build", os.path.join(ROOT, "oracle", "ref_build", "build_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build()
    out = {}
    for name, (q, s, qb, sb, r) in B.neighbor_cases().items():
        out[f"nb_{name}_q"], out[f"nb_{name}_s"] = q, s
        out[f"nb_{name}_ref"] = oracle.ref_radius_neighbors(q, s, qb, sb, r)
    for name, (p, dl) in B.subsample_cases().items():
        out[f"gs_{name}_p"] = p
        out[f"gs_{name}_ref"] = oracle.ref_grid_subsampling(p, dl)
    np.savez_compressed(B.EDGES_NPZ, **out)
    print(B.EDGES_NPZ, {k: v.shape for k, v in out.items() if k.endswith("_ref")})


if __name__ == "__main__":
    main()
