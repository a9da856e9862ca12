#!/usr/bin/env python
"""Pairs/s of a stream of large pairs of distinct sizes: eager forward against CUDA-graph slots, exact-shape and large-class.

    python tools/large_class_bench.py [--pairs 16] [--runs 3] [--json OUT]

Workload: --pairs synthetic pairs (synth.make_pair), alternating C3 and C5, every cloud size distinct and drawn with a
seeded RNG between 262145 and 976896 points, so every pair's larger cloud is radius sub-sampled.  Both clouds of a pair lie
in the same one of four size classes (262145-524288, -645120, -792576, -976896 points; --pairs / 4 pairs each), as the two
fragments of a dataset pair have similar sizes: arm c then holds four class graphs, and each captured graph of this
configuration holds several GB.  The C3 configuration (3 scales), early exit off, explicit permutations drawn once per
pair.  Each run is one serial pass of forward() over the
pairs with torch.manual_seed(i) before pair i.  Arms:
  a  eager forward()
  b  enable_cuda_graphs(True, size_classes=True): these pairs keep exact-shape slots (one capture per pair and pass: the
     8-key LRU holds fewer keys than there are pairs)
  c  enable_cuda_graphs(True, size_classes=True, large_classes=True): size-class slots, one per class key
a and c alternate run by run in one phase; b runs in a phase of its own after a and c are released, because the captured
graphs of large pairs hold several GB each (an out-of-memory error is reported in the result line instead of a rate).
Every arm makes one warm-up pass first.  Reported per arm: pairs/s (median and range of --runs runs), captures made in the
timed runs, and the peaks of torch.cuda.max_memory_allocated and max_memory_reserved over the arm's runs (in phase 1 each
includes the other model's resident memory).  A captured graph's intermediates are freed into its private pool, which stays
reserved: the reserved peak is the one that counts a slot's graphs.  The card's name and power limit are read in the same run.  Arms a and c must return identical
pose bytes and counts (exit status 1 otherwise); b draws its radius sub-sample on the device and is only reported.  Prints one JSON line.
"""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from icp_bench import card  # noqa: E402


def same(a, b):
    return np.asarray(a[0]).tobytes() == np.asarray(b[0]).tobytes() and tuple(a[2:]) == tuple(b[2:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("large_class_bench.py needs a CUDA device")
    import bufferx_b200 as bx
    from bufferx_b200.models import BUFFERX as B
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg

    torch.cuda.set_device(0)
    cfg = workload_cfg("C3")
    cfg.match.enable_early_exit = False
    rng = np.random.default_rng(2026)
    bounds = [262144, 524288, 645120, 792576, 976896]
    per = args.pairs // 4
    sizes = np.concatenate([rng.choice(np.arange(lo + 1, hi + 1), size=(per, 2), replace=False)
                            for lo, hi in zip(bounds[:-1], bounds[1:])])
    pairs = [make_pair("C3" if i % 2 == 0 else "C5", i, n_src=int(a), n_tgt=int(b)) for i, (a, b) in enumerate(sizes)]
    rs = np.random.RandomState(2024)
    perms = [[(rs.permutation(len(d["src_fds_pcd"])).astype(np.int32), rs.permutation(len(d["tgt_fds_pcd"])).astype(np.int32))
              for _ in range(cfg.patch.num_scales)] for d in pairs]
    sd = {k: v.detach().clone() for k, v in init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).state_dict().items()}

    captures = [0]
    init = B._PairSlot.__init__

    def counted_init(self, *a, **kw):
        init(self, *a, **kw)
        captures[0] += self.graph is not None

    B._PairSlot.__init__ = counted_init

    def model(**opts):
        m = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
        m.load_state_dict(sd)
        m = m.cuda().eval()
        if opts:
            m.enable_cuda_graphs(True, slots_per_shape=1, **opts)
        return m

    def run(m):
        outs = []
        for i, (d, p) in enumerate(zip(pairs, perms)):
            torch.manual_seed(i)
            outs.append(m(d, perms=p))
        return outs

    rates, caps, peak, peak_res, outs, errors, c_keys = {}, {}, {}, {}, {}, {}, None
    with torch.no_grad():
        for phase in (dict(a={}, c=dict(size_classes=True, large_classes=True)), dict(b=dict(size_classes=True))):
            models = {}
            gc.collect()
            torch.cuda.empty_cache()
            try:
                for k, opts in phase.items():
                    models[k] = model(**opts)
                    rates[k], caps[k], peak[k], peak_res[k] = [], 0, 0, 0
                for m in models.values():
                    run(m)                        # warm-up: loads every module, captures the slots' graphs
                for _ in range(args.runs):
                    for k, m in models.items():
                        torch.cuda.synchronize()
                        torch.cuda.reset_peak_memory_stats()
                        c0 = captures[0]
                        t0 = time.perf_counter()
                        outs[k] = run(m)          # every forward ends with its result on the host
                        el = time.perf_counter() - t0
                        rates[k].append(len(pairs) / el)
                        caps[k] += captures[0] - c0
                        peak[k] = max(peak[k], torch.cuda.max_memory_allocated())
                        peak_res[k] = max(peak_res[k], torch.cuda.max_memory_reserved())
            except torch.OutOfMemoryError as e:
                for k in phase:
                    errors[k] = str(e).split(".")[0]
                    rates.pop(k, None)
                    outs.pop(k, None)
            if "c" in models:
                c_keys = sorted(str(k[:2]) for k in models["c"]._slots)
            del models
    B._PairSlot.__init__ = init

    def stats(v):
        return dict(median=round(float(np.median(v)), 3), min=round(min(v), 3), max=round(max(v), 3), runs=[round(x, 3) for x in v])

    names = dict(a="a_eager_forward", b="b_graphs_exact_slots", c="c_graphs_large_classes")
    checks = dict(c_equals_a=all(same(x, y) for x, y in zip(outs["c"], outs["a"])) if "a" in outs and "c" in outs else False,
                  b_equals_a=all(same(x, y) for x, y in zip(outs["b"], outs["a"])) if "a" in outs and "b" in outs else None,
                  c_slot_keys=c_keys)
    med = {k: float(np.median(v)) for k, v in rates.items() if v}
    line = dict(
        metric="pairs/s, serial forward(), C3 configuration (3 scales), early exit off, synthetic weights",
        card=card(), pairs=args.pairs, sizes="distinct, 262145..976896 per cloud (seeded), both clouds of a pair in one of four classes, C3 / C5 alternating",
        arms={names[k]: (dict(pairs_per_s=stats(rates[k]), captures_in_timed_runs=caps[k], peak_allocated_gb=round(peak[k] / 2**30, 2),
                              peak_reserved_gb=round(peak_res[k] / 2**30, 2))
                         if k in med else errors.get(k)) for k in ("a", "b", "c")},
        speedup_c_over_a=round(med["c"] / med["a"], 3) if "a" in med and "c" in med else None,
        speedup_c_over_b=round(med["c"] / med["b"], 3) if "b" in med and "c" in med else None,
        checks=checks,
    )
    print(json.dumps(line), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(line, f, indent=1)
    sys.exit(0 if checks["c_equals_a"] else 1)


if __name__ == "__main__":
    main()
