#!/usr/bin/env python
"""Pairs/s of a stream of pairs of every size on the throughput path, with and without size classes.

    python tools/size_class_bench.py [--pairs 48] [--seconds 5] [--runs 3] [--json OUT]

Workload: 48 C2 pairs (synth.make_pair) whose cloud sizes are all distinct, drawn with a seeded RNG, the pairs alternating
between 9000..16384 points per cloud and 16385..24000 points per cloud (the (16384, 16384) and (24576, 24576) class keys),
explicit permutations drawn once per pair, early exit off.  Arms, alternated run by run in one process:
  a  eager forward()                                                          (serial)
  c  forward_async + graphs + size classes, 3 slots per class key            (6 in flight)
then, each phase after the previous one's models are released (every captured C2 graph holds a few GB of activations):
  b  forward_async + graphs, exact-shape slots (one slot per shape, 8 shapes) (6 in flight); an out-of-memory error is
     reported in the result line instead of a rate
  d  48 fixed-size C2 pairs (2 x 20000 points): exact-shape slots (d_exact) against class slots (d_class), 6 in flight,
     alternated -- what a capacity costs when every pair has the capacity's shape anyway
Every timed region is whole passes over the pairs lasting at least --seconds after a warm-up pass.  The script checks that
every arm returns the same result for every pair (pose bytes and counts) and prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

IN_FLIGHT = 6


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable ({e})"
    return dict(name=name, power_limit_sm_clock_max_sm_clock=q)


def run_async(model, pairs, perms):
    outs, handles = [], []
    for d, p in zip(pairs, perms):
        if len(handles) == IN_FLIGHT:
            outs.append(handles.pop(0).result())
        handles.append(model.forward_async(d, perms=p))
    outs += [h.result() for h in handles]
    return outs


def run_eager(model, pairs, perms):
    return [model(d, perms=p) for d, p in zip(pairs, perms)]


def timed(fn, seconds):
    """Whole passes until `seconds` have elapsed (each pass ends with every result on the host); returns (pairs/s, outputs)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n, outs = 0, None
    while True:
        outs = fn()
        n += len(outs)
        el = time.perf_counter() - t0
        if el >= seconds:
            return n / el, outs


def same(a, b):
    return np.asarray(a[0]).tobytes() == np.asarray(b[0]).tobytes() and tuple(a[2:]) == tuple(b[2:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=48)
    ap.add_argument("--seconds", type=float, default=5.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("size_class_bench.py needs a CUDA device")
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg

    torch.cuda.set_device(0)
    cfg = workload_cfg("C2")
    sd = {k: v.detach().clone() for k, v in init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).state_dict().items()}
    rng = np.random.default_rng(2025)
    lo = rng.choice(np.arange(9000, 16385), size=(args.pairs // 2, 2), replace=False)
    hi = rng.choice(np.arange(16385, 24001), size=(args.pairs - args.pairs // 2, 2), replace=False)
    sizes = [x for pair in zip(lo, hi) for x in pair]
    varied = [make_pair("C2", s, n_src=int(a), n_tgt=int(b)) for s, (a, b) in enumerate(sizes)]
    fixed = [make_pair("C2", s) for s in range(args.pairs)]
    rs = np.random.RandomState(2024)
    S = cfg.patch.num_scales

    def draw(pairs):
        return [[(rs.permutation(len(d["src_fds_pcd"])).astype(np.int32), rs.permutation(len(d["tgt_fds_pcd"])).astype(np.int32))
                 for _ in range(S)] for d in pairs]

    p_var, p_fix = draw(varied), draw(fixed)

    def model():
        m = init_synthetic_weights(bx.BufferX(workload_cfg("C2")), trained_pose=True)
        m.load_state_dict(sd)
        return m.cuda().eval()

    import gc
    models = {}
    setups = [dict(a=(dict(), varied, p_var, run_eager), c=(dict(slots_per_shape=IN_FLIGHT // 2, size_classes=True), varied, p_var, run_async)),
              dict(b=(dict(slots_per_shape=1), varied, p_var, run_async)),
              dict(d_exact=(dict(slots_per_shape=IN_FLIGHT), fixed, p_fix, run_async),
                   d_class=(dict(slots_per_shape=IN_FLIGHT, size_classes=True), fixed, p_fix, run_async))]
    rates, outs, errors, c_keys = {}, {}, {}, None
    with torch.no_grad():
        for arms in setups:
            if "c" in models:
                c_keys = sorted(str(k[:2]) for k in models["c"]._slots)
            models.clear()
            gc.collect()
            torch.cuda.empty_cache()
            for k, (opts, pairs, perms, run) in arms.items():
                models[k] = model()
                if opts:
                    models[k].enable_cuda_graphs(True, **opts)
            fns = {k: (lambda k=k, a=a: a[3](models[k], a[1], a[2])) for k, a in arms.items()}
            try:
                for k, f in fns.items():          # warm-up: captures the slots' graphs, loads every module
                    f()
                    rates[k] = []
                for _ in range(args.runs):
                    for k, f in fns.items():
                        r, o = timed(f, args.seconds)
                        rates[k].append(r)
                        outs[k] = o
            except torch.OutOfMemoryError as e:
                for k in arms:
                    errors[k] = str(e).split(".")[0]
                    rates.pop(k, None)
                    outs.pop(k, None)
    checks = dict(
        b_equals_a=all(same(x, y) for x, y in zip(outs["b"], outs["a"])) if "b" in outs else None,
        c_equals_a=all(same(x, y) for x, y in zip(outs["c"], outs["a"])),
        d_class_equals_d_exact=all(same(x, y) for x, y in zip(outs["d_class"], outs["d_exact"])),
        c_slot_keys=c_keys,
    )

    def stats(v):
        return dict(min=round(min(v), 2), median=round(float(np.median(v)), 2), max=round(max(v), 2), runs=[round(x, 2) for x in v])

    med = {k: float(np.median(v)) for k, v in rates.items() if v}
    line = dict(
        metric="pairs/s, C2 (1500 kpts, 3 scales, early exit off), fitted CostNet",
        card=card(), pairs=args.pairs, seconds_per_run=args.seconds, sizes="distinct, alternating 9000..16384 / 16385..24000 per cloud (seeded)",
        arms={"a_eager_forward": stats(rates["a"]), "b_async_graphs_exact_shapes": stats(rates["b"]) if rates.get("b") else errors.get("b"),
              "c_async_graphs_size_classes": stats(rates["c"]), "d_fixed_20k_exact_slots": stats(rates["d_exact"]),
              "d_fixed_20k_class_slots": stats(rates["d_class"])},
        speedup_c_over_a=round(med["c"] / med["a"], 3), speedup_c_over_b=round(med["c"] / med["b"], 3) if "b" in med else None,
        capacity_cost_d=round(1.0 - med["d_class"] / med["d_exact"], 4),
        checks=checks,
    )
    print(json.dumps(line), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(line, f, indent=1)
    ok = all(v for k, v in checks.items() if k not in ("c_slot_keys", "b_equals_a")) and checks["b_equals_a"] is not False
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
