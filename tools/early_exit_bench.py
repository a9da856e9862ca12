#!/usr/bin/env python
"""Pairs/s of the early-exit mode on the throughput path (forward_async, CUDA graphs, six pairs in flight).

    python tools/early_exit_bench.py [--pairs 48] [--seconds 5] [--runs 3] [--json OUT]

Workload: 48 distinct C2 pairs (synth.make_pair), the fitted CostNet (init_synthetic_weights(..., trained_pose=True)),
explicit permutations drawn once per pair, early_exit_min_inliers = 5 (the seeded descriptor gives ~27 first-scale inliers;
the reference's 50 needs a real checkpoint).  Arms, alternated run by run in one process:
  a  early exit off                                        (forward_async, graphs, 6 in flight)
  b  early exit on, threshold 5 (pairs exit)               (forward_async, graphs, 6 in flight)
  c  early exit on, unreachable threshold (never exits)    (forward_async, graphs, 6 in flight)
  d  eager forward() with early exit (host decision)       (serial)
Every timed region is whole passes over the pairs lasting at least --seconds after a warm-up pass.  The script checks on
the timed pairs: (c) == (a) bit for bit; (b) == (a) on the pairs that did not exit; (b) == the one-scale early-exit-off flow
on the pairs that exited; and (d) takes the same decision as (b).  It also times, with CUDA events, the consensus + RANSAC
that the device flow repeats after an exit (kept so one captured graph serves both outcomes).  Prints one JSON line.
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
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable ({e})"
    return dict(name=name, power_limit_and_max_sm_clock=q)


def make_model(sd, exit_on, min_inliers=5, S=3):
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    cfg = workload_cfg("C2")
    cfg.match.enable_early_exit = exit_on
    cfg.match.early_exit_min_inliers = min_inliers
    if S != cfg.patch.num_scales:
        cfg.patch.num_scales = S
        cfg.patch.search_radius_thresholds = list(cfg.patch.search_radius_thresholds)[:S]
    m = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    m.load_state_dict(sd)
    return m.cuda().eval()


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
    return np.array_equal(np.asarray(a[0]), np.asarray(b[0])) and tuple(a[2:]) == tuple(b[2:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=48)
    ap.add_argument("--seconds", type=float, default=5.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the result line to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("early_exit_bench.py needs a CUDA device")
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg

    torch.cuda.set_device(0)
    cfg = workload_cfg("C2")
    sd = {k: v.detach().clone() for k, v in init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).state_dict().items()}
    pairs = [make_pair("C2", s) for s in range(args.pairs)]
    rs = np.random.RandomState(2024)
    S = cfg.patch.num_scales
    perms = [[(rs.permutation(len(d["src_fds_pcd"])).astype(np.int32), rs.permutation(len(d["tgt_fds_pcd"])).astype(np.int32))
              for _ in range(S)] for d in pairs]

    models = dict(a=make_model(sd, False), b=make_model(sd, True, 5), c=make_model(sd, True, 10 ** 9), d=make_model(sd, True, 5))
    for k in "abc":
        models[k].enable_cuda_graphs(True, slots_per_shape=IN_FLIGHT)
    fns = dict(a=lambda: run_async(models["a"], pairs, perms), b=lambda: run_async(models["b"], pairs, perms),
               c=lambda: run_async(models["c"], pairs, perms), d=lambda: run_eager(models["d"], pairs, perms))
    rates, outs = {k: [] for k in fns}, {}
    with torch.no_grad():
        for k, f in fns.items():          # warm-up: captures every slot's graph, loads every module
            f()
        for _ in range(args.runs):
            for k, f in fns.items():
                r, o = timed(f, args.seconds)
                rates[k].append(r)
                outs[k] = o
        # ---- output equalities on the timed pairs ------------------------------------------------------------
        exited = [o[5] == 1 for o in outs["b"]]
        one_scale = make_model(sd, False, S=1).enable_cuda_graphs(True, slots_per_shape=IN_FLIGHT)
        ref1 = run_async(one_scale, [d for d, e in zip(pairs, exited) if e], [p[:1] for p, e in zip(perms, exited) if e])
        it1 = iter(ref1)
        checks = dict(
            c_equals_a=all(same(x, y) for x, y in zip(outs["c"], outs["a"])),
            c_never_exits=all(o[5] == S for o in outs["c"]),
            b_equals_a_where_not_exited=all(same(x, y) for x, y, e in zip(outs["b"], outs["a"], exited) if not e),
            b_equals_one_scale_flow_where_exited=all(same(x, next(it1)) for x, e in zip(outs["b"], exited) if e),
            d_same_decision_as_b=all(x[5] == y[5] for x, y in zip(outs["d"], outs["b"])),
            d_pose_identical_to_b=sum(same(x, y) for x, y in zip(outs["d"], outs["b"])),
        )
        # ---- what the repeated consensus + RANSAC costs an exiting pair (CUDA events, one stream) ------------------
        i0 = exited.index(True) if any(exited) else 0
        from bufferx_b200 import ops
        md = models["d"]
        md(pairs[i0], perms=perms[i0], ransac_seed=0, debug=True)
        dbg = md.last_debug
        K = cfg.patch.num_fps
        d_Mc = torch.tensor([int(dbg["offs"][1])], dtype=torch.int32, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        reps = 20
        for r in range(reps + 2):
            if r == 2:
                ev[0].record()
            inl, dI, _, _ = ops.consensus(dbg["ss"], dbg["tt"], dbg["R"], dbg["t"], d_Mc, S * K, cfg.patch.azi_n, cfg.match.inlier_th)
            md.pose_estimator.enqueue(dbg["ss"], dbg["tt"], inl, dI, S * K, None)
        ev[1].record()
        torch.cuda.synchronize()
        second_ms = ev[0].elapsed_time(ev[1]) / reps

    def stats(v):
        return dict(min=round(min(v), 2), median=round(float(np.median(v)), 2), max=round(max(v), 2), runs=[round(x, 2) for x in v])

    line = dict(
        metric="pairs/s, C2 (2x20000 pts, 1500 kpts, 3 scales), fitted CostNet, early_exit_min_inliers 5",
        card=card(), pairs=args.pairs, seconds_per_run=args.seconds,
        arms={"a_exit_off_async": stats(rates["a"]), "b_exit_on_async": stats(rates["b"]),
              "c_exit_never_async": stats(rates["c"]), "d_exit_on_eager_forward": stats(rates["d"])},
        exited_fraction=sum(exited) / len(exited),
        speedup_b_over_a=round(float(np.median(rates["b"]) / np.median(rates["a"])), 3),
        overhead_c_over_a=round(float(1.0 - np.median(rates["c"]) / np.median(rates["a"])), 4),
        speedup_b_over_d=round(float(np.median(rates["b"]) / np.median(rates["d"])), 3),
        repeated_consensus_ransac_ms=round(second_ms, 3),
        checks=checks,
    )
    print(json.dumps(line), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(line, f, indent=1)
    ok = all(v for k, v in checks.items() if k != "d_pose_identical_to_b")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
