"""Mutual matching, consensus, RANSAC and refinement (a10, a13-a15) on the GPU against float64, on edge inputs and on the
route production runs.

Each kernel is held bit for bit to the C oracle where it has that contract and to the float64 checks of
oracle/pose_cases.py (bounds derived in the docstring of tests/test_pose_fp64_cpu.py).  Outputs are written into
NaN- or sentinel-filled buffers with device counts below capacity, so rows past a count must stay untouched.  RANSAC
runs cross the 8192-iteration chunk; a run with no marginal decision must give (num_inliers, best_itr, iters_run)
exactly, and at least 90 % of the runs must be decided.  The production route (C2 seed 0, fitted CostNet, batched
tail) records every ops.mutual_nn / consensus / ransac / refine call and holds each one to float64.  The largest ratio
of each check, the decided fraction and the degenerate winners are printed with -s and recorded in DESIGN.md
section 7."""
import numpy as np
import pytest
import torch

from oracle import pose_cases as P
from oracle.pose_cases import merge, report

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def cu(a, dev, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t if dtype is None else t.to(dtype)


def i32(v, dev):
    return torch.tensor([v], dtype=torch.int32, device=dev)


KAB = [1, 63, 64, 65, 1023, 1024, 1025, 1500]


@pytest.mark.parametrize("Ka", KAB)
def test_mutual_nn_vs_fp64(dev, oracle, Ka):
    """Every Kb of the tile / loop edges, then the device-count form: the rows beyond the counts hold NaN and the
    result must equal the exact-size call."""
    from bufferx_b200 import ops
    acc = {}
    for Kb in KAB:
        a, b = P.desc_set(Ka, Kb, seed=Ka + Kb)
        s, t, dM, snn, tnn = ops.mutual_nn(cu(a, dev), cu(b, dev), want_nn=True)
        M = int(dM.item())
        snn, tnn = snn[:Ka].cpu().numpy(), tnn[:Kb].cpu().numpy()
        es, et, esnn, etnn = oracle.mutual_nn(a, b)
        assert (snn == esnn).all() and (tnn == etnn).all() and M == len(es)
        merge(acc, P.check_mutual_nn(a, b, snn, tnn, s[:M].cpu().numpy(), t[:M].cpu().numpy()))
        ca, cb = max(Ka - 7, 0), max(Kb - 5, 0)
        ap = np.concatenate([a, np.full((3, 32), np.nan, np.float32)])
        bp = np.concatenate([b, np.full((2, 32), np.nan, np.float32)])
        ap[ca:Ka] = np.nan
        bp[cb:Kb] = np.nan
        so = torch.full((Ka + 3,), -7, dtype=torch.int32, device=dev)
        to = torch.full((Ka + 3,), -7, dtype=torch.int32, device=dev)
        dMo = torch.zeros(1, dtype=torch.int32, device=dev)
        ops.mutual_nn(cu(ap, dev), cu(bp, dev), out=(so, to, dMo), d_Ka=i32(ca, dev), d_Kb=i32(cb, dev))
        es, et, _, _ = oracle.mutual_nn(a[:ca], b[:cb])
        Mo = int(dMo.item())
        assert Mo == len(es) and (so[:Mo].cpu().numpy() == es).all() and (to[:Mo].cpu().numpy() == et).all()
        assert (so[Mo:] == -7).all() and (to[Mo:] == -7).all(), "rows past the match count written"
    report(f"mutual_nn Ka={Ka}", acc)


CONSENSUS = [(n, th) for n in (1, 3, 255, 1025) for th in P.INLIER_TH] + [(4500, 1 / 3)]


@pytest.mark.parametrize("n,inlier_th", CONSENSUS)
def test_consensus_vs_fp64(dev, oracle, n, inlier_th):
    """Device count n below a capacity of n + 13 whose spare rows hold NaN; counts and the inlier list past n untouched."""
    from bufferx_b200 import ops
    acc = {}
    for k, kind in enumerate(P.KINDS):
        ss, tt, T = P.corr_set(kind, n, seed=n + k, offset=P.OFFSETS[k % 4] if kind == "generic" else 0.0)
        rng = np.random.default_rng(k)
        R = np.tile(T[:3, :3].astype(np.float32), (n, 1, 1))
        t = (T[:3, 3] + rng.normal(scale=0.05, size=(n, 3))).astype(np.float32)
        if n >= 3:
            ss[0] = 0.0
            t[1] = tt[0]
            R[2::3] = np.eye(3, dtype=np.float32)
        cap = n + 13
        pad = lambda x: np.concatenate([x, np.full((cap - n,) + x.shape[1:], np.nan, np.float32)])
        ind, dI, dbest, counts = ops.consensus(cu(pad(ss), dev), cu(pad(tt), dev), cu(pad(R), dev), cu(pad(t), dev),
                                               i32(n, dev), cap, 20, inlier_th)
        I, best = int(dI.item()), int(dbest.item())
        eind, ebest, ecounts = oracle.consensus(ss, tt, R, t, 20, inlier_th)
        c = counts.cpu().numpy()
        assert (c[:n] == ecounts).all() and best == ebest and I == len(eind) and (ind[:I].cpu().numpy() == eind).all()
        merge(acc, P.check_consensus(ss, tt, R, t, 20, inlier_th, c[:n], best, ind[:I].cpu().numpy()))
    report(f"consensus n={n} inlier_th={inlier_th:.3g}", acc)


KINDS3 = ("generic", "planar", "rot180")
# (n, kind, max_iter, confidence, inlier fraction): the runs across the 8192-iteration chunk use 10 % inliers, so that
# confidence 0.999 stops past the first chunk and duplicate draws of two inliers (a free rotation) stay rare
RUNS = [(n, "generic", 100, 0.999, 0.4) for n in (0, 1, 2, 3, 4)] + \
    [(n, kind, mi, 0.999, 0.4) for n in (255, 256, 257) for kind in KINDS3 for mi in (100, 50000)] + \
    [(n, KINDS3[j % 3], mi, conf, 0.1) for j, n in enumerate((1023, 1024, 4500))
     for mi, conf in ((8191, 1.0), (8192, 0.999), (8193, 1.0), (50000, 0.999))]


def _ransac(dev, ss, tt, ind, dist_th, similar_th, conf, max_iter, seed):
    from bufferx_b200 import ops
    n = len(ind)
    pad = np.full(n + 9, -1, np.int32)
    pad[:n] = ind
    res = ops.ransac(cu(ss, dev), cu(tt, dev), cu(pad, dev), i32(n, dev), len(pad), dist_th, similar_th, conf, max_iter, seed)
    return ops.decode_ransac_result(res.cpu())


def test_ransac_vs_fp64(dev, oracle):
    """max_iter across the 8192 chunk, confidence 0.999 and 1.0, every correspondence count; bit for bit to the oracle
    and to float64 where decided."""
    acc = {}
    for r, (n, kind, mi, conf, frac) in enumerate(RUNS):
        dt, st = P.DIST_TH[r % 3], P.SIMILAR_TH[r % 2]
        ss, tt, _ = P.corr_set(kind, n + 20, seed=n + r, inlier_frac=frac)
        ind = np.arange(n, dtype=np.int32)
        T, ninl, bitr, iters = _ransac(dev, ss, tt, ind, dt, st, conf, mi, 1000 + r)
        e = oracle.ransac(ss, tt, ind, dt, st, conf, mi, 1000 + r, want_recs=True)
        assert (ninl, bitr, iters) == (e["num_inliers"], e["best_itr"], e["iters"]) and np.abs(T - e["T"]).max() < 1e-12
        merge(acc, P.check_ransac(ss, tt, ind, dt, st, conf, mi, 1000 + r, T, ninl, bitr, iters, recs=e["recs"]))
    ss, tt, _ = P.corr_set("generic", 500, seed=9, inlier_frac=1.0, noise=0.0)       # all inliers: est_k -> 0
    ind = np.arange(500, dtype=np.int32)
    T, ninl, bitr, iters = _ransac(dev, ss, tt, ind, 0.10, 0.8, 0.999, 50000, 3)
    out = P.check_ransac(ss, tt, ind, 0.10, 0.8, 0.999, 50000, 3, T, ninl, bitr, iters)
    assert out["decided"] and ninl == 500 and iters == bitr + 1
    merge(acc, out)
    frac = acc["decided"] / acc["runs"]
    report(f"ransac {acc['runs']} runs, decided fraction {frac:.3f}", acc)
    assert frac >= 0.9, f"only {frac:.1%} of the runs were decided"


@pytest.mark.parametrize("kind", ["generic", "planar", "identity", "rot180"])
def test_refine_vs_fp64(dev, oracle, kind):
    from bufferx_b200 import ops
    acc = {}
    for offset in (0.0, 80.0):
        for dt in P.DIST_TH:
            ss, tt, T = P.corr_set(kind, 900, seed=4, spread=3.0, offset=offset, inlier_frac=0.6, noise=0.01)
            T0 = T.copy()
            T0[:3, 3] += 0.3 * dt
            Tout = torch.full((20,), float("nan"), device=dev)
            To, rounds = ops.refine(cu(ss, dev), cu(tt, dev), i32(900, dev), 900, cu(T0.reshape(16), dev, torch.float64), dt,
                                    T_out=Tout[:16])
            assert torch.isnan(Tout[16:]).all()
            eT, er = oracle.refine(ss, tt, T0.astype(np.float32), dt)
            To = To.cpu().numpy().reshape(4, 4)
            assert int(rounds.item()) == er and np.abs(To - eT).max() < 1e-5
            merge(acc, P.check_refine(ss, tt, T0, dt, To, int(rounds.item())))
    report(f"refine {kind}", acc)


@pytest.mark.parametrize("offset", [0.0, 80.0, 1e3, 1e4])
def test_refine_exact_grid_far_from_origin(dev, oracle, offset):
    """Every distance exactly 0 (weights 1 on both sides): only the fit's rounding is left, so an offset^2
    cancellation in the kernel's cross-covariance fails at 1e4 m."""
    from bufferx_b200 import ops
    ss, tt, T = P.exact_grid_set(900, offset, seed=1)
    To, rounds = ops.refine(cu(ss, dev), cu(tt, dev), i32(900, dev), 900, cu(T.reshape(16), dev, torch.float64), 0.10)
    out = P.check_refine(ss, tt, T, 0.10, To.cpu().numpy(), int(rounds.item()))
    assert out["refine_decided"] and "R" in out
    report(f"refine exact grid offset {offset:g}", out)


def test_production_route_c2(dev, oracle, monkeypatch):
    """BufferX.forward on the C2 seed-0 pair (fitted CostNet, no debug: the batched tail): every ops.mutual_nn,
    ops.consensus, ops.ransac and ops.refine call recorded (inputs and outputs copied on the stream) and held to float64.
    The route makes S mutual_nn calls, one consensus, one RANSAC and one refinement."""
    import bufferx_b200 as bx
    from bufferx_b200 import ops
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C2")
    S = cfg.patch.num_scales
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).to(dev).eval()
    data = make_pair("C2", 0)
    perms = oracle.draw_perms(cfg, data["src_fds_pcd"].shape[0], data["tgt_fds_pcd"].shape[0], 0)
    rec = {"mutual_nn": [], "consensus": [], "ransac": [], "refine": []}
    orig = {k: getattr(ops, k) for k in rec}

    def wrap(name):
        def f(*a, **kw):
            inp = [x.clone() if isinstance(x, torch.Tensor) else x for x in a]
            kin = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in kw.items() if k != "out"}
            r = orig[name](*a, **kw)
            outs = r if isinstance(r, tuple) else (r,)
            if name == "mutual_nn" and "out" in kw:
                outs = kw["out"]
            rec[name].append((inp, kin, [o.clone() if isinstance(o, torch.Tensor) else o for o in outs]))
            return r
        return f

    for k in rec:
        monkeypatch.setattr(ops, k, wrap(k))
    with torch.no_grad():
        model(data, perms=perms, ransac_seed=0)
    torch.cuda.synchronize()
    for k in rec:
        monkeypatch.setattr(ops, k, orig[k])
    assert [len(rec[k]) for k in rec] == [S, 1, 1, 1], {k: len(v) for k, v in rec.items()}
    acc = {}
    for inp, kin, outs in rec["mutual_nn"]:
        a, b = inp[0].cpu().numpy(), inp[1].cpu().numpy()
        s_l, t_l, cnt = (o.cpu().numpy() for o in outs[:3])
        M = int(cnt.reshape(-1)[0])
        es, et, esnn, etnn = oracle.mutual_nn(a, b)
        assert M == len(es) and (s_l[:M] == es).all() and (t_l[:M] == et).all()
        merge(acc, P.check_mutual_nn(a, b, esnn, etnn, s_l[:M], t_l[:M]))
        acc["zero_rows"] = acc.get("zero_rows", 0) + int((np.abs(a).sum(1) == 0).sum() + (np.abs(b).sum(1) == 0).sum())
    (ss, tt, R, t, dMc, maxMc, azi_n, inlier_th), _, (ind, dI, dbest, counts) = rec["consensus"][0]
    Mc = int(dMc.item())
    ss_, tt_ = ss[:Mc].cpu().numpy(), tt[:Mc].cpu().numpy()
    I = int(dI.item())
    merge(acc, P.check_consensus(ss_, tt_, R[:Mc].cpu().numpy(), t[:Mc].cpu().numpy(), azi_n, inlier_th,
                                 counts[:Mc].cpu().numpy(), int(dbest.item()), ind[:I].cpu().numpy()))
    inp, kin, outs = rec["ransac"][0]
    _, _, rind, rdI, _, dist_th, similar_th, conf, max_iter, seed = inp[:10]
    T, ninl, bitr, iters = ops.decode_ransac_result(outs[0].cpu())
    I = int(rdI.item())
    merge(acc, P.check_ransac(ss_, tt_, rind[:I].cpu().numpy(), dist_th, similar_th, conf, max_iter, seed, T, ninl, bitr, iters))
    inp, kin, outs = rec["refine"][0]
    n = int(inp[2].item())
    T_in = inp[4].cpu().numpy().reshape(4, 4)
    merge(acc, P.check_refine(ss_[:n], tt_[:n], T_in, inp[5], outs[0].cpu().numpy(), int(outs[1].item())))
    report(f"production route C2 seed 0: {S} matchings, consensus over {Mc}, RANSAC over {I}", acc)
