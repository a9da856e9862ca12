"""The training-stage kernels (csrc/bx_train.cu) on the GPU against float64, on edge inputs and on the route the Desc /
Pose validation forward runs.

Every kernel is held, through ops.gt_matches, ops.so2_augment, ops.equi_match and ops.so2_gt, to the checks of
oracle/train_cases.py (bounds derived in the docstring of tests/test_train_fp64_cpu.py).  The production route records
each of those calls, ops.hypotheses and the CostNet input maps inside BufferX._train_forward, and checks each call on
its own recorded inputs, which separates the kernel from the descriptor stack's rounding; pred_ind is held to the a11
bound (oracle.soft_argmax_bound).  The reference's own device arithmetic -- get_matching_indices' transform as a cuBLAS
matmul, and cal_so2_gt in torch on CUDA tensors -- is held to the same checks on the same inputs, so it can differ from
the kernels only at decisions the float64 check calls undecided; the number of differences is printed.  The largest
ratios are printed with -s and recorded in DESIGN.md section 7."""
import numpy as np
import pytest
import torch

from oracle import train_cases as C
from oracle import train_stages as TS
from oracle.train_cases import merge, report

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def cu(a, dev):
    return torch.as_tensor(np.ascontiguousarray(a)).to(dev, torch.float32).contiguous()


def _gt_kernel(dev, src, tgt, T, v):
    from bufferx_b200 import ops
    pairs, cnt = ops.gt_matches(cu(np.asarray(src).reshape(-1, 3), dev), cu(np.asarray(tgt).reshape(-1, 3), dev), cu(T, dev), v)
    return pairs[:int(cnt.item())].cpu().numpy().astype(np.int64)


def _gt_reference_cuda(dev, src, tgt, T, v, chunk=2048):
    """get_matching_indices on CUDA tensors: transform = R @ p^T + t (cuBLAS), the nearest target by torch (first
    minimum), kept where the distance < voxel."""
    s, t, Tm = cu(src, dev).reshape(-1, 3), cu(tgt, dev).reshape(-1, 3), cu(T, dev)
    if len(s) == 0 or len(t) == 0:
        return np.zeros((0, 2), np.int64)
    q = (Tm[:3, :3] @ s.T + Tm[:3, 3:4]).T
    idx, dist = [], []
    for a in range(0, len(q), chunk):
        d = torch.sqrt(((q[a:a + chunk, None, :] - t[None]) ** 2).sum(-1))
        m, j = d.min(dim=1)
        idx.append(j)
        dist.append(m)
    idx, dist = torch.cat(idx), torch.cat(dist)
    i = torch.nonzero(dist < v).reshape(-1)
    return torch.stack([i, idx[i]], 1).cpu().numpy().astype(np.int64)


# ------------------------------------------------------------------------------------------------ ground-truth matches
@pytest.mark.parametrize("group", ["grid", "dup", "offsets", "voxel_edge", "C1", "C2"])
def test_gt_matches_vs_fp64(dev, group):
    """Every M at and next to the 2048-point target tile, every N next to the 128-thread block and the compaction's 1024,
    duplicated targets, 1e2-1e4 m offsets, sources at exactly the voxel, and the C1 / C2 second-level clouds (C2: every
    5th source row in float64).  The reference's transform on CUDA is held to the same check."""
    if group in ("C1", "C2"):
        cases = {group: C.training_pair(group)}
    else:
        cases = {k: v for k, v in C.gt_cases().items()
                 if (k.startswith("M") if group == "grid" else k.startswith("offset") if group == "offsets" else k == group)}
    acc, ref_acc, differ = {}, {}, 0
    for name, (src, tgt, T, v) in cases.items():
        rows = np.arange(0, len(src), 5) if name == "C2" else None
        got = _gt_kernel(dev, src, tgt, T, v)
        if name.startswith("M") or name == "dup":
            assert np.array_equal(got, TS.matching_indices(src, tgt, T, v)), f"{name}: not the fp32 oracle's matches"
        merge(acc, C.check_gt(src, tgt, T, v, got, rows=rows))
        ref = _gt_reference_cuda(dev, src, tgt, T, v)
        merge(ref_acc, C.check_gt(src, tgt, T, v, ref, rows=rows))
        differ += len(set(map(tuple, got)) ^ set(map(tuple, ref)))
        if name == "voxel_edge":
            keep = C.gt_voxel_edge_case()[4]
            assert np.array_equal(got[:, 0], np.flatnonzero(keep))
    report(f"gt_matches {group}", acc)
    report(f"gt_matches {group}, reference transform on CUDA ({differ} pairs differ from the kernel)", ref_acc)


# ------------------------------------------------------------------------------------------------ SO(2) augmentation
@pytest.mark.parametrize("K", C.AUG_K)
def test_so2_augment_vs_fp64(dev, K):
    from bufferx_b200 import ops
    acc = {}
    for P in C.AUG_P:
        delta, ra, ang = C.aug_case(K, P, seed=K + P)
        d, r = cu(delta, dev), cu(ra, dev)
        R = ops.so2_augment(d, r, cu(ang, dev))
        merge(acc, C.check_aug(delta, ra, ang, d.cpu().numpy(), r.cpu().numpy(), R.cpu().numpy()))
    report(f"so2_augment K={K}", acc)


# ------------------------------------------------------------------------------------------------ EquiMatch
def _equi(dev, d1, d2):
    from bufferx_b200 import ops
    return ops.equi_match(d1.to(dev).contiguous(), d2.to(dev).contiguous()).cpu().numpy()


def test_equi_match_shapes_vs_fp64(dev):
    """C in {1, 31, 32, 33, 64} (idle lanes, one and two channel rounds), K in {1, 5, 7}, L in {1, 2, 20, 32}, and C K L
    exactly at 48 KB of shared memory; unit, unnormalised and cancelling maps.  Shapes beyond 48 KB are refused on the
    host."""
    from bufferx_b200 import ops
    acc = {}
    shapes = [(c, k, l) for c in C.EQ_C for k in C.EQ_K for l in C.EQ_L] + [(32, 6, 32), (6144, 1, 1), (1, 6144, 1)]
    refused = 0
    for c, k, l in shapes:
        if c * k * l > C.EQ_LIMIT:
            with pytest.raises(ops.BufferXError, match="shared memory"):
                ops.equi_match(torch.zeros(1, c, k, l, device=dev), torch.zeros(1, c, k, l, device=dev))
            refused += 1
            continue
        for kind in ("unit", "raw", "cancel"):
            d1, d2 = C.equi_case(64, c, k, l, kind, seed=c + k + l)
            merge(acc, C.check_equi(d1, d2, _equi(dev, d1, d2), C.equi_terms_kernel(c, k, l)))
    for c, k, l in ((6145, 1, 1), (32, 6, 33), (1, 6145, 1)):
        with pytest.raises(ops.BufferXError):
            ops.equi_match(torch.zeros(1, c, k, l, device=dev), torch.zeros(1, c, k, l, device=dev))
    acc["refused"] = refused
    report("equi_match shapes", acc)


@pytest.mark.parametrize("B", [0, 1, 4500])
def test_equi_match_batch_vs_fp64(dev, B):
    acc = {}
    for kind in ("unit", "raw", "cancel"):
        d1, d2 = C.equi_case(B, 32, 7, 20, kind, seed=B)
        got = _equi(dev, d1, d2)
        assert got.shape == (B, 20)
        merge(acc, C.check_equi(d1, d2, got, C.equi_terms_kernel(32, 7, 20)))
    report(f"equi_match B={B}", acc)


# ------------------------------------------------------------------------------------------------ SO(2) label
def _label_kernel(dev, s, a, b, T, azi_n, integer, A):
    from bufferx_b200 import ops
    return ops.so2_gt(cu(s, dev), cu(a, dev), cu(b, dev), cu(T, dev), azi_n, integer,
                      aug_R=None if A is None else cu(A, dev)).cpu().numpy()


@pytest.mark.parametrize("kind", ["random", "aug", "axis", "align"])
def test_so2_gt_vs_fp64(dev, kind):
    """azi_n in {1, 4, 20, 36} and P in {0, 1, 129, 4000}; the reference's cal_so2_gt on CUDA held to the same check."""
    acc, ref_acc, differ = {}, {}, 0
    for azi_n in C.GT_AZI:
        for P in C.GT_P:
            s, a, b, T, A = C.label_case(kind, P, azi_n, seed=azi_n + P)
            for integer in (True, False):
                got = _label_kernel(dev, s, a, b, T, azi_n, integer, A)
                assert got.dtype == (np.int64 if integer else np.float32) and got.shape == (P,)
                merge(acc, C.check_label(s, a, b, T, azi_n, got, integer, aug_R=A))
                if P:
                    ref = TS.so2_gt(s, a, b, T, azi_n, integer, aug_R=A, device=dev)
                    merge(ref_acc, C.check_label(s, a, b, T, azi_n, ref, integer, aug_R=A))
                    differ += int((ref != got).sum())
    report(f"so2_gt {kind}", acc)
    report(f"so2_gt {kind}, reference on CUDA ({differ} labels differ from the kernel)", ref_acc)


# ------------------------------------------------------------------------------------------------ production route
@pytest.mark.parametrize("workload", ["C1", "C2"])
@pytest.mark.parametrize("stage", ["Desc", "Pose"])
def test_production_route_vs_fp64(dev, oracle, monkeypatch, workload, stage):
    """BufferX._train_forward (eval mode, the reference's draws from NumPy's global RNG): every ops.gt_matches,
    ops.so2_augment, ops.equi_match, ops.so2_gt and ops.hypotheses call recorded -- so2_augment works in place, so its
    inputs are cloned before the call -- and held to float64 on its own inputs.  gt_label: decided labels equal
    float64's; gt_ind within its bound; equi_score within gamma_n; pred_ind within the a11 bound of the soft arg-max of
    oracle.costnet_fp64 on the recorded maps (rows 1..ele_n-2).  The reference's formulas on CUDA on the same inputs are
    held to the same checks."""
    import bufferx_b200 as bx
    from bufferx_b200 import ops
    from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg(workload)
    cfg.stage = stage
    data = add_training_clouds(make_pair(workload, 0), cfg)
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).to(dev).eval()
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    names = ("gt_matches", "so2_augment", "equi_match", "so2_gt", "hypotheses")
    rec = {k: [] for k in names + ("logits",)}
    orig = {k: getattr(ops, k) for k in names}
    clone = lambda x: x.clone() if isinstance(x, torch.Tensor) else x

    def wrap(name):
        def f(*a, **kw):
            inp, kin = [clone(x) for x in a], {k: clone(v) for k, v in kw.items()}
            r = orig[name](*a, **kw)
            after = [clone(x) for x in a]                  # in-place results (so2_augment's rows, hypotheses' ind_out)
            rec[name].append((inp, kin, clone(r) if not isinstance(r, tuple) else tuple(clone(x) for x in r), after))
            return r
        return f

    for k in names:
        monkeypatch.setattr(ops, k, wrap(k))
    logits = model.Pose.logits

    def rec_logits(es, et, *a):
        rec["logits"].append((es.clone(), et.clone()))
        return logits(es, et, *a)

    monkeypatch.setattr(model.Pose, "logits", rec_logits)
    np.random.seed(11)
    with torch.no_grad():
        out = model(data)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert out is not None
    acc, ref_acc, differ = {}, {}, 0
    # ground-truth matches (the last call: a TF32 recompute repeats the pair)
    (src, tgt, T, v), _, (pairs, cnt), _ = rec["gt_matches"][-1]
    src, tgt, Tn = src.cpu().numpy(), tgt.cpu().numpy(), T.cpu().numpy()
    got = pairs[:int(cnt.item())].cpu().numpy().astype(np.int64)
    rows = np.arange(0, len(src), 5) if workload == "C2" else None
    merge(acc, {"gt_" + k: x for k, x in C.check_gt(src, tgt, Tn, v, got, rows=rows).items()})
    ref = _gt_reference_cuda(dev, src, tgt, Tn, v)
    merge(ref_acc, {"gt_" + k: x for k, x in C.check_gt(src, tgt, Tn, v, ref, rows=rows).items()})
    differ += len(set(map(tuple, got)) ^ set(map(tuple, ref)))
    azi_n = cfg.patch.azi_n
    (s_ra, s_R, t_R, Tl, az, integer), kin, lab, _ = rec["so2_gt"][-1]
    A = kin.get("aug_R")
    args = [x.cpu().numpy() for x in (s_ra, s_R, t_R, Tl)]
    A = None if A is None else A.cpu().numpy()
    lab = lab.cpu().numpy()
    assert integer == (stage == "Desc")
    merge(acc, C.check_label(*args, azi_n, lab, integer, aug_R=A))
    rl = TS.so2_gt(*args, azi_n, integer, aug_R=A, device=dev)
    merge(ref_acc, C.check_label(*args, azi_n, rl, integer, aug_R=A))
    differ += int((rl != lab).sum())
    if stage == "Desc":
        assert torch.equal(out["gt_label"].cpu(), torch.from_numpy(lab))
        (d1, d2), _, score, _ = rec["equi_match"][-1]
        B, Cc, K, L = d1.shape
        merge(acc, C.check_equi(d1.cpu(), d2.cpu(), score.cpu().numpy(), C.equi_terms_kernel(Cc, K, L)))
        assert torch.equal(out["equi_score"].cpu(), score.cpu())
    else:
        inp, _, aug_R, after = rec["so2_augment"][-1]
        merge(acc, C.check_aug(inp[0].cpu().numpy(), inp[1].cpu().numpy(), inp[2].cpu().numpy(), after[0].cpu().numpy(),
                               after[1].cpu().numpy(), aug_R.cpu().numpy()))
        assert np.array_equal(aug_R.cpu().numpy(), A), "so2_gt did not get the applied augmentation"
        es, et = rec["logits"][-1]
        e = cfg.patch.ele_n
        d1, d2 = es[:, :, 1:e - 1].cpu().float(), et[:, :, 1:e - 1].cpu().float()
        l64 = oracle.costnet_fp64(d1, d2, sd)
        with torch.no_grad():
            l32, _ = oracle._cost_net(d1, d2, sd, azi_n, "Pose.conv.")
        ind64, bound, _, _ = oracle.soft_argmax_bound(l64, l32)
        pred = rec["hypotheses"][-1][3][12].cpu()
        assert torch.equal(pred, out["pred_ind"].cpu())
        dind = (pred.double() - ind64).abs()
        assert (dind <= bound).all(), f"pred_ind {float(dind.max()):.3g} from float64, {float((dind / bound).max()):.3g} of the a11 bound"
        acc["pred_ind"] = float((dind / bound).max())
        acc["pred_ind_err"] = float(dind.max())
    report(f"production route {workload} {stage}", acc)
    report(f"production route {workload} {stage}, reference on CUDA ({differ} differ from the kernels)", ref_acc)
