"""GPU: the training stages' validation forward (cfg.stage "Desc" / "Pose", eval mode) against the CPU oracle
(oracle/train_stages.py) -- each kernel of bx_train.cu on identical inputs, then the whole forward, then the model driven
the way the reference's Trainer.evaluate drives it."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def TS(oracle):
    from oracle import train_stages
    return train_stages


def cu(a, dev, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a)).to(dev, dtype).contiguous()


def _rel_rows(a, b):
    den = np.abs(b).max(1)
    return np.abs(a - b).max(1) / np.where(den > 0, den, 1)


def _training_pair(name, seed, stage, isolated=False):
    from bufferx_b200.synth import add_training_clouds, make_pair, workload_cfg
    cfg = workload_cfg(name)
    cfg.stage = stage
    return cfg, add_training_clouds(make_pair(name, seed), cfg, isolated=isolated)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("kind", ["c2", "dup", "empty_tgt"])
def test_gt_matches_bit_exact(dev, TS, kind):
    from bufferx_b200 import ops
    if kind == "c2":
        _, d = _training_pair("C2", 0, "Desc")
        src, tgt, T, v = d["src_sds_pcd"], d["tgt_sds_pcd"], d["relt_pose"], float(d["voxel_sizes"][0])
    else:
        rng = np.random.default_rng(7)
        tgt = rng.uniform(-1, 1, size=(3000, 3)).astype(np.float32)
        tgt[1500:] = tgt[:1500]                       # every target point twice: exact ties, the first copy must win
        src = np.concatenate([tgt[:1000] + rng.normal(scale=0.01, size=(1000, 3)), rng.uniform(-2, 2, size=(3000, 3))]).astype(np.float32)
        T, v = np.eye(4, dtype=np.float32), 0.05
        if kind == "empty_tgt":
            tgt = tgt[:0]
    pairs, cnt = ops.gt_matches(cu(src, dev), cu(tgt, dev), cu(T, dev), v)
    n = int(cnt.item())
    exp = TS.matching_indices(src, tgt, T, v)
    assert n == len(exp)
    assert np.array_equal(pairs[:n].cpu().numpy().astype(np.int64), exp)
    if kind == "dup":
        assert (exp[:, 1] < 1500).all() and n > 900


def test_so2_augment_matches_oracle(dev, TS):
    from bufferx_b200 import ops
    rng = np.random.RandomState(3)
    K, P = 700, 1024
    delta = rng.uniform(-1, 1, size=(K, P, 3)).astype(np.float32)
    ra = rng.normal(size=(K, 3)).astype(np.float32)
    ang = TS.draw_aug_angles(rng, K)
    ang[:3] = [0.0, 1e-4, 2e-3]                      # the Taylor branch of the kornia form (theta^2 <= 1e-6) and its edge
    d_delta, d_ra = cu(delta, dev), cu(ra, dev)
    R = ops.so2_augment(d_delta, d_ra, cu(ang, dev))
    e_delta, e_ra, e_R = TS.so2_augment(delta, ra, ang)
    assert np.abs(R.cpu().numpy() - e_R).max() < 1e-6
    assert np.abs(d_delta.cpu().numpy() - e_delta).max() < 1e-6
    assert np.abs(d_ra.cpu().numpy() - e_ra).max() < 1e-6


def test_equi_match_matches_oracle(dev, TS):
    from bufferx_b200 import ops
    rng = np.random.RandomState(4)
    B = 600
    d1 = torch.nn.functional.normalize(torch.from_numpy(rng.normal(size=(B, 32, 7, 20)).astype(np.float32)), dim=1)
    d2 = torch.nn.functional.normalize(d1 + 0.5 * torch.from_numpy(rng.normal(size=(B, 32, 7, 20)).astype(np.float32)), dim=1)
    d2 = torch.roll(d2, shifts=5, dims=-1)
    got = ops.equi_match(d1.to(dev).contiguous(), d2.to(dev).contiguous()).cpu().numpy()
    exp = TS.equi_match(d1.double(), d2.double()).numpy()
    assert _rel_rows(got, exp).max() < 1e-5
    srt = np.sort(exp, axis=1)
    clear = (srt[:, -1] - srt[:, -2]) > 1e-4 * np.abs(srt[:, -1])
    assert clear.mean() > 0.9 and (got.argmax(1) == exp.argmax(1))[clear].all()


def _random_rotations(rng, n):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], axis=1).reshape(n, 3, 3).astype(np.float32)


@pytest.mark.parametrize("aug", [False, True])
def test_so2_gt_matches_oracle(dev, TS, aug):
    from bufferx_b200 import ops
    rng = np.random.RandomState(5 + aug)
    P, azi_n = 4000, 20
    ra = rng.normal(size=(P, 3)).astype(np.float32)
    ra /= np.linalg.norm(ra, axis=1, keepdims=True)
    sR, tR = _random_rotations(rng, P), _random_rotations(rng, P)
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = _random_rotations(rng, 1)[0]
    T[:3, 3] = [0.3, -0.2, 0.1]
    A = TS.aug_rotations(TS.draw_aug_angles(rng, P)) if aug else None
    args = [cu(ra, dev), cu(sR, dev), cu(tR, dev), cu(T, dev)]
    dA = cu(A, dev) if aug else None
    li = ops.so2_gt(*args, azi_n, True, aug_R=dA).cpu().numpy()
    lf = ops.so2_gt(*args, azi_n, False, aug_R=dA).cpu().numpy()
    ei = TS.so2_gt(ra, sR, tR, T, azi_n, True, aug_R=A)
    ef = TS.so2_gt(ra, sR, tR, T, azi_n, False, aug_R=A)
    assert li.dtype == np.int64 and ((li >= 0) & (li < azi_n)).all()
    near_half = np.abs(ef - np.floor(ef) - 0.5) < 1e-4
    assert (li == ei)[~near_half].all()
    assert np.abs(lf - ef).max() < 1e-4


# ------------------------------------------------------------------------------------------------ whole forward
def _model(cfg, dev):
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).to(dev)
    sd = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    return model, sd


def _check_descriptors(oracle, sd, got, o_side, what):
    d, od = got.cpu().numpy(), o_side["desc"].numpy()
    rel = _rel_rows(d, od)
    assert rel.max() < 5e-4, f"{what}: descriptor rel err max {rel.max()}"
    if (rel < 1e-4).mean() < 0.999:
        # the existing bar of the inference path: an offender must be a descriptor where the fp32 oracle itself is as far
        # from the fp64 evaluation of the same network as the GPU
        sel = np.flatnonzero(rel >= 1e-4)
        t64 = oracle.desc_fp64(o_side["feat"][torch.from_numpy(sel)], sd).numpy()
        e_gpu, e_orc = _rel_rows(d[sel].astype(np.float64), t64), _rel_rows(od[sel].astype(np.float64), t64)
        assert (e_gpu <= 1.5 * e_orc + 2e-5).all(), f"{what}: GPU vs fp64 {e_gpu} against oracle vs fp64 {e_orc}"


def _compare_forward(oracle, TS, sd, cfg, stage, out, ref, what):
    aux = ref["aux"]
    if stage == "Desc":
        assert np.array_equal(out["src_kpt"].cpu().numpy(), ref["src_kpt"].numpy())
        assert np.array_equal(out["tgt_kpt"].cpu().numpy(), ref["tgt_kpt"].numpy())
        _check_descriptors(oracle, sd, out["src_des"], aux["src"], what + " src")
        _check_descriptors(oracle, sd, out["tgt_des"], aux["tgt"], what + " tgt")
        assert out["gt_label"].dtype == torch.int64 and out["gt_label"].shape == ref["gt_label"].shape
        assert torch.equal(out["gt_label"].cpu(), ref["gt_label"]), what
        es, oe = out["equi_score"].cpu().numpy(), ref["equi_score"].numpy()
        assert _rel_rows(es, oe).max() < 1e-3      # on maps that already differ by the descriptor stack's fp32 rounding
    else:
        assert out["pred_ind"].shape == ref["pred_ind"].shape and out["gt_ind"].dtype == torch.float32
        # a loose cross-check only: the two sides' maps differ by the descriptor stack's rounding.  The kernel's bound is
        # the a11 bound against float64 on its own recorded maps, test_train_fp64_gpu.py::test_production_route_vs_fp64
        assert np.abs(out["pred_ind"].cpu().numpy() - ref["pred_ind"].numpy()).max() < 2e-3
        # float labels: 1e-4 bins, plus the conditioning of acos where the cosine is next to +-1 (an fp32 cosine that is
        # a few ulps apart moves the angle by up to sqrt(2 * eps))
        g, e = out["gt_ind"].cpu().numpy(), ref["gt_ind"].numpy()
        th = e.astype(np.float64) * 2 * np.pi / cfg.patch.azi_n
        eps = 4 * 6e-8
        tol = 1e-4 + cfg.patch.azi_n / (2 * np.pi) * np.minimum(eps / np.maximum(np.abs(np.sin(th)), 1e-12), np.sqrt(2 * eps))
        circ = np.abs(g - e)
        circ = np.minimum(circ, cfg.patch.azi_n - circ)          # 20 and 0 are the same bin
        assert (circ <= tol).all() and (circ < 1e-4).mean() > 0.99, f"{what}: float label max diff {circ.max()}"
    # the statistics Trainer.evaluate derives from the dict
    lg = TS.trainer_losses(stage, out)
    lo = TS.trainer_losses(stage, {k: v for k, v in ref.items() if k != "aux"})
    for k in lo:
        tol = 0.0 if k.endswith("_acc") else 1e-4 * max(1.0, abs(lo[k]))
        assert abs(lg[k] - lo[k]) <= tol, f"{what}: {k} {lg[k]} vs {lo[k]}"


@pytest.mark.parametrize("workload", ["C1", "C2"])
@pytest.mark.parametrize("stage", ["Desc", "Pose"])
@pytest.mark.parametrize("case", ["draw", "isolated"])
def test_train_forward_against_oracle(dev, oracle, TS, workload, stage, case):
    cfg, data = _training_pair(workload, 0, stage, isolated=(case == "isolated"))
    model, sd = _model(cfg, dev)
    choice = None
    if case == "isolated":
        # an explicit match selection that keeps the isolated correspondence (the last match; empty ball query)
        n_all = len(TS.matching_indices(data["src_sds_pcd"], data["tgt_sds_pcd"], data["relt_pose"], data["voxel_sizes"][0]))
        choice = np.r_[np.arange(0, n_all - 1, max(1, (n_all - 1) // 255))[:255], n_all - 1]
    np.random.seed(11)
    ref = TS.train_forward(stage, sd, cfg, data, match_choice=choice, keep=True)
    st_o = np.random.get_state()
    if case == "draw":
        assert ref["aux"]["match_all"] >= cfg.train.pos_num and len(ref["aux"]["match"]) == cfg.train.pos_num
    else:
        kp = data["src_sds_pcd"][-1:]
        _, cnt = oracle.ball_query(data["src_fds_pcd"], kp, float(ref["aux"]["des_r"]), 4)
        assert cnt[0] == 0 and ref["aux"]["match"][-1, 0] == len(data["src_sds_pcd"]) - 1
    np.random.seed(11)
    with torch.no_grad():
        out = model(data, match_choice=choice)
    st_g = np.random.get_state()
    assert st_g[2] == st_o[2] and np.array_equal(st_g[1], st_o[1]), "NumPy draws differ from the oracle's"
    _compare_forward(oracle, TS, sd, cfg, stage, out, ref, f"{workload} {stage} {case}")


# ------------------------------------------------------------------------------------------------ drop-in
@pytest.mark.parametrize("stage", ["Desc", "Pose"])
def test_trainer_evaluate_drop_in(dev, oracle, TS, stage):
    """Driven like Trainer.evaluate: nn.DataParallel, a collate-shaped dict of CPU tensors, the global RNG, model.eval()
    and torch.no_grad().  NumPy's RNG state afterwards equals the oracle run's, which pins the draw order."""
    cfg, data = _training_pair("C1", 1, stage)
    model, sd = _model(cfg, dev)
    batch = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in data.items()}
    np.random.seed(5)
    ref = TS.train_forward(stage, sd, cfg, data, keep=True)
    st_o = np.random.get_state()
    net = torch.nn.DataParallel(model, device_ids=[0])
    net.eval()
    np.random.seed(5)
    with torch.no_grad():
        out = net(batch)
    st_g = np.random.get_state()
    assert st_g[2] == st_o[2] and np.array_equal(st_g[1], st_o[1])
    assert set(out) == ({"src_kpt", "tgt_kpt", "src_des", "tgt_des", "equi_score", "gt_label"} if stage == "Desc"
                        else {"pred_ind", "gt_ind"})
    _compare_forward(oracle, TS, sd, cfg, stage, out, ref, f"drop-in {stage}")


def test_training_mode_still_raises(dev):
    cfg, data = _training_pair("C1", 0, "Desc")
    model, _ = _model(cfg, dev)
    model.train()
    with pytest.raises(NotImplementedError, match="training-mode BatchNorm"):
        model(data)
    cfg.stage = "Weird"
    model.eval()
    with pytest.raises(NotImplementedError):
        model(data)


def test_fewer_than_two_patches_returns_none(dev, TS, capsys):
    cfg, data = _training_pair("C1", 0, "Pose")
    model, _ = _model(cfg, dev)
    with torch.no_grad():
        assert model(data, match_choice=[3]) is None
    assert "don't have enough patches" in capsys.readouterr().out
