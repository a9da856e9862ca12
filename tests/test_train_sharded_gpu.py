"""GPU: sharded training (DESIGN.md §8).  ops.dp_mean against its torch float64 restatement; two and three ranks on one
H100 over gloo (mp.spawn, every process joined) training C1 pairs through driver.train_step / train_sharded, checked
bit for bit across ranks and against a single-process emulation; world 1 against the plain single-GPU loop; NCCL with
one rank per GPU when the machine has two."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _restated(g):
    """ops.dp_mean in torch float64: contributing rows summed in rank order from the first, divided, .float()."""
    rows = g[g[:, -1] != 0, :-1].double()
    if rows.shape[0] == 0:
        return None, 0
    s = rows[0].clone()
    for r in rows[1:]:
        s = s + r
    return (s / rows.shape[0]).float(), rows.shape[0]


def _same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(-1).view(torch.int8),
                                                                      b.contiguous().view(-1).view(torch.int8))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


# --------------------------------------------------------------------------- 1. the kernel
@pytest.mark.parametrize("W", [1, 2, 3, 8])
@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 2 ** 20 + 1])
@pytest.mark.parametrize("who", ["none", "one", "all"])
def test_dp_mean_matches_float64_restatement(dev, W, n, who):
    from bufferx_b200 import ops
    g = torch.Generator().manual_seed(W * 1000 + n % 997)
    x = torch.randn((W, n + 1), generator=g) * torch.exp(torch.randn((W, n + 1), generator=g) * 3)
    x[:, n] = {"none": 0.0, "one": 0.0, "all": 1.0}[who]
    if who == "one":
        x[W - 1, n] = -2.5                                   # any non-zero flag counts
    out, count = ops.dp_mean(x.to(dev))
    want, c = _restated(x)
    assert int(count.item()) == c
    if c:
        assert _same_bits(out.cpu(), want)
        if c == 1:
            assert _same_bits(out.cpu(), x[W - 1, :n] if who == "one" else x[0, :n])    # one contributor: the identity


def test_dp_mean_nonfinite_and_magnitudes(dev):
    from bufferx_b200 import ops
    W, n = 3, 4099
    x = torch.zeros((W, n + 1))
    mags = torch.tensor([1e-30, -1e-30, 1e30, -1e30, 3.0, 1e-20, 7e25, -0.0])
    x[:, :n] = mags[torch.arange(W * n).reshape(W, n) % 8] * torch.linspace(0.5, 2, W)[:, None]
    x[1, 10], x[1, 11], x[1, 12] = float("nan"), float("inf"), -float("inf")
    x[0, 12] = float("inf")                                 # inf + -inf -> NaN
    x[2, 13] = 3e38
    x[1, 13] = 3e38                                          # float64 holds the sum; the mean rounds back into range
    x[:, n] = torch.tensor([1.0, 1.0, 1.0])
    out, count = ops.dp_mean(x.to(dev))
    want, c = _restated(x)
    assert int(count.item()) == 3 and _same_bits(out.cpu(), want)
    assert torch.isnan(out[10]) and torch.isinf(out[11]) and torch.isnan(out[12]) and torch.isfinite(out[13])
    x[1, n] = 0.0                                            # the non-finite rank does not contribute: nothing propagates
    out, _ = ops.dp_mean(x.to(dev))
    want, _ = _restated(x)
    assert _same_bits(out.cpu(), want) and torch.isfinite(out[10:12]).all()


def test_dp_mean_refusals_launch_nothing(dev):
    from bufferx_b200 import ops
    lib = ops.load_library()
    g = torch.ones((2, 5), device=dev)
    out = torch.zeros(4, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    before = ops.launch_count()
    s = ops._stream()
    for args in [(None, 2, 4, out.data_ptr(), cnt.data_ptr()), (g.data_ptr(), 2, 4, None, cnt.data_ptr()),
                 (g.data_ptr(), 2, 4, out.data_ptr(), None), (g.data_ptr(), 0, 4, out.data_ptr(), cnt.data_ptr()),
                 (g.data_ptr(), -1, 4, out.data_ptr(), cnt.data_ptr()), (g.data_ptr(), 2, -1, out.data_ptr(), cnt.data_ptr())]:
        assert lib.bx_dp_mean(*args, s) == -1
    assert ops.launch_count() == before
    for bad in [torch.ones(5, device=dev), torch.ones((2, 5), dtype=torch.float64, device=dev), torch.ones((2, 5)),
                torch.ones((0, 5), device=dev), torch.ones((2, 10), device=dev)[:, ::2]]:
        with pytest.raises(ops.BufferXError):
            ops.dp_mean(bad)
    assert ops.launch_count() == before and (out == 0).all() and (cnt == 0).all()


# --------------------------------------------------------------------------- helpers of the training runs
def _desc_loss(out):
    loss = 4 * (out["src_des"] - out["tgt_des"]).pow(2).sum(1).mean() + torch.nn.functional.cross_entropy(out["equi_score"], out["gt_label"])
    return loss, {"desc_loss": float(loss.item())}


def _pose_loss(out):
    loss = torch.nn.HuberLoss()(out["pred_ind"], out["gt_ind"].float())
    return loss, {"match_loss": float(loss.item())}


LOSS = {"Desc": _desc_loss, "Pose": _pose_loss}


def _pair(i, cfg, no_matches=False):
    from bufferx_b200.synth import add_training_clouds, make_pair
    d = add_training_clouds(make_pair("C1", i), cfg)
    if no_matches:
        d["tgt_sds_pcd"] = d["tgt_sds_pcd"] + np.float32(100.0)
    return d


def _model(stage, device):
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    cfg = workload_cfg("C1")
    cfg.stage = stage
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    for p in getattr(model, "Pose" if stage == "Desc" else "Desc").parameters():
        p.requires_grad = False
    model = model.to(device)
    model.train()
    return cfg, model, torch.optim.Adam(model.get_parameter(), lr=1e-3, weight_decay=1e-6)


def _snap(model, opt):
    return dict(model={k: v.detach().cpu().clone() for k, v in model.state_dict().items()},
                adam={k: {n: t.cpu().clone() if isinstance(t, torch.Tensor) else t for n, t in s.items()}
                      for k, s in opt.state_dict()["state"].items()})


def _equal_tree(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_equal_tree(a[k], b[k]) for k in a)
    if isinstance(a, torch.Tensor):
        return _same_bits(a, b)
    return a == b


def _seed(step, rank):
    np.random.seed(1000 * step + rank)
    torch.manual_seed(1000 * step + rank)


def _init(rank, world, port, backend):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    import datetime
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(minutes=5))
    return dev


# --------------------------------------------------------------------------- 2, 5, 6: two ranks
def _two_rank_worker(rank, world, port, out, backend):
    dev = _init(rank, world, port, backend)
    from bufferx_b200.driver import train_sharded, train_step, validate_sharded
    res = {}
    for stage in ("Desc", "Pose"):
        cfg, model, opt = _model(stage, dev)
        steps = []
        for s in range(2):
            _seed(s, rank)
            count, stepped, _ = train_step(model, opt, _pair(2 * s + rank, cfg), LOSS[stage])
            steps.append((count, stepped))
        res[stage] = dict(steps=steps, **_snap(model, opt))
    if backend == "gloo":
        # 5. a non-finite loss on rank 1: nobody steps
        cfg, model, opt = _model("Pose", dev)
        before = _snap(model, opt)["model"]
        _seed(0, rank)
        loss = _pose_loss if rank == 0 else (lambda o: (_pose_loss(o)[0] * float("nan"), {}))
        count, stepped, _ = train_step(model, opt, _pair(rank, cfg), loss)
        res["nonfinite"] = dict(count=count, stepped=stepped, before=before, **_snap(model, opt))
        # 6. train_sharded with sharded validation and snapshots
        cfg, model, opt = _model("Desc", dev)
        cfg.train.epoch, cfg.train.max_iter = 1, 10
        sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.5)
        own = []

        def eval_stats(o):
            st = {"desc_loss": float((o["src_des"] - o["tgt_des"]).pow(2).sum(1).mean()), "desc_acc": float(o["src_des"].shape[0])}
            own.append(st)
            return st
        train_set, val_set = [_pair(10 + i, cfg) for i in range(3)], [_pair(20 + i, cfg) for i in range(3)]
        hist = train_sharded(model, opt, sched, train_set, val_set, cfg, _desc_loss, eval_stats, seed=7,
                             snapshot_root=os.path.join(out, "snap"))
        means, recs = validate_sharded(model, val_set, eval_stats)
        np.random.seed(99)
        model.eval()
        with torch.no_grad():
            ev = model(val_set[0])
        res["sharded"] = dict(hist=hist, means=means, recs=recs, own=own, mine=list(range(rank, 3, world)),
                              eval={k: v.cpu() for k, v in ev.items()}, **_snap(model, opt))
        # gloo's all_gather on CUDA tensors (PyTorch lists it as CPU-only)
        try:
            t = torch.full((2,), float(rank), device=dev)
            bufs = [torch.empty_like(t) for _ in range(world)]
            dist.all_gather(bufs, t)
            torch.cuda.synchronize()
            res["gloo_cuda_all_gather"] = "ran: " + str([b.cpu().tolist() for b in bufs])
        except Exception as e:             # noqa: BLE001
            res["gloo_cuda_all_gather"] = f"refused: {type(e).__name__}: {str(e).splitlines()[0][:200]}"
    torch.save(res, os.path.join(out, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _emulate(stage, ranks, dev):
    """Single process: each rank's pair in turn from the common pre-step state and that rank's NumPy state, the results
    combined with torch float64 in rank order, then Adam on the master copy."""
    from bufferx_b200.driver import _bn_buffers
    cfg, master, opt = _model(stage, dev)
    params = [p for p in master.parameters() if p.requires_grad]
    for s in range(2):
        grads, bufs = [], []
        for r in range(ranks):
            _, work, _ = _model(stage, dev)
            work.load_state_dict(master.state_dict())
            work.train()
            _seed(s, r)
            out = work(_pair(2 * s + r, cfg))
            LOSS[stage](out)[0].backward()
            grads.append([p.grad.double() for p in work.parameters() if p.requires_grad])
            bufs.append([b.double() for b in _bn_buffers(work)])

        def mean(rows):
            acc = rows[0]
            for x in rows[1:]:
                acc = acc + x
            return acc / len(rows)
        opt.zero_grad()
        for i, p in enumerate(params):
            p.grad = mean([g[i] for g in grads]).float()
        with torch.no_grad():
            for i, b in enumerate(_bn_buffers(master)):
                b.copy_(mean([x[i] for x in bufs]).to(b.dtype))
        assert all(torch.isfinite(p.grad).all() for p in params)
        opt.step()
    return _snap(master, opt)


@pytest.fixture(scope="module")
def two_ranks(dev, tmp_path_factory):
    out = str(tmp_path_factory.mktemp("two_ranks"))
    mp.spawn(_two_rank_worker, args=(2, 29541, out, "gloo"), nprocs=2, join=True)
    return out, [torch.load(os.path.join(out, f"rank{r}.pt"), weights_only=False) for r in range(2)]


@pytest.mark.parametrize("stage", ["Desc", "Pose"])
def test_two_ranks_bit_identical_and_equal_to_emulation(dev, two_ranks, stage):
    _, (r0, r1) = two_ranks
    assert r0[stage]["steps"] == r1[stage]["steps"] == [(2, True), (2, True)]
    assert _equal_tree({k: r0[stage][k] for k in ("model", "adam")}, {k: r1[stage][k] for k in ("model", "adam")})
    em = _emulate(stage, 2, dev)
    assert _equal_tree(em, {k: r0[stage][k] for k in ("model", "adam")})


def test_nonfinite_loss_on_one_rank_skips_every_rank(two_ranks):
    _, (r0, r1) = two_ranks
    a, b = r0["nonfinite"], r1["nonfinite"]
    assert (a["count"], a["stepped"]) == (b["count"], b["stepped"]) == (2, False)
    params = [k for k in a["before"] if k.startswith("Pose.") and not k.split(".")[-1].startswith(("running", "num_batches"))]
    assert params and all(_same_bits(a["model"][k], a["before"][k]) and _same_bits(b["model"][k], a["before"][k]) for k in params)
    assert _equal_tree(a["model"], b["model"]) and a["adam"] == {} == b["adam"]
    assert not _equal_tree(a["model"], a["before"])          # the averaged running statistics still apply


def test_sharded_validation_and_best_snapshot(dev, two_ranks):
    out, (r0, r1) = two_ranks
    a, b = r0["sharded"], r1["sharded"]
    for r in (a, b):                                          # gathered per-pair statistics equal each rank's own
        recs = {int(x[0]): x for x in r["recs"]}
        assert sorted(recs) == [0, 1, 2]
        own = r["own"][-len(r["mine"]):]                      # the last validation pass
        for i, st in zip(r["mine"], own):
            assert recs[i][1] == 1.0 and recs[i][2 + 5 + 0] == st["desc_loss"] and recs[i][2 + 5 + 1] == st["desc_acc"]
    assert np.array_equal(a["recs"], b["recs"], equal_nan=True) and a["hist"] == b["hist"] and a["means"] == b["means"]
    vals = [float(x[7]) for x in a["recs"]]
    assert a["means"]["desc_loss"] == (vals[0] + vals[1] + vals[2]) / 3 and a["means"]["match_loss"] == 0
    assert _equal_tree({k: a[k] for k in ("model", "adam")}, {k: b[k] for k in ("model", "adam")})
    assert sorted(os.listdir(os.path.join(out, "snap", "Desc"))) == ["0.pth", "best.pth"]
    import bufferx_b200 as bx
    from bufferx_b200.synth import workload_cfg
    cfg = workload_cfg("C1")
    cfg.stage = "Desc"
    fresh = bx.BufferX(cfg)
    fresh.load_state_dict(torch.load(os.path.join(out, "snap", "Desc", "best.pth"), map_location="cpu"), strict=True)
    fresh = fresh.to(dev).eval()
    np.random.seed(99)
    with torch.no_grad():
        ev = fresh(_pair(20, cfg))
    assert all(_same_bits(ev[k].cpu(), a["eval"][k]) for k in a["eval"])
    print("gloo all_gather on CUDA tensors:", r0["gloo_cuda_all_gather"])


# --------------------------------------------------------------------------- 4. three ranks, an idle rank, a None pair
def _three_rank_worker(rank, world, port, out):
    dev = _init(rank, world, port, "gloo")
    from bufferx_b200.driver import train_step
    cfg, model, opt = _model("Desc", dev)
    # 5 pairs over 3 ranks: step 0 = pairs 0, 1, 2 (pair 2 has no ground-truth match: its forward returns None),
    # step 1 = pairs 3, 4 and rank 2 idle
    plan = [[_pair(30, cfg), _pair(31, cfg), _pair(32, cfg, no_matches=True)], [_pair(33, cfg), _pair(34, cfg), None]]
    rec = []
    for s, step in enumerate(plan):
        _seed(s, rank)
        count, stepped, _ = train_step(model, opt, step[rank], _desc_loss)
        rec.append(dict(count=count, stepped=stepped, **_snap(model, opt)))
    torch.save(rec, os.path.join(out, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_three_ranks_idle_rank_and_none_pair(dev, tmp_path):
    mp.spawn(_three_rank_worker, args=(3, 29551, str(tmp_path)), nprocs=3, join=True)
    rs = [torch.load(str(tmp_path / f"rank{r}.pt"), weights_only=False) for r in range(3)]
    assert [(s["count"], s["stepped"]) for s in rs[0]] == [(2, True), (2, True)]
    for s in range(2):
        for r in (1, 2):
            assert _equal_tree(rs[0][s], rs[r][s])            # parameters, Adam state, every buffer incl. num_batches_tracked
    nbt = [k for k in rs[0][0]["model"] if k.endswith("num_batches_tracked") and k.startswith("Desc.")]
    start = _snap(*_model("Desc", dev)[1:])["model"]
    assert nbt and all(int(rs[2][1]["model"][k]) >= int(start[k]) for k in nbt) and any(
        int(rs[2][1]["model"][k]) > int(start[k]) for k in nbt)                        # the idle rank took the others' count


# --------------------------------------------------------------------------- 3. world 1 against the plain loop
def test_world1_equals_plain_single_gpu_loop(dev):
    from bufferx_b200.driver import train_sharded
    cfg, model, opt = _model("Desc", dev)
    cfg.train.epoch, cfg.train.max_iter = 1, 3
    pairs = [_pair(40 + i, cfg) for i in range(4)]
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.5)
    train_sharded(model, opt, sched, pairs, [], cfg, _desc_loss, lambda o: {}, seed=5)
    _, plain, popt = _model("Desc", dev)
    np.random.seed(5)
    torch.manual_seed(5)
    for i in np.random.RandomState(5).permutation(4)[:3]:
        popt.zero_grad()
        out = plain(pairs[int(i)])
        _desc_loss(out)[0].backward()
        if all(torch.isfinite(p.grad).all() for p in plain.parameters() if p.grad is not None):
            popt.step()
    assert _equal_tree(_snap(model, opt), _snap(plain, popt))


# --------------------------------------------------------------------------- NCCL, one rank per GPU
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="NCCL needs two GPUs (one rank per device)")
def test_two_ranks_nccl(dev, tmp_path):
    mp.spawn(_two_rank_worker, args=(2, 29561, str(tmp_path), "nccl"), nprocs=2, join=True)
    r0, r1 = (torch.load(str(tmp_path / f"rank{r}.pt"), weights_only=False) for r in range(2))
    for stage in ("Desc", "Pose"):
        assert r0[stage]["steps"] == [(2, True), (2, True)]
        assert _equal_tree({k: r0[stage][k] for k in ("model", "adam")}, {k: r1[stage][k] for k in ("model", "adam")})
