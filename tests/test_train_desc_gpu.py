"""GPU: the Desc stage's training step (cfg.stage "Desc" under model.train(), CostNet frozen) against the float64 CPU oracle
(oracle/train_desc.py): the NumPy draws, batch statistics and running updates of every descriptor BatchNorm, desc / equi /
equi_score, the gradient of every Desc parameter after the trainer's loss.backward(), determinism, accumulation over a
retained graph, torch.no_grad(), a partially frozen Desc, the eval forward after a step, and the Trainer.train_epoch
drop-in."""
import copy

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


def _setup(name, seed, aligned=None, pos_num=None):
    import bufferx_b200 as bx
    from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg(name)
    cfg.stage = "Desc"
    if pos_num is not None:
        cfg.train.pos_num = pos_num
    data = add_training_clouds(make_pair(name, seed), cfg)
    if aligned is not None:
        data["is_aligned_to_global_z"] = aligned
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    return cfg, data, model, sd


def _freeze_pose(model):
    for p in model.Pose.parameters():          # train.py:36-48 for the Desc stage
        p.requires_grad = False


def _loss(out):
    from oracle import train_desc as TD
    return TD.desc_loss(out["src_des"].cpu(), out["tgt_des"].cpu(), out["tgt_kpt"].cpu().numpy(), out["equi_score"].cpu(),
                        out["gt_label"].cpu().numpy())


def _step(model, data, seed):
    model.train()
    np.random.seed(seed)
    out = model(data)
    loss = _loss(out)
    loss.backward()
    return out, loss


def _spy(model):
    """Record the samples each train_desc call fed the point layer and the upstream gradients of its (desc, equi)."""
    cap = []
    orig = model.Desc.train_desc

    def spy(inv, stats=None):
        d, e = orig(inv, stats)
        rec = dict(inv=inv.detach().cpu().numpy(), desc=d.detach().cpu(), equi=e.detach().cpu())
        if d.requires_grad:
            d.register_hook(lambda g: rec.__setitem__("g_desc", g.detach().cpu()))
            e.register_hook(lambda g: rec.__setitem__("g_equi", g.detach().cpu()))
        cap.append(rec)
        return d, e
    model.Desc.train_desc = spy
    return cap


@pytest.mark.parametrize("name,aligned", [("C1", False), ("C1", True), ("C2", False), ("C2", True)])
def test_step_matches_float64(dev, oracle, name, aligned):
    from oracle import train_desc as TD
    from oracle import train_step_cases as SC
    from oracle.train_step import bn_hparams, state64
    cfg, data, model, sd = _setup(name, 0, aligned)
    model = model.to(dev)
    _freeze_pose(model)
    cap = _spy(model)
    out, _ = _step(model, data, 11)
    st_g = np.random.get_state()
    hp = bn_hparams(model)
    np.random.seed(11)
    r = TD.train_step(sd, hp, cfg, data)
    st_o = np.random.get_state()
    assert st_g[2] == st_o[2] and np.array_equal(st_g[1], st_o[1])      # the same draws in the same order
    assert set(out) == {"src_kpt", "tgt_kpt", "src_des", "tgt_des", "equi_score", "gt_label"}
    assert all(out[k].grad_fn is not None for k in ("src_des", "tgt_des", "equi_score"))
    assert len(cap) == 2
    # batch statistics and running buffers of the ten descriptor BatchNorms (two calls each), none of CostNet's moved
    K = int(r["K"])
    got = model.last_train_stats
    bounds = {}
    for side in ("src", "tgt"):
        for key, b in zip(SC.DESC_BN, SC.check_batch_stats(got[side], r["stats"][side], SC.DESC_BN, side)):
            bounds.setdefault(key, []).append(b)
    msd = model.state_dict()
    for key in SC.DESC_BN:
        nbt0 = int(sd[key + ".num_batches_tracked"])
        assert int(msd[key + ".num_batches_tracked"]) == nbt0 + 2, key
        SC.check_running_buffers(msd, r["state"], key, bounds[key], hp[key][0], nbt0, SC.bn_count(key, K))
    for key in SC.POSE_BN:
        assert int(msd[key + ".num_batches_tracked"]) == int(sd[key + ".num_batches_tracked"]), key
    # the float64 network on the exact samples the step fed it, with the step's upstream gradients
    params, st, stats = TD.desc_params(sd), state64(sd), []
    keeps, outs = [], []
    for rec in cap:
        keep = {}
        outs.append(TD.desc_train(rec["inv"], params, st, stats, hp, keep))
        keeps.append(keep)
    for rec, (d64, e64) in zip(cap, outs):
        assert (rec["desc"].double() - d64.detach()).abs().max() < 1e-5
        assert (rec["equi"].double() - e64.detach()).abs().max() < 1e-5
    score64 = TD.equi_match(outs[0][1].detach(), outs[1][1].detach())
    err = (out["equi_score"].detach().cpu().double() - score64).abs()
    assert (err <= 1e-4 * score64.abs().amax(dim=1, keepdim=True) + 1e-5).all(), float(err.max())
    torch.autograd.backward([t for o in outs for t in o], [rec[k] .double() for rec in cap for k in ("g_desc", "g_equi")])
    TD.check_grads(model.Desc, params, TD.grad_abs_bounds(keeps, params), f"{name} aligned={aligned}")
    # gt_label: that of the validation forward
    ev = copy.deepcopy(model).eval()
    np.random.seed(11)
    with torch.no_grad():
        ref = ev(data)
    assert torch.equal(ref["gt_label"], out["gt_label"])


def test_step_is_deterministic(dev):
    cfg, data, model, sd = _setup("C2", 1)
    model = model.to(dev)
    _freeze_pose(model)
    res = []
    for _ in range(2):
        model.load_state_dict(sd)
        model.zero_grad(set_to_none=True)
        _step(model, data, 3)
        res.append(({k: v.clone() for k, v in model.state_dict().items()}, [p.grad.clone() for p in model.Desc.parameters()]))
    (s0, g0), (s1, g1) = res
    assert all(torch.equal(s0[k], s1[k]) for k in s0)
    assert all(torch.equal(a, b) for a, b in zip(g0, g1))


def test_backward_accumulates_and_no_grad_updates_stats(dev):
    cfg, data, model, sd = _setup("C1", 0, pos_num=64)
    model = model.to(dev)
    _freeze_pose(model)
    _step(model, data, 5)
    g1 = [p.grad.clone() for p in model.Desc.parameters()]
    model.load_state_dict(sd)
    np.random.seed(5)
    out = model(data)
    loss = _loss(out)
    loss.backward(retain_graph=True)
    loss.backward()
    for p, g in zip(model.Desc.parameters(), g1):
        assert torch.allclose(p.grad, 3 * g, rtol=1e-5, atol=1e-30), p.shape
    nbt = int(model.Desc.pnt_layer[1].num_batches_tracked)
    with torch.no_grad():
        np.random.seed(5)
        out = model(data)
    assert out["src_des"].grad_fn is None and out["equi_score"].grad_fn is None
    assert int(model.Desc.pnt_layer[1].num_batches_tracked) == nbt + 2
    assert int(model.Desc.conv_net.ops[1].num_batches_tracked) == nbt + 2


def test_partially_frozen_desc(dev):
    cfg, data, model, _ = _setup("C1", 0, pos_num=64)
    model = model.to(dev)
    _freeze_pose(model)
    for name, p in model.Desc.named_parameters():
        p.requires_grad = name.startswith("pnt_layer")
    _step(model, data, 6)
    for name, p in model.Desc.named_parameters():
        assert (p.grad is not None) == name.startswith("pnt_layer"), name
        if p.grad is not None:
            assert torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0, name


def test_refusals(dev):
    cfg, data, model, _ = _setup("C1", 0, pos_num=32)
    model = model.to(dev).train()
    with pytest.raises(NotImplementedError, match="training-mode BatchNorm"):
        model(data)                             # Pose parameters still require grad
    _freeze_pose(model)
    cfg.stage = "Pose"
    with pytest.raises(NotImplementedError, match="backward pass through Desc"):
        model(data)


def test_fewer_than_two_patches_returns_none(dev, capsys):
    cfg, data, model, _ = _setup("C1", 0)
    model = model.to(dev)
    _freeze_pose(model)
    model.train()
    np.random.seed(0)
    assert model(data, match_choice=[0]) is None
    assert "enough patches" in capsys.readouterr().out


def test_eval_after_step_uses_the_new_state(dev):
    import bufferx_b200 as bx
    cfg, data, model, sd = _setup("C1", 0, pos_num=128)
    model = model.to(dev)
    _freeze_pose(model)
    model.eval()
    np.random.seed(2)
    with torch.no_grad():
        before = model(data)                   # fills the caches
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-3, weight_decay=1e-6)
    _step(model, data, 4)
    opt.step()
    model.eval()
    np.random.seed(2)
    with torch.no_grad():
        after = model(data)
    fresh = bx.BufferX(cfg).to(dev)
    fresh.load_state_dict(model.state_dict())
    fresh.eval()
    np.random.seed(2)
    with torch.no_grad():
        exp = fresh(data)
    for k in ("src_des", "tgt_des", "equi_score"):
        assert torch.equal(after[k], exp[k]), k
    assert not torch.equal(after["src_des"], before["src_des"])


def test_trainer_train_epoch_drop_in(dev):
    """The body of Trainer.train_epoch (trainer.py:93-167) for the Desc stage: nn.DataParallel, model.train(), CostNet frozen
    as train.py does, Adam at cfg.optim.lr["Desc"], zero_grad, 4 ContrastiveLoss + CE, backward, the finite check, step;
    20 steps on one seeded pair, every one finite, and the last loss below the first."""
    cfg, data, model, sd = _setup("C1", 0, pos_num=128)
    model = model.to(dev)
    _freeze_pose(model)
    batch = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in data.items()}
    net = torch.nn.DataParallel(model, device_ids=[0])
    lr = cfg.optim.lr["Desc"] if isinstance(cfg.optim.lr, dict) else cfg.optim.lr
    opt = torch.optim.Adam(model.get_parameter(), lr=lr, weight_decay=1e-6)
    losses = []
    for step in range(20):
        net.train()
        opt.zero_grad()
        np.random.seed(1000)
        out = net(batch)
        loss = _loss(out)
        loss.backward()
        finite = all(torch.isfinite(p.grad).all() for p in model.get_parameter() if p.grad is not None)
        assert finite, step
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0], losses
