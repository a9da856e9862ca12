"""GPU: the Pose stage's training step (cfg.stage "Pose" under model.train()) against the float64 CPU oracle
(oracle/train_step.py): batch statistics and running updates of every BatchNorm, pred_ind, the gradients of every
Pose.conv parameter after loss.backward(), determinism, the Trainer.train_epoch drop-in, the refusals, and the eval-mode
forward after a step."""
import copy

import numpy as np
import pytest
import torch

from oracle.train_step_cases import G_ELEM, G_NORM, POSE_BN

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def TP(oracle):
    from oracle import train_step
    return train_step


def _setup(name, seed, aligned=None, trained_pose=True, pos_num=None):
    import bufferx_b200 as bx
    from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg(name)
    cfg.stage = "Pose"
    if pos_num is not None:
        cfg.train.pos_num = pos_num
    data = add_training_clouds(make_pair(name, seed), cfg)
    if aligned is not None:
        data["is_aligned_to_global_z"] = aligned
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=trained_pose)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    return cfg, data, model, sd


def _freeze_desc(model):
    for p in model.Desc.parameters():          # train.py:36-48 for the Pose stage
        p.requires_grad = False


def _step(model, data, seed):
    """One training forward + HuberLoss backward from NumPy seed ``seed`` -> (out, loss)."""
    model.train()
    np.random.seed(seed)
    out = model(data)
    loss = torch.nn.HuberLoss()(out["pred_ind"], out["gt_ind"].float())
    loss.backward()
    return out, loss


def _oracle(TP, sd, hp, cfg, data, seed):
    np.random.seed(seed)
    keep = {}
    r = TP.train_step(sd, hp, cfg, data, keep=keep)
    st = np.random.get_state()
    loss = torch.nn.functional.huber_loss(r["pred_ind"], r["gt_ind"].double())
    loss.backward()
    return r, keep, st


def _spy_costnet(model):
    """Record the equivariant maps the training step feeds CostNet (cap["es"], cap["et"], full height, on the CPU)."""
    cap = {}
    orig = model.Pose.conv.forward_train

    def spy(es, et, stats=None):
        cap["es"], cap["et"] = es.detach().cpu(), et.detach().cpu()
        return orig(es, et, stats)
    model.Pose.conv.forward_train = spy
    return cap


def _costnet_oracle(TP, sd, hp, cap, gt_ind):
    """CostNet's training forward + HuberLoss backward in float64 on the maps the GPU step fed it: the reference for pred_ind
    (the a11 bound holds against float64 on the kernel's own maps), the Pose BatchNorms and the gradients."""
    params, st, stats, keep = TP.pose_params(sd), TP.state64(sd), {"pose": []}, {}
    pred = TP.costnet_train(cap["es"][:, :, 1:6], cap["et"][:, :, 1:6], params, st, stats["pose"], hp, keep)
    torch.nn.functional.huber_loss(pred, gt_ind.detach().cpu().double()).backward()
    return dict(pred_ind=pred, params=params, state=st, stats=stats), keep


def _check_stats_and_running(model, sd0, r, sides):
    """Batch statistics and running buffers of the BatchNorms of ``sides`` ("src"/"tgt": Desc, "pose": Pose.conv) against
    the float64 oracle result ``r``; num_batches_tracked moved by exactly one per call.  Momentum comes from the model's
    modules and N / (N - 1) from the batch's sample count (oracle/train_step_cases.py)."""
    from oracle import train_step_cases as SC
    from oracle.train_step import bn_hparams
    got = model.last_train_stats
    hp = bn_hparams(model)
    K = int(r["pred_ind"].shape[0])
    bounds = {}
    for side in sides:
        keys = SC.POSE_BN if side == "pose" else SC.DESC_BN
        for key, b in zip(keys, SC.check_batch_stats(got[side], r["stats"][side], keys, side)):
            bounds.setdefault(key, []).append(b)
    msd = model.state_dict()
    for key in bounds:
        calls = 2 if key.startswith("Desc") else 1
        nbt0 = int(sd0[key + ".num_batches_tracked"])
        assert int(msd[key + ".num_batches_tracked"]) == nbt0 + calls, key
        assert int(r["state"][key + ".num_batches_tracked"]) == int(msd[key + ".num_batches_tracked"]), key
        SC.check_running_buffers(msd, r["state"], key, bounds[key], hp[key][0], nbt0, SC.bn_count(key, K))


def _check_grads(model, r, keep, TP, what):
    from oracle import train_step_cases as SC
    SC.check_grads(model.Pose.conv, r["params"], TP.grad_abs_bounds(keep, r["params"]), what)


@pytest.mark.parametrize("name,aligned", [("C1", False), ("C1", True), ("C2", False), ("C2", True)])
def test_step_matches_float64(dev, oracle, TP, name, aligned):
    cfg, data, model, sd = _setup(name, 0, aligned)
    model = model.to(dev)
    _freeze_desc(model)
    cap = _spy_costnet(model)
    out, _ = _step(model, data, 11)
    st_g = np.random.get_state()
    r, _, st_o = _oracle(TP, sd, TP.bn_hparams(model), cfg, data, 11)
    assert st_g[2] == st_o[2] and np.array_equal(st_g[1], st_o[1])      # the same draws in the same order
    assert set(out) == {"pred_ind", "gt_ind"} and out["pred_ind"].grad_fn is not None
    # the end-to-end float64 step: a loose cross-check of pred_ind (the two sides' maps differ by the descriptor stack's
    # rounding, which CostNet's batch statistics pass on), the exact draws, and the descriptor network's BatchNorms
    assert (out["pred_ind"].detach().cpu().double() - r["pred_ind"].detach()).abs().max() < 2e-3
    _check_stats_and_running(model, sd, r, ("src", "tgt"))
    # CostNet in float64 on the maps the step fed it: pred_ind within the a11 bound, the Pose BatchNorms, the gradients
    c, keep = _costnet_oracle(TP, sd, TP.bn_hparams(model), cap, out["gt_ind"])
    ind64, bound, _, _ = oracle.soft_argmax_bound(keep["logits"], keep["logits"].float())
    assert torch.allclose(ind64, c["pred_ind"].detach(), atol=1e-12)
    err = (out["pred_ind"].detach().cpu().double() - ind64).abs()
    assert (err <= torch.clamp(bound, min=1e-4)).all(), f"pred_ind err {err.max()}"
    _check_stats_and_running(model, sd, c, ("pose",))
    _check_grads(model, c, keep, TP, f"{name} aligned={aligned}")
    # gt_ind: that of the validation forward
    ev = copy.deepcopy(model).eval()
    np.random.seed(11)
    with torch.no_grad():
        ref = ev(data)
    assert torch.equal(ref["gt_ind"], out["gt_ind"])


def test_step_is_deterministic(dev):
    cfg, data, model, sd = _setup("C2", 1)
    model = model.to(dev)
    _freeze_desc(model)
    res = []
    for _ in range(2):
        model.load_state_dict(sd)
        model.zero_grad(set_to_none=True)
        _step(model, data, 3)
        res.append(({k: v.clone() for k, v in model.state_dict().items()},
                    [p.grad.clone() for p in model.Pose.conv.parameters()]))
    (s0, g0), (s1, g1) = res
    assert all(torch.equal(s0[k], s1[k]) for k in s0)
    assert all(torch.equal(a, b) for a, b in zip(g0, g1))


def test_backward_accumulates_and_no_grad_updates_stats(dev):
    cfg, data, model, sd = _setup("C1", 0, pos_num=64)
    model = model.to(dev)
    _freeze_desc(model)
    _step(model, data, 5)
    g1 = [p.grad.clone() for p in model.Pose.conv.parameters()]
    model.load_state_dict(sd)
    np.random.seed(5)
    out = model(data)
    loss = torch.nn.HuberLoss()(out["pred_ind"], out["gt_ind"].float())
    loss.backward(retain_graph=True)           # .grad accumulates, as autograd does, also over a retained graph
    loss.backward()
    for p, g in zip(model.Pose.conv.parameters(), g1):
        assert torch.allclose(p.grad, 3 * g, rtol=1e-6, atol=0.0)
    nbt = int(model.Pose.conv.ops[1].num_batches_tracked)
    with torch.no_grad():
        np.random.seed(5)
        out = model(data)
    assert out["pred_ind"].grad_fn is None
    assert int(model.Pose.conv.ops[1].num_batches_tracked) == nbt + 1
    assert int(model.Desc.pnt_layer[1].num_batches_tracked) == int(sd["Desc.pnt_layer.1.num_batches_tracked"]) + 4


def test_refusals(dev):
    cfg, data, model, _ = _setup("C1", 0, pos_num=32)
    model = model.to(dev).train()
    with pytest.raises(NotImplementedError, match="backward pass through Desc"):
        model(data)                             # Desc parameters still require grad
    _freeze_desc(model)
    cfg.stage = "Desc"
    with pytest.raises(NotImplementedError, match="training-mode BatchNorm"):
        model(data)
    cfg.stage = "Weird"
    with pytest.raises(NotImplementedError):
        model(data)


def test_eval_after_step_uses_the_new_state(dev):
    """The folded-weight caches are keyed on the parameter and buffer versions: the validation forward after one training
    step and optimizer.step() equals that of a fresh model loaded with the post-step state_dict."""
    import bufferx_b200 as bx
    cfg, data, model, sd = _setup("C1", 0, pos_num=128)
    model = model.to(dev)
    _freeze_desc(model)
    model.eval()
    np.random.seed(2)
    with torch.no_grad():
        before = model(data)                   # fills the caches
    opt = torch.optim.Adam(model.get_parameter(), lr=1e-3, weight_decay=1e-6)
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
    assert torch.equal(after["pred_ind"], exp["pred_ind"]) and torch.equal(after["gt_ind"], exp["gt_ind"])
    assert not torch.equal(after["pred_ind"], before["pred_ind"])


def test_large_activations_update_running_stats_once(dev, TP):
    """Pre-BatchNorm activations far outside fp16 range (weights scaled by 1e4: the eval route's fp16-split kernel would
    raise its flag and recompute) leave every running statistic with exactly one update per call, equal to the oracle's."""
    cfg, data, model, sd = _setup("C1", 0, pos_num=64)
    with torch.no_grad():
        for i in (0, 3):
            model.Desc.conv_net.ops[i].weight.mul_(1e4)
            model.Desc.conv_net.ops[i].bias.mul_(1e4)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model = model.to(dev)
    _freeze_desc(model)
    _step(model, data, 8)
    r, _, _ = _oracle(TP, sd, TP.bn_hparams(model), cfg, data, 8)
    _check_stats_and_running(model, sd, r, ("src", "tgt"))
    for key in POSE_BN:
        assert int(model.state_dict()[key + ".num_batches_tracked"]) == int(sd[key + ".num_batches_tracked"]) + 1


def test_trainer_train_epoch_drop_in(dev, TP):
    """The body of Trainer.train_epoch (trainer.py:93-167): nn.DataParallel, model.train(), Desc frozen as train.py does,
    Adam(get_parameter(), lr, weight_decay=1e-6), zero_grad, HuberLoss, backward, the finite check, step.  20 steps lower
    the Huber loss on a held-out pair; after one step the parameters follow the float64 oracle's Adam step."""
    cfg, data, model, sd = _setup("C1", 0, trained_pose=False, pos_num=128)
    from bufferx_b200.synth import add_training_clouds, make_pair
    held = add_training_clouds(make_pair("C1", 3), cfg)
    batches = [add_training_clouds(make_pair("C1", s), cfg) for s in (0, 1, 2)]
    batches = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in b.items()} for b in batches]
    model = model.to(dev)
    _freeze_desc(model)
    cap = _spy_costnet(model)
    net = torch.nn.DataParallel(model, device_ids=[0])
    huber = torch.nn.HuberLoss()
    lr = 1e-3
    opt = torch.optim.Adam(model.get_parameter(), lr=lr, weight_decay=1e-6)

    def held_loss():
        net.train()                            # batch statistics, as in the step; under no_grad
        np.random.seed(99)
        with torch.no_grad():
            o = net(held)
        return float(huber(o["pred_ind"], o["gt_ind"].float()))

    state0 = copy.deepcopy(model.state_dict())
    l0 = held_loss()
    model.load_state_dict(state0)
    losses = []
    for step in range(20):
        net.train()
        opt.zero_grad()
        np.random.seed(1000 + step)
        out = net(batches[step % 3])
        loss = huber(out["pred_ind"], out["gt_ind"].float())
        loss.backward()
        if any((~torch.isfinite(p.grad)).any() for p in model.get_parameter() if p.grad is not None):
            continue
        opt.step()
        losses.append(float(loss.detach()))
        if step == 0:                          # CostNet's float64 step on the maps this step fed it
            r, keep = _costnet_oracle(TP, {k: v.cpu() for k, v in state0.items()}, TP.bn_hparams(model), cap, out["gt_ind"])
            absb = TP.grad_abs_bounds(keep, r["params"])
            p64 = {k: v.detach().clone().requires_grad_(True) for k, v in r["params"].items()}
            for k in p64:
                p64[k].grad = r["params"][k].grad
            o64 = torch.optim.Adam(list(p64.values()), lr=lr, weight_decay=1e-6)
            o64.step()
            for i in [0, 3, 6, 9, 12, 15, 18, 21, 24, 27]:
                for kind in ("weight", "bias") if i == 27 else ("weight",):
                    k = f"ops.{i}.{kind}"
                    g64 = r["params"][k].grad
                    # where the float64 gradient's sign is not in doubt (10 x the gradient tolerance) and it is far above
                    # Adam's eps (1e-8), so the first step is lr sign(g) on both sides
                    decided = (g64.abs() > 10 * G_ELEM * absb[k]) & (g64.abs() > 10 * G_NORM * g64.abs().max()) & (g64.abs() > 1e-5)
                    got = getattr(model.Pose.conv.ops[i], kind).detach().cpu().double()
                    assert ((got - p64[k].detach()).abs()[decided] <= 0.05 * lr).all(), k
    assert len(losses) == 20
    assert held_loss() < l0
