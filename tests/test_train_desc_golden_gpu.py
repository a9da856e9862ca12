"""GPU: MiniSpinNet.train_desc (the Desc training step's CUDA route) on the inputs of tests/golden/train_desc_step.npz,
the reference's own modules in training mode, float64: desc, equi and equi_score, the running statistics after the
source and target calls, and every Desc gradient after the trainer's loss, within the bounds the step test uses
(oracle/train_step_cases.py).  Reads only tests/golden/ and the seeded inputs of tests/tools/gen_train_desc_golden.py."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def test_train_desc_matches_the_reference_golden(dev):
    import bufferx_b200 as bx
    import gen_train_desc_golden as G
    from bufferx_b200.models.BUFFERX import _EquiMatchFn
    from bufferx_b200.synth import init_synthetic_weights
    from oracle import train_desc as TD
    from oracle import train_step_cases as SC
    from oracle.train_step import bn_hparams, state64
    gold = np.load(os.path.join(HERE, "golden", "train_desc_step.npz"))
    cfg, sd, inv_s, inv_t, kpt, label = G.case()
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    model.load_state_dict(sd)
    model = model.to(dev).train()
    for p in model.Pose.parameters():
        p.requires_grad = False
    stats = dict(src=[], tgt=[])
    ds, es = model.Desc.train_desc(torch.from_numpy(inv_s).to(dev), stats["src"])
    dt, et = model.Desc.train_desc(torch.from_numpy(inv_t).to(dev), stats["tgt"])
    score = _EquiMatchFn.apply(es, et)
    loss = TD.desc_loss(ds.cpu(), dt.cpu(), kpt.astype(np.float64), score.cpu(), label)
    loss.backward()
    # outputs: the step test's bounds
    for got, key in ((ds, "src_desc"), (dt, "tgt_desc")):
        assert np.abs(got.detach().cpu().double().numpy() - gold[key]).max() < 1e-5, key
    for got, key in ((es, "src_equi"), (et, "tgt_equi")):
        e = got.detach().cpu().double().numpy().reshape(-1)[::G.EQUI_STRIDE]
        assert np.abs(e - gold[key]).max() < 1e-5, key
    s64 = torch.from_numpy(gold["equi_score"])
    err = (score.detach().cpu().double() - s64).abs()
    assert (err <= 1e-4 * s64.abs().amax(dim=1, keepdim=True) + 1e-5).all(), float(err.max())
    # running statistics: the float64 oracle's batch statistics bound the step's, and the golden holds the reference's
    # running buffers (the oracle reproduces them to 1e-12, tests/test_train_desc_golden_cpu.py)
    hp = bn_hparams(model)
    params, st, ostats = TD.desc_params(sd), state64(sd), dict(src=[], tgt=[])
    keeps = [{}, {}]
    o_s = TD.desc_train(inv_s, params, st, ostats["src"], hp, keeps[0])
    o_t = TD.desc_train(inv_t, params, st, ostats["tgt"], hp, keeps[1])
    TD.desc_loss(o_s[0], o_t[0], kpt.astype(np.float64), TD.equi_match(o_s[1], o_t[1]), label).backward()
    bounds = {}
    for side in ("src", "tgt"):
        for key, b in zip(SC.DESC_BN, SC.check_batch_stats(stats[side], ostats[side], SC.DESC_BN, side)):
            bounds.setdefault(key, []).append(b)
    msd = model.state_dict()
    ostate = {k[len("state."):]: torch.from_numpy(np.asarray(gold[k])) for k in gold.files if k.startswith("state.")}
    K = inv_s.shape[0]
    for key in SC.DESC_BN:
        nbt0 = int(sd[key + ".num_batches_tracked"])
        assert int(msd[key + ".num_batches_tracked"]) == int(ostate[key + ".num_batches_tracked"]) == nbt0 + 2, key
        SC.check_running_buffers(msd, ostate, key, bounds[key], hp[key][0], nbt0, SC.bn_count(key, K))
    # gradients: the golden's strided elements within G_ELEM of the absolute-value contraction, norms within G_NORM
    absb = TD.grad_abs_bounds(keeps, params)
    named = dict(model.Desc.named_parameters())
    worst = {}
    for k in params:
        g = named[k].grad.detach().cpu().double().numpy().reshape(-1)
        lim = SC.G_ELEM * absb[k].numpy().reshape(-1)[::G.GRAD_STRIDE] + 1e-30
        e = np.abs(g[::G.GRAD_STRIDE] - gold["grad." + k]) / lim
        worst[k] = float(e.max())
        assert worst[k] <= 1.0, f"{k}: elementwise err {worst[k]:.3g} x bound"
        norm = float(gold["gradnorm." + k][0])
        if norm > 10 * SC.G_ELEM * float(absb[k].norm()):
            assert abs(np.linalg.norm(g) - norm) <= SC.G_NORM * norm, k
    print("\n[train-desc-golden] gradient error / bound:", {k: round(v, 4) for k, v in worst.items()})
