"""CPU: the float64 oracle of the Pose training step (oracle/train_step.py) against the reference's own modules in
training mode (tests/golden/train_pose_step.npz, written by tests/tools/gen_train_pose_golden.py): the descriptor
network's batch-statistics forward twice (source, target), CostVolume + CostNet in training mode, every running
statistic afterwards, pred_ind and the gradients of Pose.conv after HuberLoss backward, to float64 rounding."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "train_pose_step.npz"))


def test_oracle_reproduces_reference_modules_in_training_mode(gold):
    from oracle import train_step as TP
    import gen_train_pose_golden as G
    import bufferx_b200 as bx
    cfg, sd, inv_s, inv_t, gt = G.case()
    hp = TP.bn_hparams(bx.BufferX(cfg))
    st = TP.state64(sd)
    stats = dict(src=[], tgt=[], pose=[])
    with torch.no_grad():
        _, es, _ = TP.desc_train(inv_s, st, stats["src"], hp)
        _, et, _ = TP.desc_train(inv_t, st, stats["tgt"], hp)
    params = TP.pose_params(sd)
    pred = TP.costnet_train(es[:, :, 1:6], et[:, :, 1:6], params, st, stats["pose"], hp)
    torch.nn.HuberLoss()(pred, torch.from_numpy(gt).double()).backward()
    assert np.abs(pred.detach().numpy() - gold["pred_ind"]).max() < 1e-12
    n = 0
    for k in gold.files:
        if not k.startswith("state."):
            continue
        key = k[len("state."):]
        o, r = st[key].numpy(), gold[k]
        if "num_batches_tracked" in key:
            assert int(o) == int(r) == int(sd[key]) + (2 if key.startswith("Desc") else 1), key
        else:
            assert np.abs(o - r).max() <= 1e-12 * max(1.0, np.abs(r).max()), key
        n += 1
    assert n == 3 * 19
    for k, p in params.items():
        g = p.grad.numpy().reshape(-1)
        norm = float(gold["gradnorm." + k][0])
        assert abs(np.linalg.norm(g) - norm) <= 1e-10 * norm, k
        assert np.abs(g[::G.GRAD_STRIDE] - gold["grad." + k]).max() <= 1e-10 * max(norm, 1e-300), k
