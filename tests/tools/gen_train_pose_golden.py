"""Regenerate tests/golden/train_pose_step.npz: the reference's own modules in training mode, in float64, on one small
synthetic Pose step.

    python tests/tools/gen_train_pose_golden.py /path/to/reference/checkout

Builds the unmodified reference ``BufferX`` (third-party leaves stubbed as oracle/ref_check.py does), loads the synthetic
C1 state_dict, casts it to float64 and calls ``model.train()``.  Then, on stored de-rotated point-layer inputs of a source
and a target call (K patches each), it runs the reference's own ``Desc.pnt_layer`` + max, ``Desc.conv_net``
(Cylindrical_Net) and ``Desc.pool_layer`` in patch_embedder.py's order (:81-90) for the source, then the target, then
``Pose`` (CostVolume + CostNet) on rows 1..ele_n-2 of the two equivariant maps, HuberLoss against stored labels and
backward.  Stored: pred_ind, every running statistic and num_batches_tracked afterwards, and of the gradient of
every ``Pose.conv`` parameter its norm and every GRAD_STRIDE-th element.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_check  # noqa: E402

K = 4
GRAD_STRIDE = 97


def case():
    """-> (cfg, state_dict, inv_s, inv_t, gt_ind): C1 synthetic weights (fitted CostNet), point-layer inputs of K patches
    with zero slots, as SPT leaves them, and labels in [0, 20)."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    cfg = workload_cfg("C1")
    cfg.stage = "Pose"
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    rng = np.random.RandomState(17)
    inv = rng.uniform(-1, 1, size=(2, K, 420, 10, 3)).astype(np.float32)
    inv[rng.uniform(size=(2, K, 420, 10)) < 0.3] = 0.0
    gt = (rng.uniform(size=K) * 20).astype(np.float32)
    return cfg, sd, inv[0], inv[1], gt


def main(ref_root):
    ref_check.install_stubs(0)
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    for m in [k for k in sys.modules if k in ("models", "utils") or k.startswith(("models.", "utils."))]:
        del sys.modules[m]
    import models.BUFFERX as RB
    cfg, sd, inv_s, inv_t, gt = case()
    ref = RB.BufferX(cfg)
    ref.load_state_dict(sd, strict=True)
    ref = ref.double()
    ref.train()
    for p in ref.Desc.parameters():
        p.requires_grad = False
    D = ref.Desc

    def desc(inv):
        x = D.pnt_layer(torch.from_numpy(inv).double().permute(0, 3, 1, 2))
        x = F.max_pool2d(x, kernel_size=(1, x.shape[-1])).squeeze(3)
        x = x.view(x.shape[0], x.shape[1], D.rad_n, D.ele_n, D.azi_n)
        x, _ = D.conv_net(x)
        D.pool_layer(x)                       # its running statistics move; its output only reaches desc
        return F.normalize(x, p=2, dim=1)

    es, et = desc(inv_s), desc(inv_t)
    e = cfg.patch.ele_n
    pred = ref.Pose(es[:, :, 1:e - 1], et[:, :, 1:e - 1])
    torch.nn.HuberLoss()(pred, torch.from_numpy(gt).double()).backward()
    gold = dict(pred_ind=pred.detach().numpy())        # the inputs are regenerated from the seed of case()
    for k, v in ref.state_dict().items():
        if "running_" in k or "num_batches_tracked" in k:
            gold["state." + k] = v.numpy()
    for k, p in ref.Pose.conv.named_parameters():     # every GRAD_STRIDE-th element and the norm keep the file small
        g = p.grad.numpy().reshape(-1)
        gold["grad." + k] = g[::GRAD_STRIDE]
        gold["gradnorm." + k] = np.array([np.linalg.norm(g)])
    path = os.path.join(ROOT, "tests", "golden", "train_pose_step.npz")
    np.savez_compressed(path, **gold)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "../reference")
