"""Regenerate tests/golden/train_desc_step.npz: the reference's own modules in training mode, in float64, on one small
synthetic Desc step.

    python tests/tools/gen_train_desc_golden.py /path/to/reference/checkout

Builds the unmodified reference ``BufferX`` (third-party leaves stubbed as oracle/ref_check.py does), loads the synthetic
C1 state_dict, casts it to float64, calls ``model.train()`` and freezes ``Pose`` (train.py:36-48).  Then, on stored
de-rotated point-layer inputs of a source and a target call (K patches each), it runs the reference's own
``Desc.pnt_layer`` + max, ``Desc.conv_net`` (Cylindrical_Net), ``Desc.pool_layer``, the average pooling and both
``F.normalize`` in patch_embedder.py's order (:81-90), source first, then target, and the trainer's Desc loss
(trainer.py:113-124): 4 ``loss.desc_loss.ContrastiveLoss()(src, tgt, cdist(kpt, kpt))[0]`` + CrossEntropy of
``models.BUFFERX.EquiMatch`` against stored labels, then backward.  Stored: desc, every EQUI_STRIDE-th element of equi, equi_score, the loss, every
running statistic and num_batches_tracked afterwards, and of the gradient of every ``Desc`` parameter its norm and every
GRAD_STRIDE-th element.  The zip entries carry a fixed timestamp, so a rerun writes the same bytes.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_check  # noqa: E402

K = 6
GRAD_STRIDE = 13
EQUI_STRIDE = 7


def case():
    """-> (cfg, state_dict, inv_s, inv_t, kpt, label): C1 synthetic weights, point-layer inputs of K patches with zero
    slots (as SPT leaves them), a duplicated sample in every voxel and an all-zero source patch; key-points spread so that
    some pairs fall inside ContrastiveLoss's 0.1 safe radius; labels in [0, 20)."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    cfg = workload_cfg("C1")
    cfg.stage = "Desc"
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    rng = np.random.RandomState(23)
    inv = (rng.standard_normal((2, K, 420, 10, 3)) * 0.3).astype(np.float32)
    inv[rng.uniform(size=(2, K, 420, 10)) < 0.25] = 0.0
    inv[:, :, :, 8:] = 0.0                                   # zero slots
    inv[:, :, :, 1] = inv[:, :, :, 0]                        # a duplicated sample
    inv[0, 0] = 0.0                                          # an all-zero patch
    kpt = (rng.standard_normal((K, 3)) * 0.08).astype(np.float32)
    label = rng.randint(0, 20, K).astype(np.int64)
    return cfg, sd, inv[0], inv[1], kpt, label


def main(ref_root):
    ref_check.install_stubs(0)
    if ref_root not in sys.path:
        sys.path.insert(0, ref_root)
    for m in [k for k in sys.modules if k in ("models", "utils", "loss") or k.startswith(("models.", "utils.", "loss."))]:
        del sys.modules[m]
    import models.BUFFERX as RB
    from loss import desc_loss as RL
    cfg, sd, inv_s, inv_t, kpt, label = case()
    ref = RB.BufferX(cfg)
    ref.load_state_dict(sd, strict=True)
    ref = ref.double()
    ref.train()
    for p in ref.Pose.parameters():
        p.requires_grad = False
    D = ref.Desc

    def desc(inv):                                           # patch_embedder.py:81-90
        x = D.pnt_layer(torch.from_numpy(inv).double().permute(0, 3, 1, 2))
        x = F.max_pool2d(x, kernel_size=(1, x.shape[-1])).squeeze(3)
        x = x.view(x.shape[0], x.shape[1], D.rad_n, D.ele_n, D.azi_n)
        x, _ = D.conv_net(x)
        w = D.pool_layer(x)
        f = F.avg_pool2d(x * w, kernel_size=(x.shape[2], x.shape[3]))
        return F.normalize(f.view(f.shape[0], -1), p=2, dim=1), F.normalize(x, p=2, dim=1)

    ds, es = desc(inv_s)
    dt, et = desc(inv_t)
    score = RB.EquiMatch(cfg)(es, et)
    k = torch.from_numpy(kpt).double()
    dl = RL.ContrastiveLoss()(ds, dt, RL.cdist(k, k))[0]
    loss = 4 * dl + torch.nn.CrossEntropyLoss()(score, torch.from_numpy(label))
    loss.backward()
    gold = dict(src_desc=ds.detach().numpy(), tgt_desc=dt.detach().numpy(), src_equi=es.detach().numpy().reshape(-1)[::EQUI_STRIDE],
                tgt_equi=et.detach().numpy().reshape(-1)[::EQUI_STRIDE], equi_score=score.detach().numpy(), loss=np.array([loss.item()]),
                desc_loss=np.array([dl.item()]))
    for key, v in ref.state_dict().items():
        if key.startswith("Desc.") and ("running_" in key or "num_batches_tracked" in key):
            gold["state." + key] = v.numpy()
    for key, p in D.named_parameters():                      # every GRAD_STRIDE-th element and the norm keep the file small
        g = p.grad.numpy().reshape(-1)
        gold["grad." + key] = g[::GRAD_STRIDE]
        gold["gradnorm." + key] = np.array([np.linalg.norm(g)])
    path = os.path.join(ROOT, "tests", "golden", "train_desc_step.npz")
    ref_check._savez(path, **gold)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "../reference")
