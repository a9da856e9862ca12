"""CPU: the float64 oracle of the Desc training step (oracle/train_desc.py, with train_stages._contrastive as the
contrastive loss) against the reference's own modules in training mode (tests/golden/train_desc_step.npz, written by
tests/tools/gen_train_desc_golden.py): desc, equi, equi_score, the loss, every descriptor running statistic after the
source and target calls, and the gradients of every Desc parameter, to float64 rounding (1e-12 relative)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "tools"))


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "train_desc_step.npz"))


def _close(got, ref, what, rtol=1e-12):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, what
    assert np.abs(got - ref).max() <= rtol * max(np.abs(ref).max(), 1e-300), what


def test_oracle_reproduces_reference_modules_in_training_mode(gold):
    from oracle import train_desc as TD
    from oracle.train_step import bn_hparams, state64
    import gen_train_desc_golden as G
    import bufferx_b200 as bx
    cfg, sd, inv_s, inv_t, kpt, label = G.case()
    d = np.linalg.norm(kpt[:, None] - kpt[None], axis=-1)
    assert ((d < 0.10) & ~np.eye(len(kpt), dtype=bool)).any(), "no pair inside the safe radius: its mask is untested"
    hp = {k: v for k, v in bn_hparams(bx.BufferX(cfg)).items() if k.startswith("Desc.")}
    params, st, stats = TD.desc_params(sd), state64(sd), []
    ds, es = TD.desc_train(inv_s, params, st, stats, hp)
    dt, et = TD.desc_train(inv_t, params, st, stats, hp)
    score = TD.equi_match(es, et)
    loss = TD.desc_loss(ds, dt, kpt.astype(np.float64), score, label)
    _close(ds.detach(), gold["src_desc"], "src desc")
    _close(dt.detach(), gold["tgt_desc"], "tgt desc")
    _close(es.detach().reshape(-1)[::G.EQUI_STRIDE], gold["src_equi"], "src equi")
    _close(et.detach().reshape(-1)[::G.EQUI_STRIDE], gold["tgt_equi"], "tgt equi")
    _close(score.detach(), gold["equi_score"], "equi_score")
    _close([loss.item()], gold["loss"], "loss")
    loss.backward()
    n = 0
    for k in gold.files:
        if not k.startswith("state."):
            continue
        key = k[len("state."):]
        if "num_batches_tracked" in key:
            assert int(st[key]) == int(gold[k]) == int(sd[key]) + 2, key
        else:
            _close(st[key].numpy(), gold[k], key)
        n += 1
    assert n == 3 * 10                                   # the ten descriptor BatchNorms
    assert set(params) == {k[len("gradnorm."):] for k in gold.files if k.startswith("gradnorm.")}
    # the biases of the convolutions ahead of a BatchNorm have an analytically zero gradient: both sides hold rounding
    # noise there, held to 1e-12 of the largest gradient norm
    scale = max(float(gold[k][0]) for k in gold.files if k.startswith("gradnorm."))
    for k, p in params.items():
        g = p.grad.numpy().reshape(-1)
        norm = float(gold["gradnorm." + k][0])
        lim = 1e-10 * norm + 1e-12 * scale
        assert abs(np.linalg.norm(g) - norm) <= lim, k
        assert np.abs(g[::G.GRAD_STRIDE] - gold["grad." + k]).max() <= lim, k


def test_oracle_contrastive_loss_is_the_references_safe_radius_mask(gold):
    """A mutation check of the pin: without the safe-radius mask the oracle's loss leaves the golden's."""
    from oracle import train_stages as TS
    import gen_train_desc_golden as G
    _, _, _, _, kpt, _ = G.case()
    s, t = torch.from_numpy(gold["src_desc"]), torch.from_numpy(gold["tgt_desc"])
    k = torch.from_numpy(kpt.astype(np.float64))
    with_mask, _ = TS._contrastive(s, t, k)
    without, _ = TS._contrastive(s, t, k, safe_radius=0.0)
    ref = float(gold["desc_loss"][0])
    assert abs(float(with_mask) - ref) <= 1e-12 * abs(ref)
    assert abs(float(without) - ref) > 1e-6 * abs(ref)
