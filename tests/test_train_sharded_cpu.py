"""CPU: the host side of sharded training (DESIGN.md §8): the epoch sampler, the contribution protocol of one step under
gloo with two ranks (the cross-rank mean replaced by its float64 restatement; a stub model stands in for BufferX), and
tools/train_sharded.py against a stub reference checkout."""
import copy
import os
import sys
import textwrap

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def dp_mean_f64(g):
    """ops.dp_mean restated in torch float64: the contributing rows summed in rank order from the first, divided, .float()."""
    rows = g[g[:, -1] != 0, :-1].double()
    count = torch.tensor([rows.shape[0]], dtype=torch.int32)
    if rows.shape[0] == 0:
        return torch.empty(g.shape[1] - 1), count
    s = rows[0].clone()
    for r in rows[1:]:
        s = s + r
    return (s / rows.shape[0]).float(), count


# --------------------------------------------------------------------------- sampler
def test_epoch_shard_partitions_each_epoch():
    from bufferx_b200.driver import epoch_shard
    for n, world in [(10, 1), (10, 3), (7, 2), (5, 3), (2, 4), (0, 2)]:
        for epoch in range(3):
            shards = [epoch_shard(n, r, world, epoch, 123, 10 ** 6) for r in range(world)]
            assert len({len(s) for s in shards}) == 1 and len(shards[0]) == -(-n // world)     # equal step counts
            got = [i for s in zip(*shards) for i in s if i is not None]
            assert sorted(got) == list(range(n))                                             # each index once
            assert got == np.random.RandomState(123 + epoch).permutation(n).tolist()          # one permutation, rank-major
            idle = [s.count(None) for s in shards]
            assert sum(idle) == -(-n // world) * world - n and all(s[:-1].count(None) == 0 for s in shards)
    a, b = epoch_shard(50, 0, 2, 0, 1, 100), epoch_shard(50, 0, 2, 1, 1, 100)
    assert a != b                                                                           # a new permutation per epoch
    st = np.random.get_state()[1].copy()
    assert epoch_shard(50, 1, 2, 0, 1, 7) == epoch_shard(50, 1, 2, 0, 1, 100)[:7]            # the max_iter cap
    assert (np.random.get_state()[1] == st).all()                                           # the global RNG is untouched


# --------------------------------------------------------------------------- the contribution protocol
class _Stub(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(3, 4)
        self.bn = torch.nn.BatchNorm1d(4)
        self.head = torch.nn.Linear(4, 2)
        self.frozen = torch.nn.Linear(2, 2)
        self.frozen.requires_grad_(False)

    def forward(self, d):
        y = self.head(torch.relu(self.bn(self.lin(d["x"]))))      # the BatchNorm moves its running statistics first
        return None if d.get("none") else y


def _loss(out):
    loss = (out ** 2).mean() + out[:, 0].sum()
    if not torch.isfinite(out).all() or out.shape[0] == 7:          # a 7-row batch carries a non-finite loss
        loss = loss * float("inf")
    return loss, {"match_loss": float(loss.item())}


def _script():
    """Per step, what ranks 0 and 1 get: both a pair; rank 1's forward returns None; rank 1 idle; nobody contributes;
    rank 1's loss is non-finite."""
    g = torch.Generator().manual_seed(5)
    x = lambda n=6: torch.randn((n, 3), generator=g)   # noqa: E731
    return [[dict(x=x()), dict(x=x())], [dict(x=x()), dict(x=x(), none=True)], [dict(x=x()), None],
            [dict(x=x(), none=True), dict(x=x(), none=True)], [dict(x=x()), dict(x=x(7))]]


def _state(model, opt):
    return dict(model={k: v.clone() for k, v in model.state_dict().items()},
                adam={k: {n: t.clone() if isinstance(t, torch.Tensor) else t for n, t in s.items()} for k, s in opt.state_dict()["state"].items()})


def _protocol_worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from bufferx_b200.driver import train_step
    torch.manual_seed(rank)                                   # different start states ...
    model = _Stub()
    from bufferx_b200.driver import _broadcast_state
    _broadcast_state(model)                                   # ... until rank 0's is broadcast
    model.train()
    opt = torch.optim.Adam([p for p in model.parameters()], lr=0.05, weight_decay=1e-2)
    rec = []
    for step in _script():
        count, stepped, _ = train_step(model, opt, step[rank], _loss, mean_fn=dp_mean_f64)
        rec.append(dict(count=count, stepped=stepped, **_state(model, opt)))
    torch.save(rec, os.path.join(out, f"rank{rank}.pt"))
    dist.destroy_process_group()


def _bits_equal(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_bits_equal(a[k], b[k]) for k in a)
    if isinstance(a, torch.Tensor):
        return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(-1).view(torch.uint8) if a.numel() else a,
                                                                          b.view(-1).view(torch.uint8) if b.numel() else b)
    return a == b


def test_contribution_protocol_gloo_world2(tmp_path):
    mp.spawn(_protocol_worker, args=(2, 29531, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(str(tmp_path / f"rank{r}.pt"), weights_only=False) for r in range(2))
    assert [s["count"] for s in r0] == [2, 1, 1, 0, 2] and [s["stepped"] for s in r0] == [True, True, True, False, False]
    for a, b in zip(r0, r1):
        assert _bits_equal(a, b)                              # every rank holds the same bits after every step
    # single-process emulation: each rank's pair from the common pre-step state, combined in float64 in rank order
    torch.manual_seed(0)
    master = _Stub()
    master.train()
    opt = torch.optim.Adam([p for p in master.parameters()], lr=0.05, weight_decay=1e-2)
    params = [p for p in master.parameters() if p.requires_grad]
    bufs = [master.bn.running_mean, master.bn.running_var, master.bn.num_batches_tracked]
    for step, want in zip(_script(), r0):
        grads, stats = [], []
        for d in step:
            m = copy.deepcopy(master)
            out = m(d) if d is not None else None
            if out is None:
                continue
            _loss(out)[0].backward()
            grads.append([p.grad.double() for p in m.parameters() if p.requires_grad])
            stats.append([m.bn.running_mean.double(), m.bn.running_var.double(), m.bn.num_batches_tracked.double()])
        opt.zero_grad()
        if grads:
            def mean(rows):
                s = rows[0]
                for r in rows[1:]:
                    s = s + r
                return s / len(rows)
            for i, p in enumerate(params):
                p.grad = mean([g[i] for g in grads]).float()
            with torch.no_grad():
                for i, b in enumerate(bufs):
                    b.copy_(mean([s[i] for s in stats]).to(b.dtype))
            if all(torch.isfinite(p.grad).all() for p in params):
                opt.step()
        assert _bits_equal(_state(master, opt), {k: want[k] for k in ("model", "adam")})


# --------------------------------------------------------------------------- the entry point against a stub checkout
STUB = {
    "config/__init__.py": """
        from bufferx_b200.config import make_cfg as _make_cfg
        def make_cfg(dataset, root_dir=None):
            cfg = _make_cfg(dataset, root_dir)
            cfg.optim.lr = {"Desc": 0.003, "Pose": 0.002}
            cfg.optim.weight_decay, cfg.optim.lr_decay = 2e-6, 0.25
            return cfg
        """,
    "dataset/__init__.py": "",
    "dataset/dataloader.py": """
        class _Loader:
            def __init__(self, split):
                self.dataset = [dict(split=split, i=i) for i in range(3 if split == "train" else 2)]
                self.collate_fn = lambda batch: ("collated", batch)
        CALLS = []
        def get_dataloader(dataset, split, config, num_workers=16, shuffle=True, drop_last=True):
            CALLS.append((dataset, split, config.stage, shuffle, num_workers))
            return _Loader(split)
        """,
    "loss/__init__.py": "",
    "loss/desc_loss.py": """
        import torch
        class ContrastiveLoss(torch.nn.Module):
            def forward(self, a, p, d):
                return (a - p).abs().sum() + 0 * d.sum(), None, torch.tensor(0.5)
        def cdist(a, b):
            return torch.cdist(a, b)
        """,
    "utils/tools.py": """
        import logging
        def setup_logger(path):
            return logging.getLogger("stub_train_sharded")
        """,
}


def test_entry_point_against_stub_checkout(tmp_path, monkeypatch):
    for rel, src in STUB.items():
        p = tmp_path / "ref" / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(src))
    checkout = str(tmp_path / "ref")
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k.split(".")[0] in ("config", "dataset", "loss", "utils")}
    seen = []

    def fake_train(model, optimizer, scheduler, train_set, val_set, cfg, train_loss, eval_stats, collate=None, seed=None,
                   snapshot_root=None, num_workers=0, log=None):
        stage = cfg.stage
        frozen = "Pose" if stage == "Desc" else "Desc"
        g = optimizer.param_groups[0]
        seen.append(dict(stage=stage, snapshot_root=snapshot_root, seed=seed, lr=g["lr"], wd=g["weight_decay"], gamma=scheduler.gamma,
                         n_opt=len(g["params"]), trainable=all(p.requires_grad for p in getattr(model, stage).parameters()),
                         frozen=not any(p.requires_grad for p in getattr(model, frozen).parameters()),
                         collate=collate([1]), sets=(len(train_set), len(val_set)),
                         first=getattr(model, frozen).state_dict()[next(iter(getattr(model, frozen).state_dict()))].clone()))
        out = dict(src_des=torch.ones(3, 4), tgt_des=torch.zeros(3, 4), src_kpt=torch.zeros(3, 3), tgt_kpt=torch.zeros(3, 3),
                   equi_score=torch.zeros(3, 5), gt_label=torch.zeros(3, dtype=torch.long),
                   pred_ind=torch.tensor([1.0, 2.0]), gt_ind=torch.tensor([1.0, 4.0]))
        loss, stats = train_loss(out)
        seen[-1].update(loss=float(loss), eval=eval_stats(out))
        os.makedirs(os.path.join(snapshot_root, stage), exist_ok=True)
        sd = model.state_dict()
        for k in sd:
            if k.startswith(stage) and sd[k].is_floating_point():
                sd[k] = torch.full_like(sd[k], 0.5)
        torch.save(sd, os.path.join(snapshot_root, stage, "best.pth"))
        return [stats]

    try:
        import train_sharded as TS
        res = TS.main(["--dataset", "3DMatch", "--root_dir", str(tmp_path / "data")], checkout=checkout, train=fake_train)
        from dataset.dataloader import CALLS
    finally:
        for k in [k for k in sys.modules if k.split(".")[0] in ("config", "dataset", "loss", "utils")]:
            del sys.modules[k]
        sys.modules.update(saved)
        sys.path.remove(os.path.join(ROOT, "tools"))
    assert [s["stage"] for s in seen] == ["Desc", "Pose"] and list(res) == ["Desc", "Pose"]
    d, p = seen
    root = d["snapshot_root"]
    assert root == p["snapshot_root"] and os.path.dirname(root) == os.path.join(checkout, "snapshot", "3DMatch")
    assert (d["lr"], d["wd"], d["gamma"]) == (0.003, 2e-6, 0.25) and (p["lr"], p["wd"], p["gamma"]) == (0.002, 2e-6, 0.25)
    assert d["seed"] == p["seed"] == 123                                                  # cfg.data.manual_seed
    assert d["trainable"] and d["frozen"] and p["trainable"] and p["frozen"]
    assert d["n_opt"] == p["n_opt"] == 48                                                 # get_parameter(): every parameter
    assert d["collate"] == ("collated", [1]) and d["sets"] == (3, 2)
    assert not (d["first"] == 0.5).all() and (p["first"] == 0.5).all()     # the Pose stage loaded Desc from Desc/best.pth
    assert CALLS == [("3DMatch", "train", "Desc", True, 0), ("3DMatch", "val", "Desc", False, 0),
                     ("3DMatch", "train", "Pose", True, 0), ("3DMatch", "val", "Pose", False, 0)]
    assert abs(d["loss"] - (4 * 12.0 + np.log(5))) < 1e-5 and abs(d["eval"]["desc_loss"] - 12.0) < 1e-6
    assert abs(p["loss"] - 0.75) < 1e-6 and p["eval"] == {"match_loss": p["loss"]}         # HuberLoss: (0 + 1.5) / 2
