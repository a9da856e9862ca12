"""Train BUFFER-X on every GPU of a box: the reference's ``train.py`` with ``Trainer.train`` replaced by
``bufferx_b200.driver.train_sharded`` (DESIGN.md §8), one process per GPU.  Run it from inside a reference checkout:

    cd /path/to/BUFFER-X
    PYTHONPATH=/path/to/bufferx-b200/dropin:/path/to/bufferx-b200/buffer-x_b200:/path/to/bufferx-b200:$PYTHONPATH \\
        torchrun --standalone --nproc_per_node=<GPUs> /path/to/bufferx-b200/tools/train_sharded.py --dataset 3DMatch

What it keeps from train.py / trainer.py: the arguments, the seed (cfg.data.manual_seed), the stages of
cfg.train.all_stage in order, pretrain_model and the other stage's best.pth loaded and frozen (Args, train.py:28-48),
Adam at cfg.optim.lr[stage] with cfg.optim.weight_decay, ExponentialLR(cfg.optim.lr_decay) every
cfg.optim.scheduler_interval[stage] epochs, the datasets and collate of get_dataloader, the losses of trainer.py:113-141
(training) and 187-207 (validation) built from the checkout's loss.desc_loss and torch.nn, and the snapshots under
snapshot/{dataset}/{experiment_id}/{stage}/ that test.py loads.  Rank 0 picks the experiment id and every rank uses it.
Not kept: the tensorboard writer.  Without torchrun (no WORLD_SIZE) it trains alone on cuda:0.
"""
import argparse
import copy
import datetime
import os
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

TIMEOUT = datetime.timedelta(minutes=30)      # a rank that dies makes the others raise after this, instead of hanging


def make_losses(stage):
    """(train_loss, eval_stats) of trainer.py for ``stage``, from the checkout's loss.desc_loss and torch.nn."""
    from loss.desc_loss import ContrastiveLoss, cdist
    desc_loss_fn, class_loss, huber = ContrastiveLoss(), torch.nn.CrossEntropyLoss(), torch.nn.HuberLoss()

    def desc(out, kpt):
        desc_loss, _, accuracy = desc_loss_fn(out["src_des"], out["tgt_des"], cdist(out[kpt], out[kpt]))
        eqv_loss = class_loss(out["equi_score"], out["gt_label"])
        pre_label = torch.argmax(out["equi_score"], dim=1)
        eqv_acc = (pre_label == out["gt_label"]).sum() / pre_label.shape[0]
        stats = {"desc_loss": float(desc_loss.item()), "desc_acc": float(accuracy.item()),
                 "eqv_loss": float(eqv_loss.item()), "eqv_acc": float(eqv_acc.item())}
        return 4 * desc_loss + eqv_loss, stats

    def pose(out):
        match_loss = huber(out["pred_ind"], out["gt_ind"])
        return match_loss, {"match_loss": float(match_loss.item())}

    if stage == "Desc":
        return (lambda out: desc(out, "tgt_kpt")), (lambda out: desc(out, "src_kpt")[1])
    if stage == "Pose":
        return pose, (lambda out: pose(out)[1])
    raise NotImplementedError(stage)


def main(argv=None, checkout=None, train=None):
    """train.py's __main__ over every rank.  ``checkout``: the reference checkout (default: the working directory);
    ``train``: the training loop (default: driver.train_sharded)."""
    parser = argparse.ArgumentParser(description="Generalized Training Script for Registration Models, on every GPU of a box")
    parser.add_argument("--dataset", type=str, required=True, choices=["3DMatch", "KITTI"], help="Dataset to train on (3DMatch or KITTI)")
    parser.add_argument("--root_dir", type=str, default="../datasets", help="Root directory for all datasets")
    args = parser.parse_args(argv)
    checkout = os.path.abspath(checkout or os.getcwd())
    if sys.path[0] != checkout:
        sys.path.insert(0, checkout)         # as `python train.py` puts its own directory first: config, dataset, loss, utils
    import torch.distributed as dist
    from config import make_cfg
    from dataset.dataloader import get_dataloader
    from utils.tools import setup_logger

    from bufferx_b200 import BufferX, driver
    train = train or driver.train_sharded

    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl" if torch.cuda.is_available() else "gloo", timeout=TIMEOUT)
    rank = dist.get_rank() if dist.is_initialized() else 0
    local = int(os.environ.get("LOCAL_RANK", "0"))
    device = torch.device("cuda", local) if torch.cuda.is_available() else torch.device("cpu")
    if device.type == "cuda":
        torch.cuda.set_device(device)

    timestr = time.strftime("%m%d%H%M")
    if rank == 0:
        log_dir = os.path.join(checkout, f"logs/train/{args.dataset}")
        os.makedirs(log_dir, exist_ok=True)
        logger = setup_logger(os.path.join(log_dir, f"{timestr}.log"))
        logger.info(f"Starting training on {args.dataset} over {dist.get_world_size() if dist.is_initialized() else 1} ranks...")
    cfg = make_cfg(args.dataset, root_dir=args.root_dir)
    cfg[cfg.data.dataset] = cfg.copy()
    cfg.stage = "train"
    experiment_id = cfg.train.pretrain_model.split("/")[1] if cfg.train.pretrain_model else timestr
    if dist.is_initialized():
        box = [experiment_id]
        dist.broadcast_object_list(box, 0)
        experiment_id = box[0]
    seed = cfg.data.manual_seed if cfg.data.manual_seed is not None else 0
    results = {}
    for stage in cfg.train.all_stage:
        cfg.stage = stage
        cfg.snapshot_root = os.path.join(checkout, f"snapshot/{args.dataset}/{experiment_id}")
        model = BufferX(cfg)
        parameter = model.get_parameter()
        left_stage = copy.deepcopy(cfg.train.all_stage)
        left_stage.remove(cfg.stage)
        if cfg.train.pretrain_model:
            model.load_state_dict(torch.load(cfg.train.pretrain_model, map_location="cpu"))
        for modname in left_stage:
            weight_path = os.path.join(cfg.snapshot_root, modname, "best.pth")
            if os.path.exists(weight_path):
                state_dict = torch.load(weight_path, map_location="cpu")
                model_dict = model.state_dict()
                model_dict.update({k: v for k, v in state_dict.items() if modname in k})
                model.load_state_dict(model_dict)
                if rank == 0:
                    logger.info(f"Loaded {modname} from {weight_path}")
            for p in getattr(model, modname).parameters():
                p.requires_grad = False
        optimizer = torch.optim.Adam(parameter, lr=cfg.optim.lr[cfg.stage], weight_decay=cfg.optim.weight_decay)
        scheduler = torch.optim.lr_scheduler.ExponentialLR(optimizer, gamma=cfg.optim.lr_decay)
        model = model.to(device)
        train_loader = get_dataloader(dataset=cfg.data.dataset, split="train", config=cfg, shuffle=True, num_workers=cfg.train.num_workers)
        val_loader = get_dataloader(dataset=cfg.data.dataset, split="val", config=cfg, shuffle=False, num_workers=cfg.train.num_workers)
        if rank == 0:
            logger.info(f"Training set size: {len(train_loader.dataset)}")
            logger.info(f"Validation set size: {len(val_loader.dataset)}")
        train_loss, eval_stats = make_losses(stage)
        results[stage] = train(model, optimizer, scheduler, train_loader.dataset, val_loader.dataset, cfg, train_loss, eval_stats,
                               collate=train_loader.collate_fn, seed=seed, snapshot_root=cfg.snapshot_root,
                               num_workers=cfg.train.num_workers, log=logger.info if rank == 0 else None)
    if dist.is_initialized():
        dist.destroy_process_group()
    return results


if __name__ == "__main__":
    main()
