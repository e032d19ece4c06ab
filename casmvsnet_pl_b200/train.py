"""Train CascadeMVSNet on DTU with the engine: the reference's train.py without
pytorch-lightning, test_tube or inplace_abn.

    python -m casmvsnet_pl_b200.train --root_dir DTU/mvs_training/dtu \
        --train_list lists/dtu/train.txt --val_list lists/dtu/val.txt --exp_name exp

Flags keep the names and defaults of the reference's opt.py, plus --precision (fp32 as the
reference, or tf32), the two scan lists and --log_every.  The loop is what Lightning 0.7.5 ran
for the reference's MVSSystem:

  * training steps: forward through the model's autograd path (own K1 / K2 / K3 forward and
    backward kernels), SL1 loss and level-0 metrics from losses.py in one launch pair, backward,
    optimiser step; the scheduler steps once per epoch;
  * every --log_every steps a JSON line (lr, loss, abs_err, acc_1/2/4mm) goes to
    logs/<exp_name>/metrics.jsonl; only then are values read from the device;
  * after every epoch, validation in eval mode under no_grad (the inference engine on the
    trained weights), with the mask-weighted means of train.py:157-163;
  * checkpoints in Lightning's layout, ckpts/<exp_name>/_ckpt_epoch_{e}.ckpt, keeping the 5
    best by val/acc_2mm.

Not supported (the command exits with a message): radam and ranger, --use_amp, more than one
GPU, and the BlendedMVS training set.
"""
from __future__ import annotations

import argparse
import json
import os
import time

import torch
from torch.optim import SGD, Adam
from torch.optim.lr_scheduler import CosineAnnealingLR, LambdaLR, LRScheduler, MultiStepLR

from . import train_data
from .losses import sl1_loss_and_metrics

METRIC_NAMES = ("abs_err", "acc_1mm", "acc_2mm", "acc_4mm")


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--root_dir", type=str, default="/home/ubuntu/data/mvs_training/dtu/",
                    help="root directory of dtu dataset")
    ap.add_argument("--dataset_name", type=str, default="dtu", choices=["dtu", "blendedmvs"])
    ap.add_argument("--train_list", type=str, default=None, help="training scans, one per line")
    ap.add_argument("--val_list", type=str, default=None, help="validation scans, one per line")
    ap.add_argument("--n_views", type=int, default=3)
    ap.add_argument("--levels", type=int, default=3, choices=[3])
    ap.add_argument("--depth_interval", type=float, default=2.65)
    ap.add_argument("--n_depths", nargs="+", type=int, default=[8, 32, 48])
    ap.add_argument("--interval_ratios", nargs="+", type=float, default=[1.0, 2.0, 4.0])
    ap.add_argument("--num_groups", type=int, default=1, choices=[1, 2, 4, 8])
    ap.add_argument("--loss_type", type=str, default="sl1", choices=["sl1"])
    ap.add_argument("--batch_size", type=int, default=1)
    ap.add_argument("--num_epochs", type=int, default=16)
    ap.add_argument("--num_gpus", type=int, default=1)
    ap.add_argument("--ckpt_path", type=str, default="", help="weights to start from")
    ap.add_argument("--prefixes_to_ignore", nargs="+", type=str, default=["loss"])
    ap.add_argument("--optimizer", type=str, default="sgd", choices=["sgd", "adam", "radam", "ranger"])
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--momentum", type=float, default=0.9)
    ap.add_argument("--weight_decay", type=float, default=1e-5)
    ap.add_argument("--lr_scheduler", type=str, default="steplr", choices=["steplr", "cosine", "poly"])
    ap.add_argument("--warmup_multiplier", type=float, default=1.0)
    ap.add_argument("--warmup_epochs", type=int, default=0)
    ap.add_argument("--decay_step", nargs="+", type=int, default=[20])
    ap.add_argument("--decay_gamma", type=float, default=0.1)
    ap.add_argument("--poly_exp", type=float, default=0.9)
    ap.add_argument("--use_amp", default=False, action="store_true")
    ap.add_argument("--exp_name", type=str, default="exp")
    ap.add_argument("--precision", default="fp32", choices=["fp32", "tf32"],
                    help="fp32 (as the reference) or tf32 tensor-core convolutions")
    ap.add_argument("--log_every", type=int, default=10, help="steps between JSON log lines")
    ap.add_argument("--num_workers", type=int, default=4, help="host data-loader workers")
    return ap


def check_supported(a):
    """SystemExit with a message for what this trainer does not do."""
    if a.optimizer in ("radam", "ranger"):
        raise SystemExit(f"--optimizer {a.optimizer} is not supported: use sgd or adam")
    if a.use_amp:
        raise SystemExit("--use_amp is not supported: train in fp32 or --precision tf32")
    if a.num_gpus != 1:
        raise SystemExit("--num_gpus must be 1: multi-GPU training is not supported")
    if a.dataset_name != "dtu":
        raise SystemExit("only --dataset_name dtu can be trained")
    if not a.train_list or not a.val_list:
        raise SystemExit("--train_list and --val_list are required")


# ------------------------------------------------------------------ optimiser and schedulers
def get_optimizer(a, model):
    """utils/__init__.py get_optimizer for sgd and adam (eps 1e-8 without AMP)."""
    if a.optimizer == "sgd":
        return SGD(model.parameters(), lr=a.lr, momentum=a.momentum, weight_decay=a.weight_decay)
    if a.optimizer == "adam":
        return Adam(model.parameters(), lr=a.lr, eps=1e-8, weight_decay=a.weight_decay)
    raise ValueError(f"optimizer {a.optimizer!r} not supported")


class GradualWarmupScheduler(LRScheduler):
    """Warm-up of Goyal et al., 'Accurate, Large Minibatch SGD' (the reference's
    utils/warmup_scheduler.py): the lr rises linearly from lr to lr * multiplier over
    `total_epoch` epochs.  At the first epoch past that, `after` is given lr * multiplier as its
    base and its own lr rule (at its epoch 0) decides that epoch's value; from then on only
    `after` is stepped."""

    def __init__(self, optimizer, multiplier, total_epoch, after):
        if multiplier < 1.0:
            raise ValueError("multiplier should be >= 1")
        self.multiplier, self.total_epoch, self.after = multiplier, total_epoch, after
        self.finished = False
        super().__init__(optimizer)

    def get_lr(self):
        if self.last_epoch <= self.total_epoch:
            frac = self.last_epoch / self.total_epoch
            return [b * ((self.multiplier - 1.0) * frac + 1.0) for b in self.base_lrs]
        if not self.finished:
            self.after.base_lrs = [b * self.multiplier for b in self.base_lrs]
            self.finished = True
        return self.after.get_lr()

    def step(self, epoch=None):
        if self.finished:
            self.after.step(None if epoch is None else epoch - self.total_epoch)
        else:
            super().step(epoch)


def get_scheduler(a, optimizer):
    """utils/__init__.py get_scheduler: steplr, cosine (eta_min 1e-8), poly, with the gradual
    warm-up when --warmup_epochs > 0."""
    if a.lr_scheduler == "steplr":
        s = MultiStepLR(optimizer, milestones=a.decay_step, gamma=a.decay_gamma)
    elif a.lr_scheduler == "cosine":
        s = CosineAnnealingLR(optimizer, T_max=a.num_epochs, eta_min=1e-8)
    elif a.lr_scheduler == "poly":
        s = LambdaLR(optimizer, lambda epoch: (1 - epoch / a.num_epochs) ** a.poly_exp)
    else:
        raise ValueError(f"scheduler {a.lr_scheduler!r} not recognized")
    if a.warmup_epochs > 0:
        s = GradualWarmupScheduler(optimizer, a.warmup_multiplier, a.warmup_epochs, s)
    return s


def get_learning_rate(optimizer):
    return optimizer.param_groups[0]["lr"]


# ------------------------------------------------------------------ checkpoints
def extract_model_state_dict(ckpt_path, prefixes_to_ignore=()):
    """Model weights of a Lightning checkpoint ('model.'-prefixed keys of 'state_dict') or of a
    plain state dict, without the keys that start with one of `prefixes_to_ignore`."""
    ckpt = torch.load(ckpt_path, map_location="cpu")
    if "state_dict" in ckpt:
        sd = {k[len("model."):]: v for k, v in ckpt["state_dict"].items() if k.startswith("model.")}
    else:
        sd = dict(ckpt)
    return {k: v for k, v in sd.items() if not any(k.startswith(p) for p in prefixes_to_ignore)}


def load_ckpt(model, ckpt_path, prefixes_to_ignore=()):
    """Weights-only warm start: the checkpoint's tensors over the model's own."""
    sd = model.state_dict()
    sd.update(extract_model_state_dict(ckpt_path, prefixes_to_ignore))
    model.load_state_dict(sd)


def save_checkpoint(model, path, epoch, global_step):
    """Lightning's layout: {'state_dict': {'model.<key>': tensor}, 'epoch', 'global_step'}."""
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    sd = {"model." + k: v.detach().cpu() for k, v in model.state_dict().items()}
    torch.save({"state_dict": sd, "epoch": epoch, "global_step": global_step}, path)


class TopKCheckpoints:
    """ModelCheckpoint(monitor, mode='max', save_top_k=k): keep the k best epochs' files."""

    def __init__(self, directory, k=5):
        self.directory, self.k, self.kept = directory, k, {}

    def __call__(self, model, epoch, global_step, score):
        path = os.path.join(self.directory, f"_ckpt_epoch_{epoch}.ckpt")
        if score != score:                                  # NaN never ranks
            return None
        if len(self.kept) >= self.k:
            worst = min(self.kept, key=self.kept.get)
            if score <= self.kept[worst]:
                return None
            os.remove(worst)
            del self.kept[worst]
        save_checkpoint(model, path, epoch, global_step)
        self.kept[path] = score
        return path


# ------------------------------------------------------------------ the loop
def build_model(a, device):
    from . import InPlaceABN
    from .models.mvsnet import CascadeMVSNet
    model = CascadeMVSNet(n_depths=a.n_depths, interval_ratios=a.interval_ratios,
                          num_groups=a.num_groups, norm_act=InPlaceABN, precision=a.precision)
    if a.ckpt_path:
        load_ckpt(model, a.ckpt_path, a.prefixes_to_ignore)
    return model.to(device).train()


class Trainer:
    def __init__(self, a, model, device="cuda:0"):
        self.a, self.model, self.device = a, model, device
        self.optimizer = get_optimizer(a, model)
        self.scheduler = get_scheduler(a, self.optimizer)
        self.global_step = 0

    def forward(self, s):
        return self.model(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])

    def train_step(self, s):
        """One optimiser step on a device sample -> (loss, metrics) device tensors."""
        self.model.train()
        results = self.forward(s)
        loss, metrics = sl1_loss_and_metrics(results, s["depths"], s["masks"], self.a.levels)
        self.optimizer.zero_grad(set_to_none=True)
        loss.backward()
        self.optimizer.step()
        self.global_step += 1
        return loss.detach(), metrics

    @torch.no_grad()
    def validate(self, batches):
        """Mean val loss and mask-weighted level-0 metrics over `batches` (train.py:129-173)."""
        self.model.eval()
        loss_sum = torch.zeros((), device=self.device, dtype=torch.float64)
        msum = torch.zeros(5, device=self.device, dtype=torch.float64)
        n = 0
        for batch in batches:
            s = train_data.to_device(batch, self.device)
            loss, metrics = sl1_loss_and_metrics(self.forward(s), s["depths"], s["masks"], self.a.levels)
            loss_sum += loss
            msum += metrics
            n += 1
        self.model.train()
        vals = (torch.cat([(loss_sum / n).view(1), msum[:4] / msum[4]])).tolist()
        return {"val/loss": vals[0], **{f"val/{k}": v for k, v in zip(METRIC_NAMES, vals[1:])}}

    def fit(self, train_loader, val_loader, log_path, ckpt_dir):
        a = self.a
        os.makedirs(os.path.dirname(log_path) or ".", exist_ok=True)
        keep = TopKCheckpoints(ckpt_dir, 5)
        with open(log_path, "a") as log:
            for epoch in range(a.num_epochs):
                for batch in train_loader:
                    lr = get_learning_rate(self.optimizer)
                    loss, m = self.train_step(train_data.to_device(batch, self.device))
                    if self.global_step % a.log_every == 0 or self.global_step == 1:
                        vals = torch.cat([loss.view(1), m[:4] / m[4]]).tolist()
                        rec = {"epoch": epoch, "step": self.global_step, "lr": lr, "train/loss": vals[0]}
                        rec.update({f"train/{k}": v for k, v in zip(METRIC_NAMES, vals[1:])})
                        log.write(json.dumps(rec) + "\n")
                        log.flush()
                val = self.validate(val_loader)
                path = keep(self.model, epoch, self.global_step, val["val/acc_2mm"])
                log.write(json.dumps({"epoch": epoch, "step": self.global_step, **val,
                                      "checkpoint": path}) + "\n")
                log.flush()
                print(f"epoch {epoch}: " + ", ".join(f"{k} {v:.4f}" for k, v in val.items()))
                self.scheduler.step()
        return keep.kept


def main(argv=None):
    a = build_parser().parse_args(argv)
    check_supported(a)
    if not torch.cuda.is_available():
        raise SystemExit("training needs a CUDA GPU")
    device = "cuda:0"
    train_set = train_data.DTUTrainDataset(a.root_dir, train_data.read_scan_list(a.train_list),
                                           a.n_views, a.levels, a.depth_interval)
    val_set = train_data.DTUTrainDataset(a.root_dir, train_data.read_scan_list(a.val_list),
                                         a.n_views, a.levels, a.depth_interval)
    model = build_model(a, device)
    print("number of parameters : %.2f M" % (sum(p.numel() for p in model.parameters()
                                                  if p.requires_grad) / 1e6))
    trainer = Trainer(a, model, device)
    t0 = time.time()
    kept = trainer.fit(train_data.loader(train_set, a.batch_size, True, a.num_workers),
                       train_data.loader(val_set, a.batch_size, False, a.num_workers),
                       os.path.join("logs", a.exp_name, "metrics.jsonl"),
                       os.path.join("ckpts", a.exp_name))
    print(f"trained {trainer.global_step} steps in {time.time() - t0:.1f} s; "
          f"kept {sorted(kept)}")


if __name__ == "__main__":
    main()
