"""Train CascadeMVSNet on DTU, BlendedMVS or a COLMAP capture with the engine: the reference's
train.py without pytorch-lightning, test_tube or inplace_abn.

    python -m casmvsnet_pl_b200.train --root_dir DTU/mvs_training/dtu \
        --train_list lists/dtu/train.txt --val_list lists/dtu/val.txt --exp_name exp
    python -m casmvsnet_pl_b200.train --dataset_name blendedmvs \
        --root_dir BlendedMVS/dataset_low_res --depth_interval 192.0 --exp_name exp

DTU reads its scans from --train_list / --val_list (one scan per line).  BlendedMVS reads them
from the data set's own training_list.txt / validation_list.txt next to root_dir, so the two
list flags are refused for it; it trains at 768x576 with the reference's colour jitter on the
training split and validates on the validation split.  For BlendedMVS, --depth_interval is
what the reference passes to its reader as `n_depths`: each sample's depth interval is (max
depth - depth_min) / --depth_interval, so the reference README's 192.0 spreads the coarsest
stage's 48 x 4 intervals over the reference view's depth range.

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

TensorBoard (--tensorboard): the original's log as well, under logs/<exp_name>/tensorboard/.
Every metrics.jsonl record goes there too, each key but epoch, step and checkpoint as a scalar
of that name at the record's step; and at batch 0 of every training epoch and of every
validation pass the 4-panel image train/image_GT_pred_prob / val/image_GT_pred_prob (reference
image, depth_gt, depth_pred * mask, confidence * mask; visual.py), drawn on the GPU from the
step's own forward and copied to the host once.  The training image is logged at the number of
steps completed before its step, the validation one at the current step, as Lightning numbers
them.  A run without the flag writes the same files as before, and with it the same
metrics.jsonl and checkpoints.

Reproducible runs: --deterministic turns on torch.use_deterministic_algorithms (Lightning's
Trainer(deterministic=True)); the backward then runs the library's deterministic kernels and
cuDNN's heuristically chosen deterministic algorithms.  --seed N seeds the model's
initialisation, the training loader's shuffle and its workers' colour-jitter draws.  With both,
a run's metrics.jsonl and checkpoints are the same bits every time on the same data and GPU
model.

Self-supervised fine-tuning (--loss_type photo, losses.photo_loss): the photometric SSIM + L1
loss of the --photo_topk best source views per pixel (default 1, at most n_views - 1), plus
--smooth_weight (default 0.01) times an edge-aware depth smoothness.  It needs no ground truth:

    python -m casmvsnet_pl_b200.train --dataset_name colmap --loss_type photo \
        --root_dir capture [--image_dir DIR] [--img_wh 640 512] --exp_name tta

--dataset_name colmap trains on a COLMAP capture (train_data.ColmapTrainSet) with every
reference view, in train mode, and validates on the same views in eval mode; its
--depth_interval defaults to 192 as in eval_pipeline, and the checkpoint loads through
eval_pipeline --ckpt.  A photo step logs train/loss, train/photo (sum_l 2^(1-l) P_l) and
train/smooth (sum_l 2^(1-l) S_l); on DTU it also logs the level-0 metrics and checkpoints stay
ranked by val/acc_2mm, while colmap's are ranked by the lowest val/loss.  With --tensorboard,
colmap logs the scalars but no image panel, since it has no ground truth to draw.  Refused with a
message: colmap without photo, --train_list / --val_list with colmap, --img_wh / --image_dir
without colmap, photo with blendedmvs (its per-view colour jitter makes the views disagree on
purpose), --photo_topk / --smooth_weight without photo.

Not supported (the command exits with a message): radam and ranger, --use_amp, more than one
GPU.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import time

import torch
from torch.optim import SGD, Adam
from torch.optim.lr_scheduler import CosineAnnealingLR, LambdaLR, LRScheduler, MultiStepLR

from . import train_data
from .eval_pipeline import DEFAULT_DEPTH_INTERVAL, NUM_GROUPS, depth_count
from .losses import depth_metrics, photo_loss, sl1_loss_and_metrics

METRIC_NAMES = ("abs_err", "acc_1mm", "acc_2mm", "acc_4mm")
DATASETS = ("dtu", "blendedmvs", "colmap")
PHOTO_DEFAULTS = {"photo_topk": 1, "smooth_weight": 0.01, "img_wh": [640, 512]}


def build_parser(depth_interval=2.65):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--root_dir", type=str, default="/home/ubuntu/data/mvs_training/dtu/",
                    help="root directory of dtu dataset")
    ap.add_argument("--dataset_name", type=str, default="dtu", choices=list(DATASETS))
    ap.add_argument("--train_list", type=str, default=None, help="training scans, one per line")
    ap.add_argument("--val_list", type=str, default=None, help="validation scans, one per line")
    ap.add_argument("--n_views", type=int, default=3)
    ap.add_argument("--levels", type=int, default=3, choices=[3])
    ap.add_argument("--depth_interval", type=float, default=depth_interval)
    ap.add_argument("--n_depths", nargs="+", type=depth_count, default=[8, 32, 48])
    ap.add_argument("--interval_ratios", nargs="+", type=float, default=[1.0, 2.0, 4.0])
    ap.add_argument("--num_groups", type=int, default=1, choices=NUM_GROUPS)
    ap.add_argument("--loss_type", type=str, default="sl1", choices=["sl1", "photo"])
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
    ap.add_argument("--deterministic", default=False, action="store_true",
                    help="bit-reproducible steps: torch.use_deterministic_algorithms(True)")
    ap.add_argument("--seed", type=int, default=None,
                    help="seed of the initialisation, the shuffle and the workers' jitter draws")
    # absent from the namespace unless given, so that a run without it parses as before
    ap.add_argument("--tensorboard", action="store_true", default=argparse.SUPPRESS,
                    help="also log to TensorBoard under logs/<exp_name>/tensorboard/")
    ap.add_argument("--photo_topk", type=int, default=argparse.SUPPRESS,
                    help="--loss_type photo: best source views averaged per pixel (default 1)")
    ap.add_argument("--smooth_weight", type=float, default=argparse.SUPPRESS,
                    help="--loss_type photo: weight of the edge-aware depth smoothness (default 0.01)")
    ap.add_argument("--img_wh", nargs=2, type=int, default=argparse.SUPPRESS,
                    help="colmap: network input size, multiples of 32 (default 640 512)")
    ap.add_argument("--image_dir", type=str, default=argparse.SUPPRESS,
                    help="colmap: the images (default <root_dir>/images)")
    ap.add_argument("--depth_sampling", choices=["uniform", "inverse", "adaptive"],
                    default=argparse.SUPPRESS,
                    help="plane spacing of the sweep: uniform (default), inverse (evenly in "
                         "1/depth, regressed in 1/depth) or adaptive (each finer stage's window "
                         "sized from the previous stage's probability spread); not stored in the "
                         "checkpoint")
    return ap


def parse_args(argv=None):
    """build_parser's namespace with --depth_interval's default resolved per data set
    (eval_pipeline.DEFAULT_DEPTH_INTERVAL: 192 for colmap, 2.65 otherwise)."""
    pre = argparse.ArgumentParser(add_help=False)
    pre.add_argument("--dataset_name", default="dtu", choices=list(DATASETS))
    name = pre.parse_known_args(argv)[0].dataset_name
    return build_parser(DEFAULT_DEPTH_INTERVAL[name]).parse_args(argv)


def option(a, name):
    """A photometric / colmap flag's value, or its default when it was not given."""
    return getattr(a, name, PHOTO_DEFAULTS[name])


def set_deterministic():
    """torch.use_deterministic_algorithms(True), with the cuBLAS workspace setting it asks for
    (read when cuBLAS initialises, so set before the first CUDA call), and no cuDNN autotuning."""
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    torch.backends.cudnn.benchmark = False


def check_supported(a):
    """SystemExit with a message for what this trainer does not do."""
    if a.optimizer in ("radam", "ranger"):
        raise SystemExit(f"--optimizer {a.optimizer} is not supported: use sgd or adam")
    if a.use_amp:
        raise SystemExit("--use_amp is not supported: train in fp32 or --precision tf32")
    if a.num_gpus != 1:
        raise SystemExit("--num_gpus must be 1: multi-GPU training is not supported")
    photo = a.loss_type == "photo"
    for flag in ("photo_topk", "smooth_weight"):
        if hasattr(a, flag) and not photo:
            raise SystemExit(f"--{flag} needs --loss_type photo")
    for flag in ("img_wh", "image_dir"):
        if hasattr(a, flag) and a.dataset_name != "colmap":
            raise SystemExit(f"--{flag} is only used with --dataset_name colmap")
    if photo:
        k, lam = option(a, "photo_topk"), option(a, "smooth_weight")
        if not 1 <= k <= a.n_views - 1:
            raise SystemExit(f"--photo_topk must be in 1..{a.n_views - 1} (n_views - 1), got {k}")
        if not math.isfinite(lam) or lam < 0:
            raise SystemExit(f"--smooth_weight must be finite and >= 0, got {lam}")
    if a.dataset_name == "blendedmvs":
        if photo:
            raise SystemExit("--loss_type photo is not supported with blendedmvs: its training "
                             "views are colour-jittered independently, so they do not agree "
                             "photometrically")
        for flag in ("train_list", "val_list"):
            if getattr(a, flag):
                raise SystemExit(f"--{flag} is not used with --dataset_name blendedmvs: its scans "
                                 "come from training_list.txt / validation_list.txt next to root_dir")
    elif a.dataset_name == "colmap":
        if not photo:
            raise SystemExit("--dataset_name colmap has no ground-truth depth: train it with "
                             "--loss_type photo")
        for flag in ("train_list", "val_list"):
            if getattr(a, flag):
                raise SystemExit(f"--{flag} is not used with --dataset_name colmap: every "
                                 "reference view of the model is trained and validated")
        w, h = option(a, "img_wh")
        if w <= 0 or h <= 0 or w % 32 or h % 32:
            raise SystemExit(f"--img_wh must be positive multiples of 32, got {w} {h}")
    elif not a.train_list or not a.val_list:
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
                          num_groups=a.num_groups, norm_act=InPlaceABN, precision=a.precision,
                          depth_sampling=getattr(a, "depth_sampling", "uniform"))
    if a.ckpt_path:
        load_ckpt(model, a.ckpt_path, a.prefixes_to_ignore)
    return model.to(device).train()


class Trainer:
    def __init__(self, a, model, device="cuda:0"):
        self.a, self.model, self.device = a, model, device
        self.optimizer = get_optimizer(a, model)
        self.scheduler = get_scheduler(a, self.optimizer)
        self.global_step = 0
        self.tb = None                  # a SummaryWriter while fit() logs to TensorBoard

    def forward(self, s):
        return self.model(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])

    def log_panel(self, tag, s, results, step):
        """The TensorBoard image of sample 0: reference image, depth_gt, depth_pred * mask and
        confidence * mask (the original train.py:107-114), one device -> host copy."""
        from .visual import training_panel
        with torch.no_grad():
            panel = training_panel(s["imgs"][0, 0], s["depths"]["level_0"][0],
                                   results["depth_0"][0].detach(),
                                   results["confidence_0"][0].detach(), s["masks"]["level_0"][0])
        self.tb.add_image(tag, panel.cpu().numpy(), step, dataformats="HWC")

    def log_scalars(self, rec):
        for k, v in rec.items():
            if k not in ("epoch", "step", "checkpoint"):
                self.tb.add_scalar(k, v, rec["step"])

    def objective(self, s, results):
        """(loss, logged) device tensors of --loss_type.  sl1: logged = the level-0 metric sums
        (5,).  photo: logged = [photo, smooth] = sum_l 2^(1-l) [P_l, S_l], then, when the sample
        has ground truth, the level-0 metric sums."""
        a = self.a
        if a.loss_type == "sl1":
            return sl1_loss_and_metrics(results, s["depths"], s["masks"], a.levels)
        loss, stats = photo_loss(results, s["imgs"], s["proj_mats"], s["depth_interval"],
                                 a.interval_ratios, a.levels, option(a, "photo_topk"),
                                 option(a, "smooth_weight"))
        w = torch.tensor([2.0 ** (1 - l) for l in range(a.levels)], device=stats.device)
        logged = (w[:, None] * stats[:, :2]).sum(0)
        if "depths" in s:
            logged = torch.cat([logged, depth_metrics(results["depth_0"].detach(), s["depths"]["level_0"],
                                                      s["masks"]["level_0"])])
        return loss, logged

    def record(self, prefix, loss, logged):
        """The logged values of one step or validation pass as {prefix/name: float} (one read)."""
        if self.a.loss_type == "sl1":
            vals = torch.cat([loss.view(1), logged[:4] / logged[4]]).tolist()
            return {f"{prefix}/loss": vals[0], **{f"{prefix}/{k}": v for k, v in zip(METRIC_NAMES, vals[1:])}}
        parts = [loss.view(1), logged[:2]] + ([logged[2:6] / logged[6]] if logged.numel() > 2 else [])
        vals = torch.cat([t.to(torch.float64) for t in parts]).tolist()
        names = ["loss", "photo", "smooth"] + list(METRIC_NAMES[:len(vals) - 3])
        return {f"{prefix}/{k}": v for k, v in zip(names, vals)}

    def sample(self, batch):
        """A loader's batch on the device (colmap batches are built there already)."""
        return batch if "imgs" in batch else train_data.to_device(batch, self.device)

    def train_step(self, s, log_panel=False):
        """One optimiser step on a device sample -> (loss, logged) device tensors (objective).
        With log_panel, the step's forward also goes to TensorBoard as train/image_GT_pred_prob."""
        self.model.train()
        results = self.forward(s)
        loss, metrics = self.objective(s, results)
        if log_panel:
            self.log_panel("train/image_GT_pred_prob", s, results, self.global_step)
        self.optimizer.zero_grad(set_to_none=True)
        loss.backward()
        self.optimizer.step()
        self.global_step += 1
        return loss.detach(), metrics

    @torch.no_grad()
    def validate(self, batches):
        """Mean val loss and mask-weighted level-0 metrics over `batches` (train.py:129-173)."""
        if self.a.loss_type == "photo":
            return self.validate_photo(batches)
        self.model.eval()
        loss_sum = torch.zeros((), device=self.device, dtype=torch.float64)
        msum = torch.zeros(5, device=self.device, dtype=torch.float64)
        n = 0
        for i, batch in enumerate(batches):
            s = self.sample(batch)
            results = self.forward(s)
            if i == 0 and self.tb is not None:
                self.log_panel("val/image_GT_pred_prob", s, results, self.global_step)
            loss, metrics = sl1_loss_and_metrics(results, s["depths"], s["masks"], self.a.levels)
            loss_sum += loss
            msum += metrics
            n += 1
        self.model.train()
        vals = (torch.cat([(loss_sum / n).view(1), msum[:4] / msum[4]])).tolist()
        return {"val/loss": vals[0], **{f"val/{k}": v for k, v in zip(METRIC_NAMES, vals[1:])}}

    @torch.no_grad()
    def validate_photo(self, batches):
        """--loss_type photo: the mean loss, photo and smooth terms over `batches` in eval mode,
        and the mask-weighted level-0 metrics where the samples have ground truth."""
        self.model.eval()
        loss_sum = torch.zeros((), device=self.device, dtype=torch.float64)
        lsum, n = None, 0
        for i, batch in enumerate(batches):
            s = self.sample(batch)
            results = self.forward(s)
            if i == 0 and self.tb is not None and "depths" in s:
                self.log_panel("val/image_GT_pred_prob", s, results, self.global_step)
            loss, logged = self.objective(s, results)
            loss_sum += loss
            logged = logged.to(torch.float64)
            lsum = logged if lsum is None else lsum + logged
            n += 1
        self.model.train()
        lsum[:2] /= n
        return self.record("val", loss_sum / n, lsum)

    def score(self, val):
        """The checkpoint ranking: val/acc_2mm where there is ground truth, else -val/loss."""
        return val["val/acc_2mm"] if "val/acc_2mm" in val else -val["val/loss"]

    def fit(self, train_loader, val_loader, log_path, ckpt_dir):
        a = self.a
        os.makedirs(os.path.dirname(log_path) or ".", exist_ok=True)
        keep = TopKCheckpoints(ckpt_dir, 5)
        if getattr(a, "tensorboard", False):
            from torch.utils.tensorboard import SummaryWriter
            self.tb = SummaryWriter(os.path.join(os.path.dirname(log_path), "tensorboard"))
            if a.dataset_name == "colmap":
                print("tensorboard: colmap has no ground-truth depth, so only scalars are logged "
                      "(no GT / prediction / confidence panel)")
        try:
            self._fit(train_loader, val_loader, log_path, keep)
        finally:
            if self.tb is not None:
                self.tb.close()
                self.tb = None
        return keep.kept

    def _fit(self, train_loader, val_loader, log_path, keep):
        a = self.a
        with open(log_path, "a") as log:
            for epoch in range(a.num_epochs):
                for i, batch in enumerate(train_loader):
                    lr = get_learning_rate(self.optimizer)
                    s = self.sample(batch)
                    loss, m = self.train_step(s, log_panel=i == 0 and self.tb is not None and "depths" in s)
                    if self.global_step % a.log_every == 0 or self.global_step == 1:
                        rec = {"epoch": epoch, "step": self.global_step, "lr": lr}
                        rec.update(self.record("train", loss, m))
                        self._record(log, rec)
                val = self.validate(val_loader)
                path = keep(self.model, epoch, self.global_step, self.score(val))
                self._record(log, {"epoch": epoch, "step": self.global_step, **val,
                                   "checkpoint": path})
                print(f"epoch {epoch}: " + ", ".join(f"{k} {v:.4f}" for k, v in val.items()))
                self.scheduler.step()

    def _record(self, log, rec):
        log.write(json.dumps(rec) + "\n")
        log.flush()
        if self.tb is not None:
            self.log_scalars(rec)


def build_datasets(a, device="cuda:0"):
    """(train, val) readers of --dataset_name.  colmap: one set, the scene's reference views,
    serves both (trained in train mode, validated in eval mode)."""
    if a.dataset_name == "colmap":
        scene = train_data.ColmapTrainSet(a.root_dir, a.n_views, a.levels, a.depth_interval,
                                          option(a, "img_wh"), getattr(a, "image_dir", None), device)
        return scene, scene
    if a.dataset_name == "blendedmvs":
        return tuple(train_data.BlendedMVSTrainDataset(a.root_dir, split, a.n_views, a.levels,
                                                       a.depth_interval) for split in ("train", "val"))
    return tuple(train_data.DTUTrainDataset(a.root_dir, train_data.read_scan_list(lst), a.n_views,
                                            a.levels, a.depth_interval)
                 for lst in (a.train_list, a.val_list))


def loaders(a, train_set, val_set):
    if a.dataset_name == "colmap":
        return train_set.loader(a.batch_size, True, seed=a.seed), val_set.loader(a.batch_size, False)
    return (train_data.loader(train_set, a.batch_size, True, a.num_workers, seed=a.seed),
            train_data.loader(val_set, a.batch_size, False, a.num_workers))


def main(argv=None):
    a = parse_args(argv)
    check_supported(a)
    if a.deterministic:
        set_deterministic()
    if not torch.cuda.is_available():
        raise SystemExit("training needs a CUDA GPU")
    device = "cuda:0"
    train_set, val_set = build_datasets(a, device)
    if a.seed is not None:
        torch.manual_seed(a.seed)
    model = build_model(a, device)
    print("number of parameters : %.2f M" % (sum(p.numel() for p in model.parameters()
                                                  if p.requires_grad) / 1e6))
    trainer = Trainer(a, model, device)
    t0 = time.time()
    kept = trainer.fit(*loaders(a, train_set, val_set),
                       os.path.join("logs", a.exp_name, "metrics.jsonl"),
                       os.path.join("ckpts", a.exp_name))
    print(f"trained {trainer.global_step} steps in {time.time() - t0:.1f} s; "
          f"kept {sorted(kept)}")
    return trainer


if __name__ == "__main__":
    main()
