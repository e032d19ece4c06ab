"""Record tests/golden/train/*.npz from the REAL reference's training code (needs the reference
tree, CASMVS_REFERENCE_ROOT or /root/reference; run from the repository root):

    python -m oracle.make_golden_train

reader.npz      datasets/dtu.py DTUDataset(split, img_wh=None) on the seeded fixture of
                casmvsnet_pl_b200.synth_scenes.make_dtu_train: per sample the metas, scan_vid,
                init_depth_min, depth_interval and proj_mats in full; SHA-256 digests of the
                imgs / depths / masks arrays with a few small crops; and a digest of the decoded
                fixture files, so that drift of the generator is told apart from a reader bug.
                The reference reads its scan lists by relative path, so it runs from a temporary
                working directory holding the fixture's lists as datasets/lists/dtu/*.txt.
loss.npz        losses.py SL1Loss and metrics.py on seeded 3-level inputs with errors of
                exactly 1, 2 and 4 and their float neighbours: loss, gradients (for
                loss.backward() and for (0.37 * loss).backward()) and level-0 metric sums.
schedulers.npz  utils get_optimizer / get_scheduler: the lr of each of 16 epochs for several
                optimiser / scheduler / warm-up settings, stepping once per epoch as Lightning
                does.  This pins the reference's code as it behaves on the torch it is recorded
                with.  The reference's utils/__init__.py uses LambdaLR ('poly') without importing
                it; torch's LambdaLR is injected into that module, the evident intent.
"""
from __future__ import annotations

import argparse
import contextlib
import hashlib
import importlib
import importlib.util
import os
import shutil
import sys
import tempfile

import numpy as np
import torch

from oracle.ref_loader import REFERENCE_ROOT, reference_available

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "train")
FIXTURE_SEED = 0

# (name, optimizer, lr_scheduler, warmup_epochs, warmup_multiplier, extra)
SCHEDULES = [
    ("sgd_steplr", "sgd", "steplr", 0, 1.0, {"decay_step": [2, 4, 8], "decay_gamma": 0.5}),
    ("sgd_cosine_warmup", "sgd", "cosine", 3, 2.0, {}),
    ("adam_poly", "adam", "poly", 0, 1.0, {"poly_exp": 0.9}),
    ("adam_steplr_warmup", "adam", "steplr", 2, 4.0, {"decay_step": [5, 10], "decay_gamma": 0.1}),
    ("sgd_poly_warmup", "sgd", "poly", 4, 1.0, {"poly_exp": 0.9}),
]


def sha(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(a.tobytes()).hexdigest()


def fixture_digest(root):
    """SHA-256 over the fixture as the reference's decoders see it: cam and pair files as text,
    PNG images through PIL, PFM depths through read_pfm, masks through cv2.imread(path, 0)."""
    import cv2
    from PIL import Image

    from casmvsnet_pl_b200 import io
    h = hashlib.sha256()
    for dirpath, _, files in sorted(os.walk(root)):
        for name in sorted(files):
            path = os.path.join(dirpath, name)
            h.update(os.path.relpath(path, root).encode())
            if name.endswith(".txt"):
                h.update(open(path, "rb").read())
            elif name.startswith("depth_visual"):
                h.update(np.ascontiguousarray(cv2.imread(path, 0)).tobytes())
            elif name.endswith(".png"):
                h.update(np.ascontiguousarray(np.asarray(Image.open(path))).tobytes())
            elif name.endswith(".pfm"):
                h.update(np.ascontiguousarray(io.read_pfm(path)[0]).tobytes())
    return h.hexdigest()


def _reference_package(name):
    """Import <reference>/<name> under a private name (never shadows this repository's own)."""
    from oracle.ref_loader import load_reference_models
    load_reference_models()                      # the inplace_abn / kornia stand-ins
    pkg_name = "_casmvs_reference_" + name
    if pkg_name not in sys.modules:
        path = os.path.join(REFERENCE_ROOT, name)
        spec = importlib.util.spec_from_file_location(pkg_name, os.path.join(path, "__init__.py"),
                                                      submodule_search_locations=[path])
        pkg = importlib.util.module_from_spec(spec)
        sys.modules[pkg_name] = pkg
        spec.loader.exec_module(pkg)
    return sys.modules[pkg_name]


def reference_utils():
    """The reference's utils package (get_optimizer, get_scheduler, load_ckpt, ...)."""
    u = _reference_package("utils")
    if not hasattr(u, "LambdaLR"):
        u.LambdaLR = torch.optim.lr_scheduler.LambdaLR
    return u


@contextlib.contextmanager
def _cwd(path):
    old = os.getcwd()
    os.chdir(path)
    try:
        yield
    finally:
        os.chdir(old)


def make_fixture(root):
    from casmvsnet_pl_b200.synth_scenes import make_dtu_train
    return make_dtu_train(root, seed=FIXTURE_SEED)


def record_reader(tmp):
    fixture = make_fixture(os.path.join(tmp, "dtu"))
    work = os.path.join(tmp, "work")
    os.makedirs(os.path.join(work, "datasets", "lists", "dtu"))
    for split in ("train", "val"):
        shutil.copy(os.path.join(fixture, "lists", f"{split}.txt"),
                    os.path.join(work, "datasets", "lists", "dtu", f"{split}.txt"))
    DTUDataset = importlib.import_module(_reference_package("datasets").__name__ + ".dtu").DTUDataset
    out = {"fixture_digest": np.array(fixture_digest(fixture)), "fixture_seed": np.array(FIXTURE_SEED)}
    with _cwd(work):
        for split in ("train", "val"):
            ds = DTUDataset(fixture, split, n_views=3, levels=3, depth_interval=2.65)
            rows, pms, dmin, dint, scans, dig, crops = [], [], [], [], [], [], []
            for i in range(len(ds)):
                scan, light, ref, srcs = ds.metas[i]
                s = ds[i]
                assert s["scan_vid"] == (scan, ref)
                scans.append(scan)
                rows.append([light, ref] + list(srcs))
                pms.append(s["proj_mats"].numpy())
                dmin.append(s["init_depth_min"].numpy())
                dint.append(s["depth_interval"].numpy())
                d = [sha(s["imgs"].numpy())]
                d += [sha(s["depths"][f"level_{l}"].numpy()) for l in range(3)]
                d += [sha(s["masks"][f"level_{l}"].numpy()) for l in range(3)]
                dig.append(d)
                crops.append(np.concatenate([s["imgs"].numpy()[:, :, 100:102, 200:202].ravel(),
                                             s["depths"]["level_0"].numpy()[200:202, 300:302].ravel(),
                                             s["masks"]["level_0"].numpy()[200:202, 300:302].ravel()]))
            p = split + "/"
            out.update({p + "scans": np.array(scans), p + "metas": np.array(rows, np.int64),
                        p + "proj_mats": np.stack(pms), p + "init_depth_min": np.stack(dmin),
                        p + "depth_interval": np.stack(dint), p + "digests": np.array(dig),
                        p + "crops": np.stack(crops).astype(np.float32)})
    out["digest_order"] = np.array(["imgs"] + [f"depth_{l}" for l in range(3)] +
                                   [f"mask_{l}" for l in range(3)])
    return out


def loss_inputs(seed=11, B=2, H=48, W=64):
    """Seeded 3-level (pred, gt, mask); level 0 holds errors of exactly +-1, 2, 4 and their
    float32 neighbours."""
    g = torch.Generator().manual_seed(seed)
    preds, gts, masks = [], [], []
    for l in range(3):
        h, w = H >> l, W >> l
        gt = 500 + 300 * torch.rand(B, h, w, generator=g)
        err = torch.randn(B, h, w, generator=g) * (3.0 / (l + 1))
        pred = gt + err
        mask = torch.rand(B, h, w, generator=g) > 0.3
        preds.append(pred.float())
        gts.append(gt.float())
        masks.append(mask)
    gt0, pred0, m0 = gts[0].view(-1), preds[0].view(-1), masks[0].view(-1)
    special = []
    for t in (1.0, 2.0, 4.0):
        ft = torch.tensor(t)
        for v in (ft, torch.nextafter(ft, torch.tensor(0.0)), torch.nextafter(ft, torch.tensor(9.0))):
            special += [v.item(), -v.item()]
    for i, e in enumerate(special):
        k = 7 * i + 3
        gt0[k] = 0.0                               # so that pred - gt is exactly e
        pred0[k] = e
        m0[k] = True
    return preds, gts, masks


def record_loss():
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        losses = importlib.import_module("losses")
        metrics = importlib.import_module("metrics")
    finally:
        sys.path.remove(REFERENCE_ROOT)
    preds, gts, masks = loss_inputs()
    out = {}
    for l in range(3):
        out[f"pred_{l}"], out[f"gt_{l}"], out[f"mask_{l}"] = preds[l].numpy(), gts[l].numpy(), masks[l].numpy()
    for tag, scale in (("", None), ("scaled_", 0.37)):
        ps = [p.clone().requires_grad_(True) for p in preds]
        loss = losses.SL1Loss(3)({f"depth_{l}": ps[l] for l in range(3)},
                                 {f"level_{l}": gts[l] for l in range(3)},
                                 {f"level_{l}": masks[l] for l in range(3)})
        (loss if scale is None else loss * scale).backward()
        if scale is None:
            out["loss"] = loss.detach().numpy()
        for l in range(3):
            out[f"{tag}grad_{l}"] = ps[l].grad.numpy()
    out["grad_scale"] = np.float32(0.37)
    e = metrics.abs_error(preds[0], gts[0], masks[0])
    out["abs_err_sum"] = e.sum().numpy()
    out["abs_err_sum64"] = np.float64(e.double().sum().item())
    out["acc_counts"] = np.array([metrics.acc_threshold(preds[0], gts[0], masks[0], t).sum().item()
                                  for t in (1, 2, 4)], np.float64)
    out["mask_sum"] = masks[0].float().sum().numpy()
    out["special_count"] = np.int64(18)
    return out


def record_schedulers():
    u = reference_utils()
    out = {}
    for name, opt, sched, wu, mult, extra in SCHEDULES:
        hp = argparse.Namespace(optimizer=opt, lr=1e-3, momentum=0.9, weight_decay=1e-5,
                                lr_scheduler=sched, warmup_epochs=wu, warmup_multiplier=mult,
                                decay_step=[20], decay_gamma=0.1, poly_exp=0.9, num_epochs=16,
                                use_amp=False)
        for k, v in extra.items():
            setattr(hp, k, v)
        model = torch.nn.Linear(2, 2)
        o = u.get_optimizer(hp, model)
        s = u.get_scheduler(hp, o)
        lrs = []
        for _ in range(16):
            lrs.append(u.get_learning_rate(o))
            o.step()
            s.step()
        out[name] = np.array(lrs, np.float64)
        out[name + "/config"] = np.array(repr(sorted(vars(hp).items())))
    return out


def main():
    if not reference_available():
        raise SystemExit(f"reference tree not found at {REFERENCE_ROOT}")
    os.makedirs(OUT, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        np.savez_compressed(os.path.join(OUT, "reader.npz"), **record_reader(tmp))
    np.savez(os.path.join(OUT, "loss.npz"), **record_loss())
    np.savez(os.path.join(OUT, "schedulers.npz"), **record_schedulers())
    print("wrote", sorted(os.listdir(OUT)))


if __name__ == "__main__":
    import warnings
    warnings.filterwarnings("ignore")
    main()
