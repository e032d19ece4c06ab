"""Training panels on the GPU (csrc/visual.cu through casmvsnet_pl_b200/visual.py):

  * training_panel, visualize_depth and visualize_prob equal the original project's outputs
    recorded in tests/golden/visual byte for byte, in every recorded case (DTU and BlendedMVS
    shapes, NaN / inf, constant depth, confidence levels, out-of-range images, wrapping casts and
    the no-positive-depth rule), and the numpy restatement at other sizes;
  * inputs the kernel does not cover are refused with a message;
  * `train.main([... "--tensorboard", "--deterministic", "--seed", "0"])` for two epochs: the
    event file's scalars are the metrics.jsonl records, its two image tags sit at the expected
    steps and decode to the panels the kernel drew from those steps' batches, and metrics.jsonl
    and the checkpoints are byte-identical to the same run without --tensorboard."""
import glob
import io
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from casmvsnet_pl_b200 import visual                                # noqa: E402
from oracle import visual_oracle as O                               # noqa: E402

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "visual")
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN, "*.npz"))
               if not p.endswith("cast.npz"))


def _inputs(z):
    return (torch.from_numpy(z["img"]).to(DEV), torch.from_numpy(z["depth_gt"]).to(DEV),
            torch.from_numpy(z["depth_pred"]).to(DEV), torch.from_numpy(z["conf"]).to(DEV),
            torch.from_numpy(z["mask"]).to(DEV))


@pytest.mark.parametrize("name", CASES)
def test_panels_equal_reference(name):
    z = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    img, gt, pred, conf, mask = _inputs(z)
    panel = visual.training_panel(img, gt, pred, conf, mask)
    assert panel.dtype == torch.uint8 and panel.device == torch.device(DEV)
    got = panel.cpu().numpy()
    bad = np.argwhere((got != z["panel"]).any(-1))
    assert len(bad) == 0, f"{name}: {len(bad)} pixels differ, first at {bad[:4].tolist()}"
    for key, got in (("vis_depth_gt", visual.visualize_depth(gt)),
                     ("vis_depth_pred", visual.visualize_depth(pred * mask)),
                     ("vis_prob", visual.visualize_prob(conf * mask))):
        assert got.dtype == torch.float32 and got.shape == z[key].shape
        assert np.array_equal(got.cpu().numpy(), z[key]), f"{name}: {key}"
    print(f"[visual] {name} {tuple(gt.shape)}: panel and views equal the reference"
          + (" (no positive depth: grey level 0)" if z["vis_depth_gt_raises"] else ""))


def _random_case(H, W, seed):
    g = np.random.default_rng(seed)
    img = g.normal(0.0, 1.5, (3, H, W)).astype(np.float32)
    gt = g.uniform(400.0, 950.0, (H, W)).astype(np.float32) * (g.random((H, W)) > 0.1)
    pred = (gt + g.normal(0.0, 30.0, (H, W))).astype(np.float32)
    conf = g.uniform(-0.05, 1.05, (H, W)).astype(np.float32)
    mask = g.random((H, W)) > 0.2
    flat = pred.reshape(-1)
    k = max(1, flat.size // 500)
    idx = g.choice(flat.size, 3 * k)
    flat[idx[:k]], flat[idx[k:2 * k]], flat[idx[2 * k:]] = np.nan, np.inf, -1e12
    return img, gt, pred, conf, mask


@pytest.mark.parametrize("H,W", [(1, 1), (5, 7), (33, 257), (864, 1152)])
def test_panels_equal_oracle_at_other_sizes(H, W):
    case = _random_case(H, W, H * 7 + W)
    want = O.training_panel(*case)
    got = visual.training_panel(*(torch.from_numpy(a).to(DEV) for a in case)).cpu().numpy()
    assert np.array_equal(got, want)
    # uint8 masks work as bool ones
    args = [torch.from_numpy(a).to(DEV) for a in case]
    args[4] = args[4].to(torch.uint8)
    assert np.array_equal(visual.training_panel(*args).cpu().numpy(), want)


def test_no_positive_depth_is_grey_level_zero():
    d = torch.tensor([[0.0, -3.0], [float("nan"), float("-inf")]], device=DEV)
    got = visual.visualize_depth(d)
    jet0 = torch.tensor(O.colormaps()["JET"][0], dtype=torch.float32) / 255
    assert torch.equal(got.cpu(), jet0.view(3, 1, 1).expand(3, 2, 2))


def test_refuses_inputs_it_does_not_cover():
    img, gt, pred, conf, mask = _inputs(dict(np.load(os.path.join(GOLDEN, "constant.npz"))))
    good = [img, gt, pred, conf, mask]

    def refused(i, t, what):
        args = list(good)
        args[i] = t
        with pytest.raises(ValueError, match=what):
            visual.training_panel(*args)

    refused(0, img.double(), "float32")
    refused(1, gt.cpu(), "CUDA")
    refused(2, pred.t(), "shape")
    refused(2, pred.t().contiguous().t(), "contiguous")
    refused(3, conf[:, ::2], "shape")
    refused(0, img.transpose(1, 2).contiguous().transpose(1, 2), "contiguous")
    refused(4, mask.float(), "bool or torch.uint8")
    refused(3, conf[:-1], "shape")
    with pytest.raises(ValueError, match="non-empty"):
        visual.visualize_depth(torch.zeros(0, 4, device=DEV))
    with pytest.raises(ValueError, match=r"\(H, W\)"):
        visual.visualize_prob(torch.zeros(2, 3, 4, device=DEV))
    with pytest.raises(ValueError, match="contiguous"):
        visual.visualize_prob(torch.zeros(8, 8, device=DEV)[:, ::2])
    if torch.cuda.device_count() > 1:
        refused(1, gt.to("cuda:1"), "other inputs")


# ------------------------------------------------------------------------------ the trainer
# Runs train.main in a child process; with --tensorboard, every training_panel call's inputs and
# output are saved to panels.npz in the working directory.
_RUN = """import sys
import numpy as np
sys.path.insert(0, %r)
from casmvsnet_pl_b200 import train, visual
calls = []
draw = visual.training_panel
def recorded(*args):
    out = draw(*args)
    calls.append([t.cpu().numpy() for t in args] + [out.cpu().numpy()])
    return out
visual.training_panel = recorded
train.main(sys.argv[1:])
if calls:
    np.savez("panels.npz", **{f"{i}_{k}": a for i, c in enumerate(calls) for k, a in enumerate(c)})
""" % ROOT


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    from casmvsnet_pl_b200.synth_scenes import make_dtu_train
    base = tmp_path_factory.mktemp("tb")
    root = make_dtu_train(str(base / "dtu"), seed=0)
    argv = ["--root_dir", root, "--train_list", os.path.join(root, "lists", "train.txt"),
            "--val_list", os.path.join(root, "lists", "val.txt"), "--num_epochs", "2",
            "--optimizer", "adam", "--log_every", "1", "--num_workers", "2", "--exp_name", "tb",
            "--deterministic", "--seed", "0"]
    out = {}
    for name, extra in (("tb", ["--tensorboard"]), ("plain", [])):
        cwd = base / name
        cwd.mkdir()
        subprocess.run([sys.executable, "-c", _RUN] + argv + extra, check=True, cwd=str(cwd),
                       timeout=900)
        out[name] = cwd
    return out


def _events(cwd):
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    files = glob.glob(str(cwd / "logs" / "tb" / "tensorboard" / "events.out.tfevents.*"))
    assert len(files) == 1, files
    acc = EventAccumulator(files[0], size_guidance={"scalars": 0, "images": 0})
    acc.Reload()
    return acc


def test_tensorboard_scalars_are_the_jsonl_records(runs):
    acc = _events(runs["tb"])
    recs = [json.loads(line) for line in open(runs["tb"] / "logs" / "tb" / "metrics.jsonl")]
    want = {}
    for r in recs:
        for k, v in r.items():
            if k not in ("epoch", "step", "checkpoint"):
                want.setdefault(k, []).append((r["step"], np.float32(v)))
    assert set(acc.Tags()["scalars"]) == set(want)
    assert {"lr", "train/loss", "train/abs_err", "train/acc_1mm", "train/acc_2mm", "train/acc_4mm",
            "val/loss", "val/abs_err", "val/acc_1mm", "val/acc_2mm", "val/acc_4mm"} == set(want)
    for tag, pts in want.items():
        got = [(e.step, np.float32(e.value)) for e in acc.Scalars(tag)]
        assert len(got) == len(pts), tag
        for (s0, v0), (s1, v1) in zip(got, pts):
            assert s0 == s1 and (v0 == v1 or (np.isnan(v0) and np.isnan(v1))), (tag, s0, v0, s1, v1)
    print(f"[visual] {sum(len(p) for p in want.values())} scalars over {len(want)} tags match "
          f"{len(recs)} metrics.jsonl records")


def test_tensorboard_images_are_the_kernel_panels(runs):
    from PIL import Image
    acc = _events(runs["tb"])
    recs = [json.loads(line) for line in open(runs["tb"] / "logs" / "tb" / "metrics.jsonl")]
    per_epoch = max(r["step"] for r in recs if r["epoch"] == 0)
    assert set(acc.Tags()["images"]) == {"train/image_GT_pred_prob", "val/image_GT_pred_prob"}
    train_ev = acc.Images("train/image_GT_pred_prob")
    val_ev = acc.Images("val/image_GT_pred_prob")
    assert [e.step for e in train_ev] == [0, per_epoch]
    assert [e.step for e in val_ev] == [per_epoch, 2 * per_epoch]
    z = np.load(runs["tb"] / "panels.npz")
    # calls in order: train epoch 0, val epoch 0, train epoch 1, val epoch 1
    events = [train_ev[0], val_ev[0], train_ev[1], val_ev[1]]
    assert len(z.files) == 6 * len(events)
    for i, ev in enumerate(events):
        img, gt, pred, conf, mask, drawn = (z[f"{i}_{k}"] for k in range(6))
        H, W = gt.shape
        assert drawn.shape == (H, 4 * W, 3) and (ev.height, ev.width) == (H, 4 * W)
        png = np.asarray(Image.open(io.BytesIO(ev.encoded_image_string)).convert("RGB"))
        assert np.array_equal(png, drawn), f"event {i}: PNG differs from the kernel's panel"
        again = visual.training_panel(*(torch.from_numpy(a).to(DEV) for a in (img, gt, pred, conf, mask)))
        assert np.array_equal(again.cpu().numpy(), drawn)
        assert np.array_equal(O.training_panel(img, gt, pred, conf, mask), drawn)
    print(f"[visual] images at train steps {[e.step for e in train_ev]}, val steps "
          f"{[e.step for e in val_ev]}; {H}x{4 * W} panels equal the kernel's and the oracle's")


def test_tensorboard_leaves_the_run_unchanged(runs):
    tb, plain = runs["tb"], runs["plain"]
    assert open(tb / "logs" / "tb" / "metrics.jsonl", "rb").read() == \
        open(plain / "logs" / "tb" / "metrics.jsonl", "rb").read()
    assert sorted(os.listdir(plain / "logs" / "tb")) == ["metrics.jsonl"]
    assert not (plain / "panels.npz").exists()
    names = sorted(os.listdir(tb / "ckpts" / "tb"))
    assert names and names == sorted(os.listdir(plain / "ckpts" / "tb"))
    for n in names:
        assert open(tb / "ckpts" / "tb" / n, "rb").read() == open(plain / "ckpts" / "tb" / n, "rb").read(), n
