"""The training workflow on the GPU: the fused loss / metric kernel against the reference's
SL1Loss and metrics (tests/golden/train/loss.npz), the reader's device normalisation, one
trainer step against a hand-written step with the reference's loss formula, and a short run
whose checkpoint reproduces the trainer's eval-mode depth through eval_pipeline's loader."""
import copy
import hashlib
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from casmvsnet_pl_b200 import losses, train, train_data          # noqa: E402
from oracle.make_golden_train import FIXTURE_SEED                   # noqa: E402

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train")


@pytest.fixture(autouse=True)
def _grad_mode():
    with torch.enable_grad():            # conftest runs GPU tests under no_grad by default
        yield


def _golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return {k: z[k] for k in z.files}


def _loss_inputs(g):
    preds = {f"depth_{l}": torch.from_numpy(g[f"pred_{l}"]).to(DEV).requires_grad_(True) for l in range(3)}
    gts = {f"level_{l}": torch.from_numpy(g[f"gt_{l}"]).to(DEV) for l in range(3)}
    masks = {f"level_{l}": torch.from_numpy(g[f"mask_{l}"]).to(DEV) for l in range(3)}
    return preds, gts, masks


def _loss64(g):
    """The loss formula in float64 on the float32 differences."""
    total = 0.0
    for l in range(3):
        x = (g[f"pred_{l}"] - g[f"gt_{l}"]).astype(np.float32)[g[f"mask_{l}"]].astype(np.float64)
        ax = np.abs(x)
        total += 2.0 ** (1 - l) * np.where(ax < 1, 0.5 * ax * ax, ax - 0.5).mean()
    return total


def _run_loss(g, scale=None):
    preds, gts, masks = _loss_inputs(g)
    loss, metrics = losses.sl1_loss_and_metrics(preds, gts, masks)
    (loss if scale is None else loss * scale).backward()
    return loss.detach(), metrics, [preds[f"depth_{l}"].grad for l in range(3)]


def test_loss_kernel_matches_reference():
    g = _golden("loss")
    loss, metrics, grads = _run_loss(g)
    for l in range(3):
        assert torch.equal(grads[l].cpu(), torch.from_numpy(g[f"grad_{l}"])), f"level {l} gradient"
    scale = float(g["grad_scale"])
    _, _, sgrads = _run_loss(g, scale)
    for l in range(3):
        assert torch.equal(sgrads[l].cpu(), torch.from_numpy(g[f"scaled_grad_{l}"])), f"level {l} (scaled)"
    ours, ref, l64 = loss.item(), float(g["loss"]), _loss64(g)
    print(f"loss: kernel {ours!r}, reference fp32 {ref!r}, fp64 formula {l64!r}")
    assert abs(ours - ref) <= 1e-6 * abs(ref)
    assert abs(ours - l64) <= np.spacing(np.float32(l64))
    m = metrics.cpu().numpy()
    assert m[0] == np.float32(g["abs_err_sum64"])
    assert m[1:4].tolist() == g["acc_counts"].tolist() and m[4] == float(g["mask_sum"])
    dm = losses.depth_metrics(*(torch.from_numpy(g[k + "_0"]).to(DEV) for k in ("pred", "gt", "mask")))
    assert torch.equal(dm, metrics)


def test_loss_kernel_is_deterministic_and_nan_on_empty_mask():
    g = _golden("loss")
    a, b = _run_loss(g), _run_loss(g)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(x, y) for x, y in zip(a[2], b[2]))
    preds, gts, masks = _loss_inputs(g)
    masks["level_1"] = torch.zeros_like(masks["level_1"])
    loss = losses.SL1Loss(3)(preds, gts, masks)
    assert torch.isnan(loss).item()
    loss.backward()
    assert torch.count_nonzero(preds["depth_1"].grad).item() == 0


def test_loss_and_metrics_make_no_host_sync():
    g = _golden("loss")
    preds, gts, masks = _loss_inputs(g)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = losses.loss_dict["sl1"](3)(preds, gts, masks)
        loss.backward()
        m = losses.depth_metrics(preds["depth_0"].detach(), gts["level_0"], masks["level_0"])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert m.is_cuda and loss.is_cuda


@pytest.fixture(scope="module")
def fixture_root(tmp_path_factory):
    from casmvsnet_pl_b200.synth_scenes import make_dtu_train
    return make_dtu_train(str(tmp_path_factory.mktemp("dtu_train")), seed=FIXTURE_SEED)


def _dataset(root, split="train"):
    return train_data.DTUTrainDataset(root, train_data.read_scan_list(os.path.join(root, "lists", f"{split}.txt")))


def _batch(ds, idx):
    return train_data.to_device(torch.utils.data.default_collate([ds[i] for i in idx]), DEV)


def test_reader_images_match_reference(fixture_root):
    g = _golden("reader")
    ds = _dataset(fixture_root)
    order = list(g["digest_order"])
    for i in (0, 4, 9, 20):
        imgs = _batch(ds, [i])["imgs"][0].cpu().numpy()
        assert hashlib.sha256(imgs.tobytes()).hexdigest() == g["train/digests"][i][order.index("imgs")], i


def _args(**kw):
    a = train.build_parser().parse_args([])
    a.train_list = a.val_list = "unused"
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _model(a):
    torch.manual_seed(0)
    return train.build_model(a, DEV)


def rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _hand_written_step(model, s, a):
    """The reference's loss by boolean indexing (losses.py:10-17), backward, SGD."""
    model.train()
    opt = torch.optim.SGD(model.parameters(), lr=a.lr, momentum=a.momentum, weight_decay=a.weight_decay)
    res = model(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])
    ref = 0
    for l in range(3):
        m = s["masks"][f"level_{l}"]
        ref = ref + F.smooth_l1_loss(res[f"depth_{l}"][m], s["depths"][f"level_{l}"][m]) * 2 ** (1 - l)
    opt.zero_grad()
    ref.backward()
    opt.step()
    return ref.detach()


def _flat(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()])


def test_trainer_step_matches_hand_written_step(fixture_root):
    """One SGD step at the training shape (640x512, V = 3, D = 48/32/8, B = 1).  The backward
    is not bit-reproducible run to run (float atomics in conv3d_wgrad and cuDNN's 2D
    backward), so a second hand-written step gives the noise floor the per-tensor comparison
    is read against; a warm-up step first settles cuDNN's algorithm choice."""
    a = _args(optimizer="sgd")
    model = _model(a)
    twins = [copy.deepcopy(model) for _ in range(3)]
    s = _batch(_dataset(fixture_root), [3])
    _hand_written_step(twins[0], s, a)                              # warm-up
    loss, _ = train.Trainer(a, model, DEV).train_step(s)
    ref = _hand_written_step(twins[1], s, a)
    _hand_written_step(twins[2], s, a)
    print(f"step loss: trainer {loss.item():.6f}, hand-written {ref.item():.6f}")
    assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item())
    whole = rel(_flat(model), _flat(twins[1]))
    worst = max(rel(p.detach(), q.detach()) for p, q in zip(model.parameters(), twins[1].parameters()))
    noise = max(rel(p.detach(), q.detach()) for p, q in zip(twins[2].parameters(), twins[1].parameters()))
    print(f"parameters after one step: rel-L2 {whole:.2e} overall; worst tensor {worst:.2e} "
          f"(two hand-written steps: {noise:.2e})")
    assert whole < 1e-6
    assert worst < 1e-5


def test_short_run_checkpoint_reproduces_eval_depth(fixture_root, tmp_path):
    from casmvsnet_pl_b200 import eval_pipeline
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    from casmvsnet_pl_b200 import InPlaceABN
    a = _args(optimizer="adam", num_epochs=1, log_every=1)
    model = _model(a)
    trainer = train.Trainer(a, model, DEV)
    ds = _dataset(fixture_root)
    log_path = str(tmp_path / "logs" / "metrics.jsonl")
    kept = trainer.fit(train_data.loader(ds, 1, True, 2, seed=0),
                       train_data.loader(_dataset(fixture_root, "val"), 1, False, 2),
                       log_path, str(tmp_path / "ckpts"))
    recs = [json.loads(line) for line in open(log_path)]
    steps = [r for r in recs if "train/loss" in r]
    vals = [r for r in recs if "val/loss" in r]
    assert len(steps) == len(ds) and len(vals) == 1
    first, last = steps[0]["train/loss"], np.mean([r["train/loss"] for r in steps[-5:]])
    print(f"train/loss first step {first:.4f}, mean of the last 5 steps {last:.4f}; val {vals[0]}")
    assert last < first
    assert len(kept) == 1
    path = next(iter(kept))
    assert os.path.basename(path) == "_ckpt_epoch_0.ckpt"

    s = _batch(_dataset(fixture_root, "val"), [5])
    with torch.no_grad():
        model.eval()
        want = model(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])["depth_0"]
        fresh = CascadeMVSNet(norm_act=InPlaceABN, precision=a.precision)
        fresh = eval_pipeline.load_checkpoint(fresh, path).eval().to(DEV)
        got = fresh(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])["depth_0"]
    assert torch.equal(got, want)
