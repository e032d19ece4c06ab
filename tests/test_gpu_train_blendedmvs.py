"""BlendedMVS training on the GPU: the fused colour-jitter + normalise kernel against
torchvision-on-PIL (tests/golden/train/jitter.npz) and the host oracle, the reader's device
images against the reference's digests, per-sample depth ranges in a batch, one trainer step
against a hand-written step, and train.main end to end with its checkpoint read back."""
import copy
import hashlib
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from casmvsnet_pl_b200 import _lib, train, train_data                      # noqa: E402
from casmvsnet_pl_b200 import io as cio                                    # noqa: E402
from oracle import jitter_oracle as J                                      # noqa: E402
from oracle.make_golden_train_blendedmvs import FIXTURE_ROOT, N_DEPTHS_ARG, SEED   # noqa: E402

DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train")


@pytest.fixture(autouse=True)
def _grad_mode():
    with torch.enable_grad():            # conftest runs GPU tests under no_grad by default
        yield


def _golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return {k: z[k] for k in z.files}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _jn(imgs, jit):
    return cio.jitter_normalize_images(torch.from_numpy(np.ascontiguousarray(imgs)).to(DEV),
                                       torch.from_numpy(np.asarray(jit, np.float32)).to(DEV))


def test_jitter_kernel_matches_torchvision_golden():
    g = _golden("jitter")
    imgs = g["images"][g["image_index"]]
    out = _jn(imgs, g["jitter"]).cpu().numpy()
    for i in range(len(out)):
        assert np.array_equal(out[i], J.normalize(g["jittered"][i])), (i, g["jitter"][i])
        assert _sha(out[i]) == g["normalized_sha"][i], i
    for i, j in enumerate(g["odd_jitter"]):                 # 17x33, N = 1: the scalar path
        o = _jn(g["odd_image"][None], j[None]).cpu().numpy()[0]
        assert _sha(o) == g["odd_normalized_sha"][i], i


def _full_size_case(seed=0, N=6):
    rng = np.random.default_rng(seed)
    imgs = rng.integers(0, 256, (N, 576, 768, 3), dtype=np.uint8)
    imgs[1] = np.clip(imgs[1].astype(np.int32) // 6 + 200, 0, 255)      # bright: saturates at 255
    imgs[2] = imgs[2] // 10                                              # dark: saturates at 0
    jit = np.array([[1, 0.75, 0.5], [1, 1.25, 1.5], [0, 0.75, 1.5], [0, 1.25, 0.5], [1, 1.0, 1.0],
                    [0, 1.1, 0.7]], np.float32)[:N]
    return imgs, jit


def test_jitter_kernel_matches_oracle_at_training_size_and_is_deterministic():
    imgs, jit = _full_size_case()
    a = _jn(imgs, jit)
    b = _jn(imgs, jit)
    assert torch.equal(a, b)
    want = J.jitter_normalize(imgs, jit)
    got = a.cpu().numpy()
    for i in range(len(imgs)):
        assert np.array_equal(got[i], want[i]), (i, jit[i])
    assert torch.equal(_jn(imgs[4:5], jit[4:5]), cio.normalize_images(torch.from_numpy(imgs[4:5]).to(DEV)))
    odd = imgs[0, :31, :45].copy()
    for j in jit[:4]:
        assert np.array_equal(_jn(odd[None], j[None]).cpu().numpy()[0],
                              J.jitter_normalize(odd[None], j[None])[0]), j


def test_jitter_kernel_makes_no_host_sync():
    imgs, jit = _full_size_case(N=4)
    x, j = torch.from_numpy(imgs).to(DEV), torch.from_numpy(jit).to(DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = cio.jitter_normalize_images(x, j)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(out, _jn(imgs, jit))


def test_jitter_kernel_rejects_bad_arguments():
    x = torch.zeros(2, 8, 8, 3, dtype=torch.uint8, device=DEV)
    j = torch.ones(2, 3, device=DEV)
    with pytest.raises(_lib.CasMVSError):
        cio.jitter_normalize_images(x.float(), j)
    with pytest.raises(_lib.CasMVSError):
        cio.jitter_normalize_images(x, j[:1])
    with pytest.raises(_lib.CasMVSError):
        cio.jitter_normalize_images(x, j.double())
    with pytest.raises(_lib.CasMVSError):
        cio.jitter_normalize_images(x.cpu(), j)                        # host input, no device
    with pytest.raises(_lib.CasMVSError, match="multiple of 4"):
        cio.jitter_normalize_images(torch.zeros(2, 3, 5, 3, dtype=torch.uint8, device=DEV), j)
    lib = _lib.load()
    import ctypes
    p = ctypes.c_void_p(x.data_ptr())
    m = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    assert lib.casmvs_jitter_normalize_u8_fwd(p, None, p, p, 1, 8, 8, m, m, None) < 0
    assert b"null" in lib.casmvs_last_error()
    bad = ctypes.c_void_p(x.data_ptr() + 4)
    assert lib.casmvs_jitter_normalize_u8_fwd(p, p, p, bad, 1, 8, 8, m, m, None) < 0
    assert b"misaligned" in lib.casmvs_last_error()
    z = (ctypes.c_float * 3)(0.5, 0.0, 0.5)
    assert lib.casmvs_jitter_normalize_u8_fwd(p, p, p, p, 1, 8, 8, m, z, None) < 0


def _batch(ds, idx, seeds=None):
    samples = []
    for k, i in enumerate(idx):
        if seeds is not None:
            torch.manual_seed(seeds[k])
        samples.append(ds[i])
    return train_data.to_device(torch.utils.data.default_collate(samples), DEV)


@pytest.mark.parametrize("split", ["train", "val"])
def test_device_images_match_reference(split):
    g = _golden("blendedmvs_reader")
    order = list(g["digest_order"])
    ds = train_data.BlendedMVSTrainDataset(FIXTURE_ROOT, split, 3, 3, N_DEPTHS_ARG)
    for i in range(len(ds)):
        imgs = _batch(ds, [i], [int(SEED) + i])["imgs"][0].cpu().numpy()
        assert _sha(imgs) == g[split + "/digests"][i][order.index("imgs")], i


def _args(**kw):
    a = train.build_parser().parse_args(["--dataset_name", "blendedmvs"])
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _model(a):
    torch.manual_seed(0)
    return train.build_model(a, DEV)


def test_batch_keeps_per_sample_depth_ranges():
    """B = 2 from two scans: each sample's eval-mode depth is its B = 1 depth (to the noise of
    a batch-size-dependent cuDNN algorithm), and far from the depth with the ranges swapped."""
    ds = train_data.BlendedMVSTrainDataset(FIXTURE_ROOT, "all", 3, 3, N_DEPTHS_ARG)
    idx = [0, len(ds) - 1]
    assert ds.metas[idx[0]][0] != ds.metas[idx[1]][0]
    s2 = _batch(ds, idx)
    assert s2["init_depth_min"][0] != s2["init_depth_min"][1]
    assert s2["depth_interval"][0] != s2["depth_interval"][1]
    model = _model(_args()).eval()
    with torch.no_grad():
        fwd = lambda s, dmin, dint: model(s["imgs"], s["proj_mats"], dmin, dint)["depth_0"]  # noqa: E731
        both = fwd(s2, s2["init_depth_min"], s2["depth_interval"])
        swapped = fwd(s2, s2["init_depth_min"].flip(0), s2["depth_interval"].flip(0))
        for k, i in enumerate(idx):
            s1 = _batch(ds, [i])
            one = fwd(s1, s1["init_depth_min"], s1["depth_interval"])[0]
            err = (both[k] - one).abs().max().item()
            far = (swapped[k] - one).abs().max().item()
            print(f"sample {i}: |B=2 - B=1| max {err:.2e}; with swapped ranges {far:.2e}")
            assert err <= 1e-3 * s1["depth_interval"].item()
            assert far > 100 * max(err, 1e-6)


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


def test_trainer_step_matches_hand_written_step():
    """One SGD step on a jittered B = 2 batch at 768x576 (V = 3, D = 48/32/8), read against the
    run-to-run noise of two hand-written steps, as test_gpu_train does for DTU."""
    a = _args(optimizer="sgd")
    model = _model(a)
    twins = [copy.deepcopy(model) for _ in range(3)]
    ds = train_data.BlendedMVSTrainDataset(FIXTURE_ROOT, "train", 3, 3, N_DEPTHS_ARG)
    s = _batch(ds, [1, 4], [int(SEED) + 1, int(SEED) + 4])
    assert s["imgs"].shape == (2, 3, 3, 576, 768)
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


def test_loaders_with_one_seed_give_identical_jittered_batches():
    ds = train_data.BlendedMVSTrainDataset(FIXTURE_ROOT, "train", 3, 3, N_DEPTHS_ARG)
    runs = []
    for _ in range(2):
        runs.append([(b["jitter"].clone(), train_data.to_device(b, DEV)["imgs"].cpu())
                     for b in train_data.loader(ds, 2, True, 2, seed=5)])
    other = [b["jitter"] for b in train_data.loader(ds, 2, True, 2, seed=6)]
    assert len(runs[0]) == 3
    for (ja, ia), (jb, ib) in zip(*runs):
        assert torch.equal(ja, jb) and torch.equal(ia, ib)
    assert not all(torch.equal(x, y) for x, (y, _) in zip(other, runs[0]))


def _fallbacks_of_one_step(img_wh):
    """tf32 fallback launches (layers no wgmma kernel covers) of one training step and of one
    eval-mode forward at img_wh."""
    ds = train_data.BlendedMVSTrainDataset(FIXTURE_ROOT, "train", 3, 3, N_DEPTHS_ARG, img_wh)
    a = _args(precision="tf32")
    model = _model(a)
    s = _batch(ds, [0], [int(SEED)])
    f0 = _lib.fallback_count()
    train.Trainer(a, model, DEV).train_step(s)
    f1 = _lib.fallback_count()
    with torch.no_grad():
        model.eval()(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])
    return f1 - f0, _lib.fallback_count() - f1


def test_tf32_fallbacks_do_not_depend_on_the_image_size():
    """At 768x576 the eval-mode forward (validation, eval_pipeline) runs every tf32 layer on
    the tensor cores.  A training step's backward has dgrad layers without a wgmma kernel; the
    kernel choice depends on channels, kind and stride only, so the count is that of any other
    training shape (640x512 here, DTU's)."""
    step_bmvs, eval_bmvs = _fallbacks_of_one_step((768, 576))
    step_dtu, _ = _fallbacks_of_one_step((640, 512))
    print(f"tf32 fallback layers per training step: {step_bmvs} at 768x576, {step_dtu} at 640x512; "
          f"eval forward at 768x576: {eval_bmvs}")
    assert eval_bmvs == 0
    assert step_bmvs == step_dtu


def test_main_trains_validates_and_checkpoint_reads_back(tmp_path, monkeypatch):
    from casmvsnet_pl_b200 import InPlaceABN, eval_pipeline
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    from casmvsnet_pl_b200.synth_scenes import make_blendedmvs_train
    root = make_blendedmvs_train(str(tmp_path / "bmvs"), n_views=(28, 6))
    monkeypatch.chdir(tmp_path)
    step_fallbacks, _ = _fallbacks_of_one_step((768, 576))
    fb0 = _lib.fallback_count()
    torch.manual_seed(0)                  # model init, shuffle order and the workers' jitter
    trainer = train.main(["--dataset_name", "blendedmvs", "--root_dir", root, "--depth_interval", "192.0",
                          "--num_epochs", "1", "--optimizer", "adam", "--log_every", "1",
                          "--num_workers", "2", "--precision", "tf32", "--exp_name", "bmvs"])
    recs = [json.loads(line) for line in open(tmp_path / "logs" / "bmvs" / "metrics.jsonl")]
    steps = [r for r in recs if "train/loss" in r]
    vals = [r for r in recs if "val/loss" in r]
    assert len(steps) == 21 and len(vals) == 1
    assert _lib.fallback_count() - fb0 == 21 * step_fallbacks, "validation ran a tf32 fallback layer"
    first, last = steps[0]["train/loss"], np.mean([r["train/loss"] for r in steps[-5:]])
    print(f"train/loss first step {first:.4f}, mean of the last 5 steps {last:.4f}; val {vals[0]}")
    assert last < first
    path = str(tmp_path / "ckpts" / "bmvs" / "_ckpt_epoch_0.ckpt")
    assert vals[0]["checkpoint"] == os.path.join("ckpts", "bmvs", "_ckpt_epoch_0.ckpt")

    val = train_data.BlendedMVSTrainDataset(root, "val", 3, 3, 192.0)
    s = _batch(val, [2])
    with torch.no_grad():
        model = trainer.model.eval()
        want = model(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])["depth_0"]
        fresh = CascadeMVSNet(norm_act=InPlaceABN, precision="tf32")
        fresh = eval_pipeline.load_checkpoint(fresh, path).eval().to(DEV)
        got = fresh(s["imgs"], s["proj_mats"], s["init_depth_min"], s["depth_interval"])["depth_0"]
    assert torch.equal(got, want)
    eval_pipeline.main(["--dataset_name", "blendedmvs", "--split", "val", "--root_dir", root,
                        "--img_wh", "768", "576", "--n_views", "3", "--depth_interval", "192.0", "--ckpt", path,
                        "--out", str(tmp_path / "results")])
    assert os.listdir(tmp_path / "results" / "depth" / val.scans[0])
