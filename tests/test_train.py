"""The training workflow's host side against goldens recorded from the reference
(oracle/make_golden_train.py -> tests/golden/train/*.npz): the DTU training reader, the
learning-rate schedules, checkpoints and the CLI's refusals.  CPU only."""
import hashlib
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import train, train_data
from oracle.make_golden_train import FIXTURE_SEED, SCHEDULES, fixture_digest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train")


def _golden(name):
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return {k: z[k] for k in z.files}


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def fixture_root(tmp_path_factory):
    from casmvsnet_pl_b200.synth_scenes import make_dtu_train
    root = make_dtu_train(str(tmp_path_factory.mktemp("dtu_train")), seed=FIXTURE_SEED)
    g = _golden("reader")
    assert fixture_digest(root) == str(g["fixture_digest"]), \
        "synth_scenes.make_dtu_train no longer writes the fixture the goldens were recorded on"
    return root


@pytest.mark.parametrize("split", ["train", "val"])
def test_reader_matches_reference(fixture_root, split):
    g = _golden("reader")
    p = split + "/"
    ds = train_data.DTUTrainDataset(fixture_root, train_data.read_scan_list(
        os.path.join(fixture_root, "lists", f"{split}.txt")))
    assert len(ds) == len(g[p + "metas"])
    order = list(g["digest_order"])
    for i, (scan, light, ref, srcs) in enumerate(ds.metas):
        assert scan == g[p + "scans"][i]
        assert [light, ref] + srcs == g[p + "metas"][i].tolist()
        s = ds[i]
        assert s["scan_vid"] == (scan, ref)
        assert np.array_equal(s["proj_mats"].numpy(), g[p + "proj_mats"][i])
        assert np.array_equal(s["init_depth_min"].numpy(), g[p + "init_depth_min"][i])
        assert np.array_equal(s["depth_interval"].numpy(), g[p + "depth_interval"][i])
        assert s["imgs_u8"].shape == (3, 512, 640, 3) and s["imgs_u8"].dtype == torch.uint8
        for l in range(3):
            d, m = s["depths"][f"level_{l}"], s["masks"][f"level_{l}"]
            assert d.shape == (512 >> l, 640 >> l) and m.dtype == torch.bool
            assert _sha(d.numpy()) == g[p + "digests"][i][order.index(f"depth_{l}")], (i, l)
            assert _sha(m.numpy()) == g[p + "digests"][i][order.index(f"mask_{l}")], (i, l)


def test_depth_pyramid_is_cv2_nearest():
    """The slicing in train_data.depth_pyramid is cv2.resize(fx=fy=0.5, INTER_NEAREST) + crop."""
    import cv2
    full = np.random.default_rng(0).random((1200, 1600), dtype=np.float32)
    want = cv2.resize(full, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_NEAREST)[44:556, 80:720]
    got = train_data.depth_pyramid(full)
    assert np.array_equal(got["level_0"], want)
    for l in (1, 2):
        want = cv2.resize(want, None, fx=0.5, fy=0.5, interpolation=cv2.INTER_NEAREST)
        assert np.array_equal(got[f"level_{l}"], want)


def _hparams(opt, sched, wu, mult, extra):
    a = train.build_parser().parse_args([])
    a.optimizer, a.lr_scheduler, a.warmup_epochs, a.warmup_multiplier = opt, sched, wu, mult
    for k, v in extra.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("name,opt,sched,wu,mult,extra", SCHEDULES, ids=[s[0] for s in SCHEDULES])
def test_lr_schedule_matches_reference(name, opt, sched, wu, mult, extra):
    import warnings
    g = _golden("schedulers")
    a = _hparams(opt, sched, wu, mult, extra)
    o = train.get_optimizer(a, torch.nn.Linear(2, 2))
    s = train.get_scheduler(a, o)
    lrs = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for _ in range(16):
            lrs.append(train.get_learning_rate(o))
            o.step()
            s.step()
    assert np.array_equal(np.array(lrs, np.float64), g[name]), (lrs, g[name])


def _cpu_model(seed=0):
    from casmvsnet_pl_b200 import InPlaceABN, synth
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    m = CascadeMVSNet(norm_act=InPlaceABN)
    synth.randomize_model_(m, seed)
    return m


def test_checkpoint_round_trip(tmp_path):
    from casmvsnet_pl_b200 import eval_pipeline
    model = _cpu_model(3)
    path = str(tmp_path / "ckpts" / "exp" / "_ckpt_epoch_0.ckpt")
    train.save_checkpoint(model, path, epoch=0, global_step=7)
    ck = torch.load(path, map_location="cpu")
    assert ck["epoch"] == 0 and ck["global_step"] == 7
    assert all(k.startswith("model.") for k in ck["state_dict"])
    loaded = eval_pipeline.load_checkpoint(_cpu_model(4), path)
    want = model.state_dict()
    for k, v in loaded.state_dict().items():
        assert torch.equal(v, want[k]), k
    # the weights-only warm start, with a prefix ignored
    warm = _cpu_model(4)
    before = {k: v.clone() for k, v in warm.state_dict().items()}
    train.load_ckpt(warm, path, ["cost_reg_0"])
    for k, v in warm.state_dict().items():
        assert torch.equal(v, before[k] if k.startswith("cost_reg_0") else want[k]), k


def test_checkpoint_loads_in_reference(tmp_path):
    from oracle.ref_loader import reference_available
    if not reference_available():
        pytest.skip("reference tree not available")
    from oracle.make_golden_train import reference_utils
    from oracle.ref_loader import load_reference_models
    mvsnet, _, abn = load_reference_models()
    model = _cpu_model(5)
    path = str(tmp_path / "_ckpt_epoch_3.ckpt")
    train.save_checkpoint(model, path, epoch=3, global_step=100)
    ref = mvsnet.CascadeMVSNet(norm_act=abn)
    reference_utils().load_ckpt(ref, path, ["loss"])
    want = model.state_dict()
    for k, v in ref.state_dict().items():
        assert torch.equal(v, want[k]), k


@pytest.mark.parametrize("argv,msg", [(["--optimizer", "radam"], "radam"),
                                      (["--optimizer", "ranger"], "ranger"),
                                      (["--use_amp"], "use_amp"),
                                      (["--num_gpus", "2"], "num_gpus")])
def test_cli_rejects_unsupported(argv, msg):
    with pytest.raises(SystemExit) as e:
        train.main(argv + ["--train_list", "x", "--val_list", "y"])
    assert msg in str(e.value.code)


@pytest.mark.parametrize("argv,flag", [(["--n_depths", "8", "32", "44"], "--n_depths"),
                                       (["--n_depths", "0", "32", "48"], "--n_depths"),
                                       (["--n_depths", "-8"], "--n_depths"),
                                       (["--num_groups", "3"], "--num_groups"),
                                       (["--num_groups", "16"], "--num_groups")])
def test_cli_refuses_bad_depths_and_groups_at_parsing(argv, flag, capsys):
    from casmvsnet_pl_b200 import eval_pipeline
    with pytest.raises(SystemExit) as e:
        train.build_parser().parse_args(argv)
    assert e.value.code == 2 and f"argument {flag}" in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        eval_pipeline.parse_args(["--root_dir", "x"] + argv)
    assert e.value.code == 2 and f"argument {flag}" in capsys.readouterr().err


def test_cli_accepts_the_depths_and_groups_the_network_runs():
    from casmvsnet_pl_b200 import eval_pipeline
    for g in (1, 2, 4, 8):
        argv = ["--num_groups", str(g), "--n_depths", "8", "24", "192"]
        a = train.build_parser().parse_args(argv)
        b = eval_pipeline.parse_args(["--root_dir", "x"] + argv)
        assert a.num_groups == b.num_groups == g and a.n_depths == b.n_depths == [8, 24, 192]


def test_top_k_checkpoints_keep_the_best(tmp_path):
    keep = train.TopKCheckpoints(str(tmp_path), k=2)
    m = torch.nn.Linear(1, 1)
    for e, score in enumerate([0.5, 0.7, 0.6, 0.4, 0.8]):
        keep(m, e, e, score)
    assert sorted(os.listdir(tmp_path)) == ["_ckpt_epoch_1.ckpt", "_ckpt_epoch_4.ckpt"]
