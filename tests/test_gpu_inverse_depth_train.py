"""Training in the inverse-depth mode (README "Wide depth ranges"):

  * train.Trainer steps with --depth_sampling inverse (640x512 in fp32 and tf32, the shape
    sweep's training cases, and 768x576 at B = 2 with per-item depth ranges), every autograd
    call recorded as test_gpu_train_step_fp64.py records them: the convolutions and K1 checked with that file's
    float64 checks, K3 (RegressInverseFn) forward and backward with test_gpu_regress_fp64.py's
    per-element checks of the inverse regression.  Every stage's recorded hypotheses equal rules
    3-4 restated in float32 (oracle/inverse_depth_fp64.py) bit for bit, a finer stage's on the
    previous stage's recorded depth;
  * two `train --depth_sampling inverse --deterministic --seed 0` processes, with the sl1 loss on
    a DTU-layout set and with the photometric loss on a COLMAP capture, write the same log and
    checkpoint bits, and the checkpoints differ from a uniform run's."""
import os
import subprocess
import sys

import pytest
import torch

import test_gpu_regress_fp64 as R
import test_gpu_shape_sweep_fp64 as SW
import test_gpu_train_step_fp64 as T
from casmvsnet_pl_b200 import _lib, ops, synth_scenes, train
from casmvsnet_pl_b200 import autograd as AG
from oracle import inverse_depth_fp64 as INV
from oracle import regress_fp64 as RG
from oracle import warp_cost_fp64 as W

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _grad_mode():
    with torch.enable_grad():            # conftest runs GPU tests under no_grad by default
        yield


@pytest.fixture
def rec_inv(monkeypatch):
    r = T.Recorder()
    vol = ops.volume_storage

    def conv_fwd(args, y, fb):
        x, w, kind, stride, precision = args
        return dict(x=vol(x.detach()).clone(), w=w.detach().clone(), kind=kind, stride=stride,
                    precision=precision, y=vol(y).clone(), fb=fb)

    def conv_bwd(grads, out):
        gx, gw = out[:2]
        return dict(gy=vol(grads[0]).clone(), gx=None if gx is None else vol(gx).clone(),
                    gw=None if gw is None else gw.clone())

    def warp_fwd(args, cost, fb):
        feats, proj, dv, G = args
        f = feats.detach().permute(0, 1, 3, 4, 2).clone(memory_format=torch.contiguous_format)
        return dict(f=f, P=proj.clone(), dv=dv.clone(), G=G, cost=vol(cost).clone())

    def warp_bwd(grads, out):
        return dict(gcost=vol(grads[0]).clone(), gf=out[0].permute(0, 1, 3, 4, 2).clone())

    def reg_fwd(args, out, fb):
        logits, dv = args
        return dict(logits=logits.detach().contiguous().clone(), dv=dv.clone(),
                    depth=out[0].detach().clone(), conf=out[1].clone())

    def reg_bwd(grads, out):
        return dict(gdepth=grads[0].contiguous().clone(), glogits=out[0].clone())

    T._wrap(monkeypatch, AG.Conv3dFn, conv_fwd, conv_bwd, r, r.conv, r.conv_bwd)
    T._wrap(monkeypatch, AG.WarpCostFn, warp_fwd, warp_bwd, r, r.warp, r.warp_bwd)
    T._wrap(monkeypatch, AG.RegressInverseFn, reg_fwd, reg_bwd, r, r.reg, r.reg_bwd)
    return r


def _check_k1_k3_inverse(case, rec, steps, n_depths):
    assert len(rec.warp) == len(rec.warp_bwd) == len(rec.reg) == len(rec.reg_bwd) == 3, case
    wb = {b["id"]: b for b in rec.warp_bwd}
    rb = {b["id"]: b for b in rec.reg_bwd}
    for i, c in enumerate(rec.warp):
        tag = f"{case} L{T.LEVELS[i]}"
        B, V, h, w, C = c["f"].shape
        # rules 3-4 bit for bit: the coarsest stage's planes are known in advance, a finer
        # stage's follow from the previous stage's recorded depth
        cur = None if i == 0 else rec.reg[i - 1]["depth"].cpu().numpy()
        want = INV.hypotheses_f32(steps, T.LEVELS[i], n_depths[T.LEVELS[i]], h, w, cur)
        assert torch.equal(c["dv"].cpu(), torch.from_numpy(want.copy())), tag
        fam = "staged" if ops.ladder_supported(V, C, c["G"]) else "gather"
        rep = W.check_cost(c["cost"], c["f"], c["P"], c["dv"], c["G"], T.EPS_K1[fam])
        print(f"[inverse train-fp64] {tag} warp_cost [{fam}]: {rep.describe()}")
        assert rep.ok, f"{tag} warp_cost: {rep.describe()}"
        b = wb[i]
        rep = W.check_warp_cost_bwd(b["gf"], c["f"], c["P"], c["dv"], b["gcost"], c["G"],
                                    T.EPS_K1["bwd"])
        print(f"[inverse train-fp64] {tag} warp_cost_bwd: {rep.describe()}")
        assert rep.ok, f"{tag} warp_cost_bwd: {rep.describe()}"
    for i, c in enumerate(rec.reg):
        tag = f"{case} L{T.LEVELS[i]}"
        depth, conf, index, _ = ops.regress(c["logits"], c["dv"], want_index=True, inverse=True)
        assert torch.equal(depth, c["depth"]) and torch.equal(conf, c["conf"]), tag
        # test_gpu_regress_fp64.py's per-element checks of the inverse regression
        R._check_k3(f"[inverse train] {tag}", c["logits"], c["dv"], depth, conf, index,
                    inverse=True)
        b = rb[i]
        g64, b0, A = RG.regress_bwd_ref(c["logits"], c["dv"], b["gdepth"], inverse=True)
        R._report(f"[inverse train] {tag} bwd", "k3_inv_bwd",
                  RG.check(b["glogits"], g64, b0, A, R.EPS["k3_inv_bwd"], ("b", "d", "y", "x")))


def _inverse_step(case, rec_inv, precision, W_, H, V=3, G=1, n_depths=(8, 32, 48), B=1):
    a = train.build_parser().parse_args(["--precision", precision, "--optimizer", "sgd",
                                         "--depth_sampling", "inverse", "--num_groups", str(G),
                                         "--n_views", str(V), "--n_depths", *map(str, n_depths)])
    torch.manual_seed(0)
    model = train.build_model(a, DEV)
    assert model.depth_sampling == "inverse"
    tr = train.Trainer(a, model, DEV)
    s = T._sample(B, W_, H, seed=1, V=V)
    if B > 1:           # per-item depth ranges: per-item steps in every stage
        s["init_depth_min"] = torch.tensor([[425.0 + 26.5 * b] for b in range(B)], device=DEV)
        s["depth_interval"] = torch.tensor([[2.65 + 0.4 * b] for b in range(B)], device=DEV)
    f0 = _lib.fallback_count()
    loss, _ = tr.train_step(s)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).item()
    steps = INV.steps_f32(s["init_depth_min"], s["depth_interval"], a.n_depths, a.interval_ratios, B)
    with torch.no_grad():
        fallbacks = T._check_conv_calls(case, rec_inv, precision == "tf32")
        want = T._expected_fallbacks(precision == "tf32", G)
        assert fallbacks == want and _lib.fallback_count() - f0 == len(want), (fallbacks, want)
        _check_k1_k3_inverse(case, rec_inv, steps, a.n_depths)


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_inverse_training_step_vs_fp64(precision, rec_inv):
    _inverse_step(f"dtu_{precision}_inverse", rec_inv, precision, 640, 512)


# test_gpu_shape_sweep_fp64.py's training cases (G = 2, G = 4; V = 4 with odd D/8 on the gather
# K1 path), and a 768x576 step at B = 2 with per-item depth ranges
TRAIN_CASES = {**SW.TRAIN_CASES, "blendedmvs_b2": (768, 576, 3, 1, (8, 32, 48), 2)}


@pytest.mark.parametrize("case", list(TRAIN_CASES))
def test_inverse_training_cases_vs_fp64(case, rec_inv):
    W_, H, V, G, Ds, *B = TRAIN_CASES[case]
    _inverse_step(f"{case}_inverse", rec_inv, "tf32", W_, H, V, G, Ds, B[0] if B else 1)


# ------------------------------------------------------------------------------- the CLI
CODE = "import sys\nsys.path.insert(0, %r)\nfrom casmvsnet_pl_b200 import train\ntrain.main(sys.argv[1:])\n" % ROOT


def _runs(argv, tmp_path, tag, n=2):
    runs = []
    for i in range(n):
        cwd = tmp_path / f"{tag}{i}"
        cwd.mkdir()
        subprocess.run([sys.executable, "-c", CODE] + argv, check=True, cwd=str(cwd), timeout=900)
        runs.append(cwd)
    return runs


def _ckpts(run):
    d = run / "ckpts" / "det"
    return {n: torch.load(d / n, map_location="cpu")["state_dict"] for n in sorted(os.listdir(d))}


def _same_runs(runs, uniform):
    logs = [open(r / "logs" / "det" / "metrics.jsonl", "rb").read() for r in runs]
    assert logs[0] and logs[0] == logs[1]
    c0, c1, cu = _ckpts(runs[0]), _ckpts(runs[1]), _ckpts(uniform)
    assert c0 and c0.keys() == c1.keys() and cu
    for n in c0:
        for k, v in c0[n].items():
            assert torch.equal(v, c1[n][k]), f"{n}: {k}"
    # the inverse runs trained other weights than the uniform run with the same seed
    last, last_u = c0[sorted(c0)[-1]], cu[sorted(cu)[-1]]
    assert any(not torch.equal(v, last_u[k]) for k, v in last.items() if v.is_floating_point())


@pytest.mark.parametrize("loss", ["sl1", "photo"])
def test_two_deterministic_inverse_runs_write_the_same_bits(loss, tmp_path):
    if loss == "sl1":
        root = synth_scenes.make_dtu_train(str(tmp_path / "dtu"), seed=0)
        argv = ["--root_dir", root, "--train_list", os.path.join(root, "lists", "train.txt"),
                "--val_list", os.path.join(root, "lists", "val.txt"), "--num_epochs", "1",
                "--optimizer", "adam", "--log_every", "1", "--num_workers", "0"]
    else:
        root = str(tmp_path / "capture")
        synth_scenes.make_colmap(root, n_views=6, image_wh=(160, 128), n_points=2000, seed=2,
                                 textured=True)
        argv = ["--dataset_name", "colmap", "--loss_type", "photo", "--root_dir", root, "--img_wh",
                "160", "128", "--n_views", "3", "--num_epochs", "1", "--log_every", "1",
                "--optimizer", "adam"]
    argv += ["--exp_name", "det", "--deterministic", "--seed", "0"]
    runs = _runs(argv + ["--depth_sampling", "inverse"], tmp_path, "inv")
    uniform = _runs(argv, tmp_path, "uni", n=1)[0]
    _same_runs(runs, uniform)
