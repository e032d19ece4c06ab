"""Adaptive depth ranges on the GPU (README "Adaptive depth ranges", rule in csrc/regress.cu):

  * K4 (adaptive_hypotheses_kernel) bit for bit against the float32 restatement, in both output
    forms, with the floor, the 1e-7 clamp and NaN spreads active;
  * K3's spread within oracle/adaptive_depth_fp64.spread_ref's per-element bound at every new
    instantiation, with depth, confidence and index bit-identical to the call without spread;
  * the per-pixel-step staged K1 against float64 (oracle/warp_cost_fp64), including a window wide
    enough that stage_boxes halves its runs;
  * a profiler run, in a child process, that launches every new kernel;
  * ladder and materialised cascades, the cascade against the adaptive oracle, GraphedCascade;
  * training with either loss, deterministic reruns and eval_pipeline --ckpt."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import ABN, ops, synth
from oracle import adaptive_depth_fp64 as AD
from oracle import warp_cost_fp64 as W

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS_K3 = 2.0 ** -19          # the K3 reductions' eps (test_gpu_regress_fp64.py: "k3")


def _maps(B, hi, wi, seed, scale=6.0):
    g = torch.Generator().manual_seed(seed)
    cur = 425.0 + 500.0 * torch.rand(B, hi, wi, generator=g)
    spread = scale * torch.rand(B, hi, wi, generator=g)
    return cur, spread


def _bits(a):
    return torch.as_tensor(np.ascontiguousarray(a)).view(torch.int32)


# ------------------------------------------------------------------------------- K4
@pytest.mark.parametrize("case", ["float", "per_item", "edges"])
@pytest.mark.parametrize("D", [2, 8, 32])
def test_k4_matches_restatement(case, D):
    B, hi, wi = 2, 64, 80
    cur, spread = _maps(B, hi, wi, D)
    step = 2.5 if case == "float" else torch.tensor([[2.5], [5.3]])
    if case == "edges":
        spread[0, :8] = 0.0                       # the floor r = g
        cur[1, :8] = 3.0                          # the 1e-7 clamp
        spread[1, 8:16] = float("nan")            # a NaN spread: r = g
        spread[0, 16:24, :8] = 200.0              # a window far wider than the uniform one
    want = AD.hypotheses_f32(cur, spread, D, step)
    lo, st = AD.hypotheses_f32(cur, spread, D, step, first_only=True)
    if case == "edges":
        assert (lo == np.float32(1e-7)).any() and np.isnan(spread.numpy()).any()
    stp = step.to(DEV) if torch.is_tensor(step) else step
    got = ops.adaptive_hypotheses(cur.to(DEV), spread.to(DEV), D, stp)
    assert torch.equal(got.cpu().view(torch.int32), _bits(want))
    f, s = ops.adaptive_hypotheses(cur.to(DEV), spread.to(DEV), D, stp, first_only=True)
    assert torch.equal(f.cpu().view(torch.int32), _bits(lo))
    assert torch.equal(s.cpu().view(torch.int32), _bits(st))
    # the per-pixel-step Ladder materialises the same planes
    lad = ops.Ladder(f, s, D, B, 2 * hi, 2 * wi, DEV)
    assert torch.equal(lad.materialize().cpu().view(torch.int32), _bits(want))


# ------------------------------------------------------------------------------- K3
# stage shapes of cfg2 (640x512) and 1152x864: (D, h, w) of stages 2 and 1, plus D = 8 (the
# per-thread kernel) and D = 256 (the generic kernel: the plane-parallel one needs too much smem)
K3_SHAPES = [(48, 128, 160), (32, 256, 320), (48, 216, 288), (32, 432, 576), (8, 256, 320),
             (256, 32, 40)]


def _check_spread(tag, logits, hyp, spread, is_prob=False):
    sig, bound = AD.spread_ref(logits.cpu(), hyp.cpu(), is_prob, EPS_K3)
    err = (spread.cpu().double() - sig).abs()
    bad = err > bound
    print(f"[k3 spread] {tag}: worst err/bound {float((err / bound.clamp_min(1e-30)).max()):.3f}")
    assert not bool(bad.any()), f"{tag}: {int(bad.sum())} spreads outside the bound"


@pytest.mark.parametrize("scale", [1.0, 4.0, 30.0])
@pytest.mark.parametrize("shape", K3_SHAPES)
def test_k3_spread_vs_fp64(shape, scale):
    D, h, w = shape
    g = torch.Generator(device=DEV).manual_seed(D * 1000 + h + int(scale))
    B = 2
    logits = scale * torch.randn(B, D, h, w, generator=g, device=DEV)
    step = torch.tensor([2.5, 4.1], device=DEV)
    first = 425.0 + 300.0 * torch.rand(B, h, w, generator=g, device=DEV)
    pix_step = 0.2 + 8.0 * torch.rand(B, h, w, generator=g, device=DEV)
    for form in ("tensor", "per_item", "per_pixel"):
        if form == "per_item":
            lad = ops.Ladder(torch.tensor([425.0, 610.0], device=DEV), step, D, B, h, w, DEV)
        else:
            lad = ops.Ladder(first, pix_step, D, B, h, w, DEV)
        hyp = lad.materialize()
        tag = f"D={D} {h}x{w} scale {scale} {form}"
        base = ops.regress(logits, hyp, want_index=True, want_prob=True)
        if form == "tensor":
            out = ops.regress(logits, hyp, want_index=True, want_prob=True, want_spread=True)
            for a, b in zip(base, out[:4]):
                assert torch.equal(a, b), f"{tag}: spread changed the regression"
            spread = out[4]
            prob = torch.softmax(logits, 1)
            pb = ops.regress(prob, hyp, input_is_prob=True, want_index=True)
            po = ops.regress(prob, hyp, input_is_prob=True, want_index=True, want_spread=True)
            for a, b in zip(pb, po[:4]):
                assert (a is None and b is None) or torch.equal(a, b), f"{tag}: prob input"
            _check_spread(tag + " input_is_prob", prob, hyp, po[4], True)
        else:
            d, c, i, spread = ops.regress_ladder(logits, lad, want_index=True, want_spread=True)
            for a, b in zip(base[:3], (d, c, i)):
                assert torch.equal(a, b), f"{tag}: ladder with spread != regress"
            if form == "per_pixel":
                nd, nc, ni = ops.regress_ladder(logits, lad, want_index=True)
                for a, b in zip(base[:3], (nd, nc, ni)):
                    assert torch.equal(a, b), f"{tag}: per-pixel ladder != regress"
        _check_spread(tag, logits, hyp, spread)


# ------------------------------------------------------------------------------- K1
def _k1_case(V, C, G, wide, seed):
    import test_gpu_warp_cost_fp64 as K
    B, D = 2, 8
    level = {8: 0, 16: 1, 32: 2}[C]
    h, w = (24, 160) if wide else (64, 96)
    g = torch.Generator(device=DEV).manual_seed(seed)
    feats = K._feats(g, B, V, C, h, w)
    P = K._proj("default", V, w << level, h << level, level, B)
    first = 500.0 + 200.0 * torch.rand(B, h, w, generator=g, device=DEV)
    step = 0.5 + 6.0 * torch.rand(B, h, w, generator=g, device=DEV)
    if wide:
        # a band of pixels whose window spans most of the scene: planes 0 and 1 alone leave the box
        first[:, 2:22, 16:144] = 120.0
        step[:, 2:22, 16:144] = 60.0
    lad = ops.Ladder(first, step, D, B, h, w, DEV)
    spec = ("ladder", B, V, C, G, h, w, D)
    return K, spec, feats, P, lad


@pytest.mark.parametrize("wide", [False, True])
@pytest.mark.parametrize("G", [1, 8])
@pytest.mark.parametrize("C", [8, 16, 32])
@pytest.mark.parametrize("V", [2, 3])
def test_k1_pixel_step_vs_fp64(V, C, G, wide):
    K, spec, feats, P, lad = _k1_case(V, C, G, wide, V * 100 + C + G + int(wide))
    dv = lad.materialize()
    if wide:
        assert K._wide(spec, P, dv.cpu()), "the wide window does not make stage_boxes halve its runs"
    f = K._cl5(feats)
    first = None
    for blocked in (False, True):
        for rnd in (False, True):
            y = ops.warp_cost_ladder(feats, P, lad, G, round_tf32=rnd, blocked=blocked)
            y = W.from_blocked(y) if blocked else ops.volume_storage(y)
            if rnd:
                assert torch.equal(y.contiguous().view(torch.int32),
                                   W.tf32_rna(first.contiguous()).view(torch.int32))
                continue
            if first is not None:
                assert torch.equal(y, first), "blocked != channels-last"
                continue
            first = y
    rep = W.check_cost(first, f, P, dv, G, K.EPS["staged"])
    print(f"[k1 pix] V={V} C={C} G={G} wide={wide}: {rep.describe()}")
    assert rep.ok, rep.describe()
    assert rep.loose_share <= K.LOOSE_CEIL["cost"], rep.describe()
    # the per-pixel-step ladder and the materialised planes run the same arithmetic
    mat = ops.volume_storage(ops.warp_cost(feats, P, dv, G, ops.NHWC))
    assert torch.equal(mat, first)


# ------------------------------------------------------------------------------- coverage
def _new_kernels():
    exp = {"adaptive_hypotheses_kernel"}
    for c in (8, 16, 32):
        for blk in ("true", "false"):
            exp.add(f"warp_var_smem_pg_pix_kernel<{c}, .*{blk}>")
            for v in (1, 2):
                for gwc in ("true", "false"):
                    if not (v == 2 and gwc == "false"):
                        exp.add(f"warp_var_smem_pix_kernel<{v}, {c}, .*{gwc}, {blk}>")
    exp |= {"regress_spread_kernel<true, 8, false>", "regress_spread_kernel<false, 8, false>",
            "regress_spread_kernel<true, 0, false>", "regress_spread_kernel<false, 0, false>",
            "regress_spread_kernel<false, 8, true>", "regress_spread_kernel<false, 0, true>",
            "regress_par_spread_kernel<true, false>", "regress_par_spread_kernel<false, false>",
            "regress_par_spread_kernel<false, true>"}
    return exp


def _child_coverage(path):
    """Launches every new kernel under torch.profiler and saves the kernel names to `path`.  Runs in
    a child process: a profiling session leaves state behind in the process that ran it, and a
    later session in the same process (test_gpu_regress_fp64.py::test_kernel_coverage) must see
    its own kernels."""
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        cur, spread = _maps(1, 8, 8, 0)
        ops.adaptive_hypotheses(cur.to(DEV), spread.to(DEV), 8, 2.5)
        for D in (8, 32, 256):
            lg = torch.randn(1, D, 16, 16, device=DEV)
            dv = 400 + torch.arange(D, device=DEV, dtype=torch.float32).view(1, -1, 1, 1).expand(1, D, 16, 16)
            ops.regress(lg, dv.contiguous(), want_spread=True)
            ops.regress(torch.softmax(lg, 1), dv.contiguous(), input_is_prob=True, want_spread=True)
            lad = ops.Ladder(torch.full((1, 16, 16), 400.0, device=DEV), torch.ones(1, 16, 16, device=DEV),
                             D, 1, 16, 16, DEV)
            ops.regress_ladder(lg, lad)
        for V in (2, 3):
            for C in (8, 16, 32):
                for G in (1, 8):
                    _, _, feats, P, lad = _k1_case(V, C, G, False, 1)
                    for blocked in (False, True):
                        ops.warp_cost_ladder(feats, P, lad, G, blocked=blocked)
        torch.cuda.synchronize()
    torch.save(sorted({e.name for e in prof.events()}), path)


def test_every_new_kernel_launched(tmp_path):
    path = str(tmp_path / "names.pt")
    code = ("import sys\nsys.path.insert(0, %r)\nsys.path.insert(0, %r)\n"
            "import test_gpu_adaptive_depth as T\nT._child_coverage(sys.argv[1])\n"
            % (ROOT, os.path.join(ROOT, "tests")))
    subprocess.run([sys.executable, "-c", code, path], check=True, timeout=600)
    names = torch.load(path)
    missing = [k for k in _new_kernels() if not any(re.search(re.escape(k).replace(r"\.\*", ".*"), n)
                                                    for n in names)]
    assert not missing, missing


# ------------------------------------------------------------------------------- cascade
def _model(G, precision, sampling="adaptive", seed=0):
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(seed)
    m = CascadeMVSNet(num_groups=G, norm_act=ABN, precision=precision, depth_sampling=sampling)
    synth.randomize_model_(m, seed)
    return m.eval().to(DEV)


@pytest.mark.parametrize("G", [1, 8])
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("size", [(640, 512, 3), (1152, 864, 5)])
def test_ladder_equals_materialised(size, precision, G):
    W_, H, V = size
    m = _model(G, precision)
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=V, W=W_, H=H, seed=1)
    imgs, pm = imgs.to(DEV), pm.to(DEV)
    with torch.no_grad():
        a = m(imgs, pm, dmin, dint)
        m.fuse_hypotheses = False
        b = m(imgs, pm, dmin, dint)
        m.set_depth_sampling("uniform")
        u = m(imgs, pm, dmin, dint)
    assert a.keys() == b.keys() == u.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k
    assert not torch.equal(a["depth_0"], u["depth_0"])      # the mode is not a no-op


def test_cascade_vs_adaptive_oracle():
    """cfg2 at B = 2 with distinct per-item depth ranges, fp32, against the oracle per stage."""
    m = _model(1, "fp32")
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    imgs, pm, dmin, dint = synth.make_inputs(B=2, V=3, W=640, H=512, seed=3)
    dmin_t = torch.tensor([[float(dmin)], [float(dmin) * 0.9]])
    dint_t = torch.tensor([[float(dint)], [float(dint) * 1.3]])
    nt = torch.get_num_threads()
    torch.set_num_threads(min(16, nt))
    ref = AD.cascade_forward_adaptive(sd, imgs, pm, dmin_t, dint_t)
    torch.set_num_threads(nt)
    m.return_index = True
    with torch.no_grad():
        res = m(imgs.to(DEV), pm.to(DEV), dmin_t.to(DEV), dint_t.to(DEV))
    for l in (2, 1, 0):
        d, r = res[f"depth_{l}"].cpu(), ref[f"depth_{l}"]
        rel = float((d - r).abs().mean() / r.abs().mean())
        cd = float((res[f"confidence_{l}"].cpu() - ref[f"confidence_{l}"]).abs().mean())
        idx = float((res[f"depth_index_{l}"].cpu() != ref[f"depth_index_{l}"]).float().mean())
        print(f"[adaptive cascade] level {l}: depth rel-L1 {rel:.3e} conf {cd:.3e} index {100 * idx:.4f} %")
        assert rel < 1e-3 and cd < 1e-4 and idx < 2e-3, (l, rel, cd, idx)


def test_graphed_equals_eager():
    from casmvsnet_pl_b200.graph import GraphedCascade
    m = _model(1, "tf32")
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=3, W=640, H=512, seed=2)
    imgs, pm = imgs.to(DEV), pm.to(DEV)
    g = GraphedCascade(m, imgs, pm, dmin, dint)
    imgs2, pm2, _, _ = synth.make_inputs(B=1, V=3, W=640, H=512, seed=4)
    out = g(imgs2.to(DEV), pm2.to(DEV))
    with torch.no_grad():
        eager = m(imgs2.to(DEV), pm2.to(DEV), dmin, dint)
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(out[k], eager[k]), k


# ------------------------------------------------------------------------------- training
@pytest.mark.parametrize("loss", ["sl1", "photo"])
def test_training_deterministic_and_eval_ckpt(loss, tmp_path):
    import test_gpu_inverse_depth_train as T
    from casmvsnet_pl_b200 import eval_pipeline as ep, synth_scenes
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
    runs = T._runs(argv + ["--depth_sampling", "adaptive"], tmp_path, "ada")
    uniform = T._runs(argv, tmp_path, "uni", n=1)[0]
    T._same_runs(runs, uniform)
    import json
    for line in open(runs[0] / "logs" / "det" / "metrics.jsonl"):
        rec = json.loads(line)
        for k, v in rec.items():
            if "loss" in k and isinstance(v, float):
                assert np.isfinite(v), (k, v)
    if loss == "photo":
        d = runs[0] / "ckpts" / "det"
        ckpt = str(d / sorted(os.listdir(d))[-1])
        out = tmp_path / "out"
        ep.main(["--dataset_name", "colmap", "--root_dir", root, "--img_wh", "128", "96", "--n_views",
                 "3", "--conf", "0", "--min_geo_consistent", "0", "--out", str(out), "--ckpt", ckpt,
                 "--depth_sampling", "adaptive"])
        assert os.path.getsize(out / "points" / "capture.ply") > 0
