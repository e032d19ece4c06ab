"""Inverse-depth plane sweep on the GPU (README "Wide depth ranges"):

  * K4's inverse hypotheses (full tensor, first rung) equal the float32 restatement of
    oracle/inverse_depth_fp64.py bit for bit: coarse and fine stages, the far clamp, float and
    per-batch device depth parameters, D in {8, 32, 48}, ratios (1, 2, 4) and (1, 2.5, 5.5);
  * rule 1's refusal for device tensors;
  * the fused ladder path and the materialised path give the same depth and confidence bits
    (K3's inverse forward and backward against float64: test_gpu_regress_fp64.py);
  * the cascade in inverse mode against the inverse cascade oracle at 640x512 (V = 3) and
    1152x864 (V = 5), fp32 and tf32, with the full-size parity test's bounds;
  * steps held in CPU tensors are copied to the device;
  * GraphedCascade equals eager; eval_pipeline --depth_sampling inverse on a COLMAP capture."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import ABN, _lib, ops, synth
from oracle import casmvs_oracle as O
from oracle import inverse_depth_fp64 as INV

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _params(kind, B):
    if kind == "float":
        return 1.5, 0.38
    return (torch.tensor([[1.5], [0.9]][:B], device=DEV), torch.tensor([[0.38], [0.61]][:B], device=DEV))


@pytest.mark.parametrize("ratios", [(1, 2, 4), (1, 2.5, 5.5)])
@pytest.mark.parametrize("kind", ["float", "tensor"])
def test_hypotheses_bit_exact(kind, ratios):
    n_depths = (8, 32, 48)
    B = 2
    dmin, dint = _params(kind, B)
    st = ops.inverse_steps(dmin, dint, n_depths, ratios, B, DEV)
    ref = INV.steps_f32(dmin, dint, n_depths, ratios, B)
    g = torch.Generator(device=DEV).manual_seed(1)
    for level, (h, w) in ((2, (32, 40)), (1, (64, 80)), (0, (128, 160))):
        D = n_depths[level]
        if level == 2:
            got = ops.inverse_hypotheses(st, level, D, h, w, DEV)
            want = INV.hypotheses_f32(ref, level, D, h, w)
            assert torch.equal(got.cpu(), torch.from_numpy(np.ascontiguousarray(want))), level
            continue
        cur = 0.9 + 80.0 * torch.rand(B, h // 2, w // 2, generator=g, device=DEV)
        cur[:, :3] = 500.0                                 # far beyond the far plane: clamped
        got = ops.inverse_hypotheses(st, level, D, h, w, DEV, current_depth=cur)
        first = ops.inverse_hypotheses(st, level, D, h, w, DEV, current_depth=cur, first_only=True)
        want = INV.hypotheses_f32(ref, level, D, h, w, cur.cpu().numpy())
        u0 = INV.first_rung_f32(ref, level, D, cur.cpu().numpy())
        assert torch.equal(got.cpu(), torch.from_numpy(np.ascontiguousarray(want))), level
        assert torch.equal(first.cpu(), torch.from_numpy(np.ascontiguousarray(u0))), level
        clamp = INV.first_rung_f32(ref, level, D, np.full((B, 1, 1), 500.0, np.float32))
        assert bool((first[:, :4] == torch.from_numpy(clamp[:, :1, :1]).to(DEV)).all())
        lad = ops.Ladder(first, st.step[level], D, B, h, w, DEV, inverse=True)
        assert torch.equal(lad.materialize(), got)


def test_device_tensor_refusal():
    with pytest.raises(_lib.CasMVSError, match="batch item 0"):
        ops.inverse_steps(torch.tensor([[-1.0], [2.0]], device=DEV),
                          torch.tensor([[1.0], [1.0]], device=DEV), [8, 32, 48], [1, 2, 4], 2)
    with pytest.raises(_lib.CasMVSError, match="batch item 1"):
        ops.inverse_steps(torch.tensor([[1.0], [2.0]], device=DEV),
                          torch.tensor([[1.0], [float("nan")]], device=DEV), [8, 32, 48], [1, 2, 4], 2)


def _model(G=1, precision="fp32", sampling="inverse"):
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(0)
    m = CascadeMVSNet(num_groups=G, norm_act=ABN, precision=precision, depth_sampling=sampling)
    synth.randomize_model_(m, 0)
    return m.eval().to(DEV)


@pytest.mark.parametrize("G", [1, 8])
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("size", [(640, 512, 3), (1152, 864, 5)], ids=["cfg2", "1152x864_V5"])
def test_ladder_equals_materialised(size, precision, G):
    W, H, V = size
    model = _model(G, precision)
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=V, W=W, H=H, seed=3)
    out = {}
    with torch.no_grad():
        for fuse in (True, False):
            model.fuse_hypotheses = fuse
            out[fuse] = model(imgs.to(DEV), pm.to(DEV), dmin, dint)
    for k in out[True]:
        assert torch.equal(out[True][k], out[False][k]), k
    d = out[True]["depth_0"]
    assert bool(torch.isfinite(d).all())


FULL = {   # the benchmarked sizes: test_gpu_cascade.py's FULL_CONFIGS cfg2 and cfg4_view
    "cfg2": dict(W=640, H=512, V=3, G=1),
    "cfg4_view": dict(W=1152, H=864, V=5, G=1),
}
_ORACLE = {}


def _oracle(name):
    if name not in _ORACLE:
        c = FULL[name]
        from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
        torch.manual_seed(0)
        m = CascadeMVSNet(num_groups=c["G"], norm_act=ABN)
        synth.randomize_model_(m, 0)
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        imgs, pm, dmin, dint = synth.make_inputs(B=1, V=c["V"], W=c["W"], H=c["H"], seed=0)
        nt = torch.get_num_threads()
        torch.set_num_threads(min(16, nt))
        ref = INV.cascade_forward_inverse(sd, imgs, pm, dmin, dint, num_groups=c["G"])
        torch.set_num_threads(nt)
        _ORACLE[name] = (sd, imgs, pm, dmin, dint, ref)
    return _ORACLE[name]


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("name", list(FULL))
def test_cascade_inverse_vs_oracle(name, precision):
    """The cascade in inverse mode against the oracle's inverse cascade on the same weights and
    inputs, per stage, with test_gpu_cascade.py::test_full_size_parity_vs_oracle's bounds on the
    depth, the confidence and the index."""
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    sd, imgs, pm, dmin, dint, ref = _oracle(name)
    model = CascadeMVSNet(num_groups=FULL[name]["G"], norm_act=ABN, precision=precision,
                          depth_sampling="inverse")
    model.load_state_dict(sd)
    model = model.eval().to(DEV)
    model.return_index = True
    res = model(imgs.to(DEV), pm.to(DEV), dmin, dint)
    for l in (2, 1, 0):
        d, r = res[f"depth_{l}"].cpu(), ref[f"depth_{l}"]
        rel = float((d - r).abs().mean() / r.abs().mean())
        cd = (res[f"confidence_{l}"].cpu() - ref[f"confidence_{l}"]).abs()
        idx = float((res[f"depth_index_{l}"].cpu() != ref[f"depth_index_{l}"]).float().mean())
        print(f"[inverse cascade] {name}/{precision} level {l}: depth rel-L1 {rel:.3e}  conf mean "
              f"{float(cd.mean()):.3e}  index mismatch {100 * idx:.4f} %")
        assert rel < 1e-3, (l, rel)
        assert float(cd.mean()) < (1e-2 if precision == "tf32" else 1e-4)
        assert idx < (5e-2 if precision == "tf32" else 2e-3)
    # the uniform cascade is a different computation: the inverse mode is not a no-op
    model.set_depth_sampling("uniform")
    assert not torch.equal(model(imgs.to(DEV), pm.to(DEV), dmin, dint)["depth_0"], res["depth_0"])


def test_cpu_steps_are_moved_to_the_device():
    st_cpu = ops.inverse_steps(torch.tensor([[1.5], [0.9]]), torch.tensor([[0.38], [0.61]]),
                               (8, 32, 48), (1, 2, 4), 2)
    st_dev = ops.inverse_steps(torch.tensor([[1.5], [0.9]], device=DEV),
                               torch.tensor([[0.38], [0.61]], device=DEV), (8, 32, 48), (1, 2, 4), 2)
    assert st_cpu.u_near.device.type == "cpu" and st_dev.u_near.is_cuda
    cur = 1.0 + 50 * torch.rand(2, 16, 20, device=DEV)
    for level, cur_l in ((2, None), (1, cur)):
        a = ops.inverse_hypotheses(st_cpu, level, (8, 32, 48)[level], 32, 40, DEV, current_depth=cur_l)
        b = ops.inverse_hypotheses(st_dev, level, (8, 32, 48)[level], 32, 40, DEV, current_depth=cur_l)
        assert torch.equal(a, b)


@pytest.mark.parametrize("kind", ["float", "tensor"])
def test_graphed_cascade_equals_eager(kind):
    from casmvsnet_pl_b200.graph import GraphedCascade
    model = _model(1, "tf32")
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=3, W=640, H=512, seed=2)
    if kind == "tensor":
        dmin = torch.tensor([[float(dmin)]], device=DEV)
        dint = torch.tensor([[float(dint)]], device=DEV)
    imgs, pm = imgs.to(DEV), pm.to(DEV)
    with torch.no_grad():
        eager = model(imgs, pm, dmin, dint)
    g = GraphedCascade(model, imgs, pm, dmin, dint, warmup=1)
    out = g()
    torch.cuda.synchronize()
    for k in eager:
        assert torch.equal(out[k], eager[k]), k


def test_eval_pipeline_colmap_inverse(tmp_path):
    from casmvsnet_pl_b200 import eval_pipeline as ep, io as cio, synth_scenes
    root = tmp_path / "capture"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), depth=3.0, n_points=3000,
                             seed=7)
    out, out_u = tmp_path / "out", tmp_path / "out_uniform"
    args = ["--dataset_name", "colmap", "--root_dir", str(root), "--img_wh", "128", "96",
            "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0"]
    ep.main(args + ["--out", str(out), "--depth_sampling", "inverse"])
    ep.main(args + ["--out", str(out_u)])
    assert os.path.getsize(out / "points" / "capture.ply") > 0
    metas = cio.read_pair_file(str(out / "capture" / "pair.txt"))
    assert len(metas) == 8
    for ref, _ in metas:
        assert os.path.isfile(out / "capture" / "cams" / f"{ref:08d}_cam.txt")
    depth_files = [f for _, _, fs in os.walk(out / "depth") for f in fs
                   if f.startswith("depth_") and f.endswith(".pfm")]
    assert len(depth_files) == 8, depth_files
    # the flag reached the model: the same weights and views give other depth maps
    f = sorted(depth_files)[0]
    inv = cio.read_pfm(str(out / "depth" / "capture" / f))[0]
    uni = cio.read_pfm(str(out_u / "depth" / "capture" / f))[0]
    assert inv.shape == uni.shape and not np.array_equal(inv, uni)
