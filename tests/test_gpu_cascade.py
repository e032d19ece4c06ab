"""End-to-end parity of the three-stage cascade on the GPU against the reference's
golden outputs and the oracle, plus full-size (BASELINE cfg2) property checks."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from casmvsnet_pl_b200 import ABN, ops, synth                     # noqa: E402
from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet         # noqa: E402
from oracle import casmvs_oracle as O                             # noqa: E402
from oracle.make_golden import sd_checksum, seeded_state_dict     # noqa: E402

DEV = "cuda:0"


def build(G, precision):
    sd = seeded_state_dict((8, 32, 48), (1, 2, 4), G, seed=0)
    m = CascadeMVSNet(num_groups=G, norm_act=ABN, precision=precision)
    m.load_state_dict(sd)
    return m.eval().to(DEV), sd


def report(tag, res, ref):
    out = {}
    for l in (2, 1, 0):
        d, r = res[f"depth_{l}"].cpu(), ref[f"depth_{l}"]
        rel = ((d - r).abs().mean() / r.abs().mean()).item()
        c = (res[f"confidence_{l}"].cpu() - ref[f"confidence_{l}"]).abs().max().item()
        print(f"{tag} level {l}: depth rel-L1 {rel:.3e}  max|Δ| {(d - r).abs().max():.3e} mm  "
              f"conf max|Δ| {c:.3e}")
        out[l] = rel
    return out


@pytest.mark.parametrize("tag,G", [("var", 1), ("gwc8", 8)])
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_cascade_vs_reference_golden(golden, tag, G, precision):
    g = golden(f"cascade_{tag}_160x128")
    model, sd = build(G, precision)
    if sd_checksum(sd) != float(g["sd_checksum"]):
        pytest.skip("torch RNG/init drifted from the fixture's build; regenerate goldens")
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=3, W=160, H=128, seed=0)
    res = model(imgs.to(DEV), pm.to(DEV), dmin, dint)
    rel = report(f"{tag}/{precision}", res, g)
    # north_star: depth within 1e-3 relative L1 of the reference (fp32)
    for l in (2, 1, 0):
        assert rel[l] < 1e-3
    # abs_err metric (metrics.py:1-3) against a synthetic ground truth placed ~4.5 mm (the
    # reference's DTU validation abs_err, README.md:70) around the reference output: the two
    # implementations' abs_err agree within 1e-3 (relative).  fp32 mode agrees to < 1e-5 mm.
    gen = torch.Generator().manual_seed(1)
    gt = g["depth_0"] + 5.6 * torch.randn(g["depth_0"].shape, generator=gen)
    a = (res["depth_0"].cpu() - gt).abs().mean()
    b = (g["depth_0"] - gt).abs().mean()
    print(f"abs_err ours {a:.6f} mm, reference {b:.6f} mm, signed mean diff "
          f"{(res['depth_0'].cpu() - g['depth_0']).mean():.2e} mm")
    assert abs(a - b) / b < 1e-3
    if precision == "fp32":
        assert abs(a - b) < 1e-5


def test_cascade_tensor_params_batch2(golden):
    g = golden("cascade_var_tensorparams_96x64")
    model, sd = build(1, "fp32")
    if sd_checksum(sd) != float(g["sd_checksum"]):
        pytest.skip("RNG drift")
    imgs, pm, _, _ = synth.make_inputs(B=2, V=3, W=96, H=64, seed=1)
    res = model(imgs.to(DEV), pm.to(DEV), g["init_depth_min"].to(DEV), g["depth_interval"].to(DEV))
    rel = report("tensor-params", res, g)
    assert max(rel.values()) < 1e-3


def test_predict_depth_vs_oracle_cfg1():
    """BASELINE cfg1: single ref view 160x128, 2 src views, 1 stage D=8, variance."""
    model, sd = build(1, "fp32")
    feats = synth.make_level_feats(1, 3, 0, W=160, H=128, seed=3)
    pm = synth.projection_matrices(3, 160, 128)[:, 0].unsqueeze(0)
    dv = O.initial_hypotheses(425.0, 2.65 * 8, 8, 1, 128, 160).contiguous()
    d_ref, c_ref, inter = O.predict_depth(feats, pm, dv, sd, "cost_reg_0.", 1, True)
    d, c = model.predict_depth(feats.to(DEV), pm.to(DEV), dv.to(DEV), model.cost_reg_0)
    rel = ((d.cpu() - d_ref).abs().mean() / d_ref.abs().mean()).item()
    print(f"cfg1 depth rel-L1 {rel:.3e}, conf max|Δ| {(c.cpu() - c_ref).abs().max():.3e}")
    assert rel < 1e-4


# --------------------------------------------------------------------------------------------
# Parity AT THE BENCHMARKED SIZES, both precisions, against the oracle on identical inputs
# (VERDICT r1 weak #1).  The tf32 mode is the one bench.py measures: its size-dependent
# machinery (persistent-CTA item decomposition, depth chunks, Cout slices, side-stream overlap,
# programmatic dependent launch) only exists at these sizes.
FULL_CONFIGS = {
    # BASELINE.json configs[1..4]; cfg4 is ONE of its 8 reference views, cfg5 keeps the
    # V=7 / D=64,32,8 geometry at half resolution (960x544) to bound the oracle's CPU time
    "cfg2": dict(W=640, H=512, V=3, G=1, n_depths=(8, 32, 48)),
    "cfg3_gwc8": dict(W=640, H=512, V=3, G=8, n_depths=(8, 32, 48)),
    "cfg4_view": dict(W=1152, H=864, V=5, G=1, n_depths=(8, 32, 48)),
    "cfg5_half": dict(W=960, H=544, V=7, G=1, n_depths=(8, 32, 64)),
}
_ORACLE_CACHE = {}


def _oracle_full(name):
    if name not in _ORACLE_CACHE:
        c = FULL_CONFIGS[name]
        torch.manual_seed(0)
        m = CascadeMVSNet(n_depths=list(c["n_depths"]), num_groups=c["G"], norm_act=ABN)
        synth.randomize_model_(m, 0)
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        imgs, pm, dmin, dint = synth.make_inputs(B=1, V=c["V"], W=c["W"], H=c["H"], seed=0)
        nt = torch.get_num_threads()
        torch.set_num_threads(min(16, nt))        # oneDNN over-subscribes on the 128-core box
        ref = O.cascade_forward(sd, imgs, pm, dmin, dint, c["n_depths"], (1, 2, 4), c["G"],
                                want_index=True)
        torch.set_num_threads(nt)
        _ORACLE_CACHE[name] = (sd, imgs, pm, dmin, dint, ref)
    return _ORACLE_CACHE[name]


@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("name", list(FULL_CONFIGS))
def test_full_size_parity_vs_oracle(name, precision):
    from casmvsnet_pl_b200 import _lib
    c = FULL_CONFIGS[name]
    sd, imgs, pm, dmin, dint, ref = _oracle_full(name)
    model = CascadeMVSNet(n_depths=list(c["n_depths"]), num_groups=c["G"], norm_act=ABN,
                          precision=precision)
    model.load_state_dict(sd)
    model = model.eval().to(DEV)
    model.return_index = True
    fb0 = _lib.fallback_count()
    res = model(imgs.to(DEV), pm.to(DEV), dmin, dint)
    torch.cuda.synchronize()
    assert _lib.fallback_count() == fb0, "a tf32 layer fell back to the CUDA-core kernel"
    for l in (2, 1, 0):
        d, r = res[f"depth_{l}"].cpu(), ref[f"depth_{l}"]
        rel = ((d - r).abs().mean() / r.abs().mean()).item()
        cd = (res[f"confidence_{l}"].cpu() - ref[f"confidence_{l}"]).abs()
        idx = (res[f"depth_index_{l}"].cpu() != ref[f"depth_index_{l}"]).float().mean().item()
        print(f"{name}/{precision} level {l}: depth rel-L1 {rel:.3e} max|d| {(d - r).abs().max():.3e} mm  "
              f"conf max|d| {cd.max():.3e} mean {cd.mean():.3e}  index mismatch {100 * idx:.4f} %")
        # north_star: depth within 1e-3 relative L1 of the reference
        assert rel < 1e-3
        assert cd.mean().item() < (1e-2 if precision == "tf32" else 1e-4)
        # the index is exact given identical probabilities (test_gpu_kernels.py); through the
        # whole cascade a pixel can flip only when sum(p*d) sits on an integer boundary
        assert idx < (5e-2 if precision == "tf32" else 2e-3)
    # abs_err (metrics.py:1-3) against a synthetic ground truth ~4.5 mm around the reference
    # output: the two implementations' abs_err agree within 1e-3 (north_star)
    gen = torch.Generator().manual_seed(1)
    gt = ref["depth_0"] + 5.6 * torch.randn(ref["depth_0"].shape, generator=gen)
    a = (res["depth_0"].cpu() - gt).abs().mean().item()
    b = (ref["depth_0"] - gt).abs().mean().item()
    print(f"{name}/{precision} abs_err ours {a:.6f} mm, oracle {b:.6f} mm")
    assert abs(a - b) < 1e-3 and abs(a - b) / b < 1e-3
    if precision == "tf32":
        # the benchmarked execution form: CUDA-graph replay == eager, bit for bit
        from casmvsnet_pl_b200.graph import GraphedCascade
        model.return_index = False
        g = GraphedCascade(model, imgs.to(DEV), pm.to(DEV), dmin, dint, warmup=1)
        out = g()
        torch.cuda.synchronize()
        assert torch.equal(out["depth_0"], res["depth_0"])
        assert torch.equal(out["confidence_2"], res["confidence_2"])


def test_full_size_cfg2_properties():
    """640x512, V=3, D=48/32/8: size-independent properties (the oracle needs seconds
    per stage at this size, so only K1 at level 2 is compared directly)."""
    model, sd = build(1, "fp32")
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=3, W=640, H=512, seed=0)
    res = model(imgs.to(DEV), pm.to(DEV), dmin, dint)
    for l, (h, w) in {2: (128, 160), 1: (256, 320), 0: (512, 640)}.items():
        d, c = res[f"depth_{l}"], res[f"confidence_{l}"]
        assert d.shape == (1, h, w) and c.shape == (1, h, w)
        assert torch.isfinite(d).all() and torch.isfinite(c).all()
        assert (c >= 0).all() and (c <= 1 + 1e-5).all()            # Σ of <=4 probabilities
    assert (res["depth_2"] >= dmin).all() and (res["depth_2"] <= dmin + dint * 4 * 47).all()
    # determinism
    res2 = model(imgs.to(DEV), pm.to(DEV), dmin, dint)
    assert all(torch.equal(res[k], res2[k]) for k in res)
    # batch independence of the hot path (data-parallel sharding relies on it):
    # B=2 == 2 x B=1 bit for bit, given the same features (cuDNN may pick a different
    # algorithm per batch size for the 2D FeatureNet, so features are computed once)
    imgs2, pm2, _, _ = synth.make_inputs(B=2, V=3, W=320, H=256, seed=5)
    pm2 = pm2.to(DEV)
    with torch.no_grad():
        f2 = model.feature(imgs2.reshape(6, 3, 256, 320).to(DEV))["level_1"]
        f2 = f2.view(2, 3, *f2.shape[1:])
        dv2 = ops.uniform_hypotheses(dmin, dint * 2, 32, 2, 128, 160, DEV)
        db, cb = model.predict_depth(f2, pm2[:, :, 1], dv2, model.cost_reg_1)
        for i in range(2):
            di, ci = model.predict_depth(f2[i:i + 1], pm2[i:i + 1, :, 1], dv2[i:i + 1],
                                         model.cost_reg_1)
            assert torch.equal(db[i], di[0]) and torch.equal(cb[i], ci[0])
    # K1 at full level-2 size against the oracle
    feats = synth.make_level_feats(1, 3, 2, seed=1)
    pml = pm[:, :, 2]
    dv = O.initial_hypotheses(dmin, dint * 4, 48, 1, 128, 160).contiguous()
    want = O.variance_cost_volume(feats, pml, dv)
    got = ops.warp_cost(feats.to(DEV), pml.to(DEV), dv.to(DEV), 1, ops.NCHW).cpu()
    err = (got - want).abs().max().item()
    print(f"K1 cfg2 level-2 max|err| {err:.3e} (max|ref| {want.abs().max():.2f})")
    # w=160: the reference's own normalise/un-normalise round trip moves a sample by
    # ~2e-5 px; on white-noise features (texel-to-texel jumps up to ~6) that is 1e-4 on a
    # warped value and ~3e-4 on the variance.  The fp64 test in test_gpu_kernels.py shows the
    # kernel is at least as close to exact arithmetic as the reference.
    assert err < 5e-5 * want.abs().max().item() + 1e-4


def test_feature_net_channels_last_matches_oracle():
    model, sd = build(1, "fp32")
    x = torch.randn(2, 3, 64 + 32, 96)
    with torch.no_grad():
        f = model.feature(x.to(DEV))
    ref = O.feature_pyramid(x, sd)
    for k in ref:
        assert ops.is_channels_last_feats(f[k])
        # fp32 mode runs on this library's CUDA-core kernels (no cuDNN): fp32-accurate against
        # the oracle (eval-mode ABN folded into the weights: one extra rounding per weight)
        scale = ref[k].abs().max().item()
        err = (f[k].cpu() - ref[k]).abs().max().item()
        print(k, "max err / scale", err / scale)
        assert err < 1e-5 * scale


def test_feature_net_tensor_path_matches_fp32_path():
    """tf32 mode: 3x3 convs as planar wgmma convolutions + own first block / merges, against
    the fp32 cuDNN path of the same model (10-bit operand mantissas through 8 conv layers)."""
    model, sd = build(1, "tf32")
    x = torch.randn(3, 3, 128, 160)
    with torch.no_grad():
        f = model.feature(x.to(DEV))
        model.set_precision("fp32")
        ref = model.feature(x.to(DEV))
    for k in ref:
        assert ops.is_channels_last_feats(f[k]) and f[k].shape == ref[k].shape
        scale = ref[k].abs().max().item()
        err = (f[k] - ref[k]).abs()
        print(k, "max", err.max().item() / scale, "mean", err.mean().item() / scale)
        assert err.max().item() < 1e-2 * scale and err.mean().item() < 1e-3 * scale


def test_graph_and_pipeline_match_eager():
    """CUDA-graph replay and the host-buffer pipeline (views in flight on separate streams, or
    serial compute) give bit-identical results to eager calls (same kernels per view)."""
    from casmvsnet_pl_b200.graph import GraphedCascade, PipelinedCascade
    model, _ = build(1, "tf32")
    views = [synth.make_inputs(B=1, V=3, W=160, H=128, seed=s) for s in (0, 1, 2, 3, 4)]
    dmin, dint = views[0][2], views[0][3]
    eager = []
    for imgs, pm, _, _ in views:
        r = model(imgs.to(DEV), pm.to(DEV), dmin, dint)
        eager.append((r["depth_0"].cpu(), r["confidence_2"].cpu()))
    g = GraphedCascade(model, views[0][0].to(DEV), views[0][1].to(DEV), dmin, dint)
    for (imgs, pm, _, _), (d, c) in zip(views, eager):
        r = g(imgs.to(DEV), pm.to(DEV))
        assert torch.equal(r["depth_0"].cpu(), d) and torch.equal(r["confidence_2"].cpu(), c)
    # default: three slots, one compute stream per slot (consecutive views overlap on the GPU);
    # and the serial-compute form with two slots
    for kw in ({}, {"slots": 2, "concurrent": False}):
        pipe = PipelinedCascade(model, views[0][0].to(DEV), views[0][1].to(DEV), dmin, dint, **kw)
        # inputs resident in the slots' static buffers (bench.py `value`): every slot replays view 0
        store = torch.empty(7, *eager[0][0].shape[1:], device=DEV)
        last = pipe.run_resident(7, keep=lambda k: store[k:k + 1])
        torch.cuda.synchronize()
        assert torch.equal(last["depth_0"].cpu(), eager[0][0])
        assert all(torch.equal(store[k:k + 1].cpu(), eager[0][0]) for k in range(7))
        got = []
        for rnd in range(2):                        # second round: every slot is being re-used
            for imgs, pm, _, _ in views:
                r = pipe.submit(imgs.pin_memory(), pm.pin_memory())
                if r is not None:
                    got.append((r[0].clone(), r[1].clone()))
        got += [(a.clone(), b.clone()) for a, b in pipe.drain()]
        assert len(got) == 2 * len(views)
        for (d, c), (gd, gc) in zip(eager + eager, got):
            assert torch.equal(gd, d) and torch.equal(gc, c)


def test_weight_image_lifetime_and_graph_generation():
    """ADVICE r1: operand images are tied to their packed buffer, not dropped globally.  A second
    model (new packed buffers) leaves a captured graph of the first one valid; re-packing the
    first model's weights frees its images, which the graph wrapper detects instead of
    replaying a use-after-free."""
    from casmvsnet_pl_b200 import _lib
    from casmvsnet_pl_b200.graph import GraphedCascade
    model, sd = build(1, "tf32")
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=3, W=160, H=128, seed=0)
    imgs, pm = imgs.to(DEV), pm.to(DEV)
    want = {k: v.clone() for k, v in model(imgs, pm, dmin, dint).items()}
    g = GraphedCascade(model, imgs, pm, dmin, dint, warmup=1)
    gen = _lib.weight_cache_generation()
    other, _ = build(8, "tf32")                     # packs 3 more CostRegNets + a FeatureNet
    other(imgs, pm, dmin, dint)                     # (may drop stale images of dead models)
    out = g()                                       # ... which does not invalidate this graph
    assert all(torch.equal(out[k], want[k]) for k in want)
    # in-place edit of a parameter -> re-pack on the next eager call -> old images released
    with torch.no_grad():
        model.cost_reg_0.prob.bias.add_(1.0)
    model(imgs, pm, dmin, dint)
    assert _lib.weight_cache_generation() > gen
    with pytest.raises(_lib.CasMVSError):
        g()
    # the other model's graph is untouched by all of this
    g2 = GraphedCascade(other, imgs, pm, dmin, dint, warmup=1)
    want2 = {k: v.clone() for k, v in other(imgs, pm, dmin, dint).items()}
    del model, g
    out2 = g2()
    assert all(torch.equal(out2[k], want2[k]) for k in want2)


@pytest.mark.parametrize("G", [1, 8])
def test_ladder_fusion_is_bit_identical(G):
    """Generating the hypothesis ladder inside K1 / K3 (fuse_hypotheses) gives exactly the
    outputs of the path that materialises (B,D,h,w) hypotheses through K4, for float and
    tensor-valued depth parameters."""
    model, _ = build(G, "tf32")
    imgs, pm, dmin, dint = synth.make_inputs(B=2, V=3, W=160, H=128, seed=2)
    imgs, pm = imgs.to(DEV), pm.to(DEV)
    tparams = (torch.tensor([[425.0], [431.5]], device=DEV), torch.tensor([[2.65], [2.5]], device=DEV))
    for a, b in ((dmin, dint), tparams):
        model.fuse_hypotheses = True
        model.return_index = True
        fused = {k: v.clone() for k, v in model(imgs, pm, a, b).items()}
        model.fuse_hypotheses = False
        plain = model(imgs, pm, a, b)
        for k in plain:
            assert torch.equal(fused[k], plain[k]), k
    # the Ladder helper itself reproduces K4's tensors bit for bit
    cur = plain["depth_1"]
    lad = ops.Ladder(ops.depth_first(cur, 8, 2.65), 2.65, 8, 2, 128, 160, DEV)
    assert torch.equal(lad.materialize(), ops.depth_hypotheses(cur, 8, 2.65, upsample=True))
