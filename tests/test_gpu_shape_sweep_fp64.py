"""The cascade element by element against float64 at the depth counts, image sizes, group counts,
view counts and batch sizes the command lines accept, not only at the benchmarked ones.

Each case of CASES names the edges it exists for; test_case_table_edges asserts every one of
them by construction (odd D/8, many depth chunks, the conv5 output dims, h % 16, ...).  At every
case, CascadeMVSNet(precision="tf32").eval() with fuse_hypotheses runs its real stage path
(ladder K1 + blocked CostRegNet + fused tail + regress_ladder where the staged K1 kernel covers
the stage, materialised hypotheses + gather K1 + channels-last CostRegNet otherwise), with every
library call recorded.  Then:

  * every FeatureNet, K1, K3 and K4 call against its float64 oracle on the call's own inputs, at
    the committed EPS / LOOSE_CEIL of test_gpu_featurenet_fp64, test_gpu_warp_cost_fp64 and
    test_gpu_regress_fp64 (imported); K1's TF32-rounded store equals tf32_rna of the unrounded
    output bit for bit;
  * every CostRegNet call re-run by casmvs_costreg_fwd on its recorded input and parameters with
    a caller-owned NaN-filled workspace and the two-layer conv11 -> prob path: its logits equal
    the cascade's (the fused tail, where it ran) as int32, and every layer of every batch element
    is checked against float64 by test_gpu_cfg5_batch_fp64.check_costreg_elements.  conv0 of a
    4-channel input (num_groups 4, and 2 zero-padded to 4) has no tensor-core kernel: the test
    asserts it is the only layer on the CUDA-core kernel and checks it at the `direct` eps;
  * four cases again in the fp32 precision; the B = 3 cases equal three B = 1 forwards bit for
    bit (test_gpu_cfg5_batch_fp64's call digests name the first library call that differs);
  * the *_inv cases with the inverse-depth sweep (README "Wide depth ranges"), together over
    G in {1, 2, 4, 8}, V in {2, 3, 4, 9}, odd D/8, D = 192, 32x32 and 2048x96, B = 3 with
    distinct (B, 1) depth ranges, interval ratios (1, 2.5, 5.5) and a far / near ratio >= 10
    (wide_range).  K1 takes its hypotheses from INV.ladder_f32, K3 and K4 the inverse checks of
    test_gpu_regress_fp64; FeatureNet's calls must equal the uniform run's bit for bit, and
    CostRegNet's fused tail the two-layer re-run bit for bit, per element on costreg_fp64 cases;
  * odd-D stage shapes under CASMVS_TMA_DCHUNK = 1, 2, 3 in child processes: every layer within
    eps and the fused tail bit-identical to the two-layer path under every chunking;
  * a training step at num_groups 2, num_groups 4 and D = 8 / 24 / 56 with 4 views, through
    test_gpu_train_step_fp64's recorder (forward, dgrad and wgrad of every CostRegNet conv, K1,
    K3 and their backward), and train.py / eval_pipeline runs with --num_groups 2.

The CPU part checks the edge predicates of the case table and that the per-layer check fails,
naming the layer and the plane, on simulated workspaces whose last depth chunk of an odd-D layer
holds one wrong plane or whose last plane was never written."""
import os
import subprocess
import sys
import time

import pytest
import torch

import test_gpu_cfg5_batch_fp64 as CFG5
import test_gpu_conv_fp64 as CONV_T
import test_gpu_featurenet_fp64 as FEAT_T
import test_gpu_regress_fp64 as REG_T
import test_gpu_train_step_fp64 as TS
import test_gpu_warp_cost_fp64 as K1_T
from casmvsnet_pl_b200 import ABN, _lib, ops, synth
from oracle import conv3d_fp64 as R
from oracle import warp_cost_fp64 as W
from test_gpu_train_step_fp64 import rec  # noqa: F401  (fixture)

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ------------------------------------------------------------------------------- case table
# name: image W, H, views V, num_groups G, depths per stage (fine -> coarse), batch B, an fp32
# pass too, and the edges the case exists for (EDGES)
CASES = {
    "32x32_d8": dict(W=32, H=32, V=2, G=1, Ds=(8, 8, 8), B=1, fp32=True,
                     edges=("d8_every_stage", "conv5_1x1")),
    "32x32_g8_b3": dict(W=32, H=32, V=3, G=8, Ds=(8, 16, 24), B=3, fp32=False,
                        edges=("d8_odd", "conv5_1x1", "batch3")),
    "1184x800_d24_d40": dict(W=1184, H=800, V=3, G=1, Ds=(8, 24, 40), B=1, fp32=True,
                             edges=("d8_odd", "tail_partial_chunk", "conv5_37x25", "h16_partial")),
    "800x608_g4_v4_d56": dict(W=800, H=608, V=4, G=4, Ds=(8, 32, 56), B=1, fp32=True,
                              edges=("d8_odd", "conv5_25x19", "h16_partial")),
    "800x608_g2_b3": dict(W=800, H=608, V=3, G=2, Ds=(16, 32, 48), B=3, fp32=False,
                          edges=("conv5_25x19", "h16_partial", "batch3")),
    "1152x864_d192": dict(W=1152, H=864, V=3, G=1, Ds=(8, 32, 192), B=1, fp32=False,
                          edges=("many_chunks",)),
    "640x512_g8_d40_d96": dict(W=640, H=512, V=2, G=8, Ds=(8, 40, 96), B=1, fp32=False,
                               edges=("d8_odd", "many_chunks", "tail_partial_chunk")),
    "768x576_v9_d128": dict(W=768, H=576, V=9, G=1, Ds=(16, 64, 128), B=1, fp32=False,
                            edges=("many_chunks", "generic_k1")),
    "1600x1184_dtu_full": dict(W=1600, H=1184, V=3, G=1, Ds=(8, 32, 48), B=1, fp32=False,
                               edges=("h16_partial",)),
    "2048x96_g2_aspect": dict(W=2048, H=96, V=2, G=2, Ds=(8, 24, 56), B=1, fp32=True,
                              edges=("aspect", "d8_odd")),
    "2560x1440_large": dict(W=2560, H=1440, V=2, G=1, Ds=(8, 32, 48), B=1, fp32=False,
                            edges=("large",)),
    "960x544_g4_v9_d56": dict(W=960, H=544, V=9, G=4, Ds=(8, 56, 24), B=1, fp32=False,
                              edges=("d8_odd", "generic_k1")),
    # the inverse-depth sweep; depth=(init_depth_min, depth_interval) where not synth's DTU range
    "32x32_g8_b3_inv": dict(W=32, H=32, V=3, G=8, Ds=(8, 16, 24), B=3, fp32=False,
                            sampling="inverse", costreg_fp64=True,
                            edges=("d8_odd", "conv5_1x1", "batch3")),
    "2048x96_g2_wide_inv": dict(W=2048, H=96, V=2, G=2, Ds=(8, 24, 56), B=1, fp32=False,
                                sampling="inverse", depth=(100.0, 1400.0 / (55 * 4)),
                                edges=("aspect", "d8_odd", "wide_range")),
    "800x608_g4_v4_ratios_inv": dict(W=800, H=608, V=4, G=4, Ds=(8, 32, 56), B=1, fp32=False,
                                     sampling="inverse", ratios=(1, 2.5, 5.5),
                                     edges=("d8_odd", "conv5_25x19")),
    "1152x864_d192_inv": dict(W=1152, H=864, V=3, G=1, Ds=(8, 32, 192), B=1, fp32=False,
                              sampling="inverse", edges=("many_chunks",)),
    "960x544_g4_v9_inv": dict(W=960, H=544, V=9, G=4, Ds=(8, 56, 24), B=1, fp32=False,
                              sampling="inverse", edges=("d8_odd", "generic_k1")),
}
INV_CASES = [n for n, c in CASES.items() if c.get("sampling") == "inverse"]
TAIL_CHUNK = 16            # the fused tail's largest depth chunk, in u9 slices (conv3d_tail.cu)


def stages(c):
    """level -> (Cin as CostRegNet takes it, D, h, w); level 2 is the coarse stage."""
    return {l: (c["G"] if c["G"] > 1 else 8 << l, c["Ds"][l], c["H"] >> l, c["W"] >> l)
            for l in range(3)}


def depth_range(c):
    """(near, far) of the coarse stage: init_depth_min and its last uniform plane."""
    dmin, dint = c.get("depth", (synth.DEPTH_MIN, synth.DEPTH_INTERVAL))
    return dmin, dmin + (c["Ds"][2] - 1) * dint * c.get("ratios", (1, 2, 4))[2]


def conv5_dims(c):
    """(w, h) of conv5's output at the coarse stage."""
    _, _, h, w = stages(c)[2]
    return w // 8, h // 8


EDGES = {
    "d8_every_stage": lambda c: all(D == 8 for _, D, _, _ in stages(c).values()),
    "d8_odd": lambda c: any(D // 8 % 2 == 1 and D > 8 for _, D, _, _ in stages(c).values()),
    "many_chunks": lambda c: stages(c)[2][1] >= 96,
    "tail_partial_chunk": lambda c: any(D // 2 > TAIL_CHUNK and D // 2 % TAIL_CHUNK
                                        for _, D, _, _ in stages(c).values()),
    "conv5_1x1": lambda c: conv5_dims(c) == (1, 1),
    "conv5_37x25": lambda c: conv5_dims(c) == (37, 25),
    "conv5_25x19": lambda c: conv5_dims(c) == (25, 19),
    "h16_partial": lambda c: conv5_dims(c)[1] % 16 != 0 and conv5_dims(c)[1] > 16,
    "aspect": lambda c: c["W"] >= 16 * c["H"],
    "large": lambda c: c["W"] * c["H"] >= 2560 * 1440,
    "batch3": lambda c: c["B"] == 3,
    # 8 source views: no gather instantiation (1, 2, 4, 6 sources), the run-time-V kernel
    "generic_k1": lambda c: c["V"] - 1 not in (1, 2, 4, 6),
    # the range the inverse sweep exists for
    "wide_range": lambda c: depth_range(c)[1] >= 10 * depth_range(c)[0],
}
RUNS = [(n, "tf32") for n in CASES] + [(n, "fp32") for n, c in CASES.items() if c["fp32"]]
BATCH_CASES = [n for n, c in CASES.items() if c["B"] > 1]
RECORDED = FEAT_T.RECORDED + REG_T.RECORDED + ("warp_cost", "warp_cost_ladder", "costreg")
SUMMARY = {}           # (case, precision) -> {family: worst eps needed}


# ------------------------------------------------------------------------------- recording
@pytest.fixture
def sweep_rec(monkeypatch):
    """Records (name, args, kwargs, output, fallback launches) of every library call of the
    inference path; .orig holds the unpatched functions (FeatureNet's check re-runs some)."""
    calls = []
    orig = {n: getattr(ops, n) for n in RECORDED}

    def wrap(name):
        def f(*a, **k):
            f0 = _lib.fallback_count()
            out = orig[name](*a, **k)
            calls.append((name, a, k, out, _lib.fallback_count() - f0))
            return out
        return f
    for n in RECORDED:
        monkeypatch.setattr(ops, n, wrap(n))
    return FEAT_T._Rec(calls, orig)


def _model(c, precision):
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(0)
    m = CascadeMVSNet(n_depths=list(c["Ds"]), interval_ratios=list(c.get("ratios", (1, 2, 4))),
                      num_groups=c["G"], norm_act=ABN, precision=precision,
                      depth_sampling=c.get("sampling", "uniform"))
    synth.randomize_model_(m, 0)
    m = m.eval().to(DEV)
    m.return_index = True
    return m


def _note(worst, fam, need):
    worst[fam] = max(worst.get(fam, 0.0), need)


# ------------------------------------------------------------------------------- per-call checks
def check_k1_call(tag, rec_, name, a, k, out, worst):
    feats, P, hyp, G = a[:4]
    rnd = k.get("round_tf32", False)
    B, V, C, h, w = feats.shape
    if name == "warp_cost_ladder":
        y = R.from_blocked(out) if k.get("blocked", False) else ops.volume_storage(out)
        dv, fam = REG_T.ladder_hyp(hyp), "staged"
        unrounded = lambda: rec_.orig[name](feats, P, hyp, G, round_tf32=False)   # noqa: E731
    else:
        y, dv = ops.volume_storage(out), hyp
        fam = "staged" if ops.ladder_supported(V, C, G) else "gather"
        unrounded = lambda: rec_.orig[name](feats, P, hyp, G, ops.NHWC)           # noqa: E731
    if rnd:
        y0 = ops.volume_storage(unrounded())
        assert torch.equal(y.contiguous().view(torch.int32),
                           W.tf32_rna(y0.contiguous()).view(torch.int32)), \
            f"{tag}: TF32-rounded cost volume differs from tf32_rna of the unrounded one"
        y = y0
    rep = W.check_cost(y, feats.permute(0, 1, 3, 4, 2).contiguous(), P, dv, G, K1_T.EPS[fam])
    _note(worst, f"k1_{fam}", rep.eps_needed)
    print(f"[sweep] {tag} [{fam}]: {rep.describe()}")
    assert rep.ok, f"{tag} [{fam}]: {rep.describe()}"
    assert rep.loose_share <= K1_T.LOOSE_CEIL["cost"], f"{tag} [{fam}] loose: {rep.describe()}"


def costreg_kernels(cin, tf32):
    """The eps family of each CostRegNet layer's kernel: the CUDA-core kernel in fp32 and where
    no tensor-core kernel covers the layer."""
    out = []
    for i in range(11):
        L = ops.costreg_layer_info(cin, i)
        tc = tf32 and ops.conv3d_tensor_core(L["cin"], L["cout"], L["kind"], L["stride"],
                                             i in CONV_T._SKIP)
        out.append(("tma" if L["stride"] == 1 else "tma2") if tc else "direct")
    return out


def costreg_layers(params, cin, kernels):
    """CFG5.costreg_layers, with the fp32 weights where the CUDA-core kernel multiplies them."""
    layers = CFG5.costreg_layers(params, cin)
    for L, kern in zip(layers, kernels):
        if kern == "direct":
            L["w"] = params[L["w_off"]:L["w_off"] + 27 * L["cin"] * L["cout"]].view(
                27, L["cin"], L["cout"])
    return layers


def rerun_costreg(x, params, cin, precision, blocked_in, B, D, h, w):
    """casmvs_costreg_fwd, two-layer tail, caller-owned NaN-filled workspace -> ws, logits,
    fallback launches."""
    lib = _lib.load()
    ws_bytes = lib.casmvs_costreg_workspace_bytes(B, cin, D, h, w)
    ws = torch.full((ws_bytes // 4,), float("nan"), device=DEV)
    logits = torch.empty(B, D, h, w, device=DEV)
    f0 = _lib.fallback_count()
    _lib.check(lib.casmvs_costreg_fwd(ops._ptr(x), ops._ptr(params), ops._ptr(logits), B, cin, D,
                                      h, w, precision | (ops.BLOCKED if blocked_in else 0),
                                      ops._ptr(ws), ws_bytes, ops._stream()), "costreg")
    torch.cuda.synchronize()
    return ws, logits, _lib.fallback_count() - f0


def _assert_bits(tag, got, want):
    diff = got.view(torch.int32) != want.view(torch.int32)
    assert not diff.any(), (f"{tag}: {int(diff.sum())} of {diff.numel()} logits differ, first at "
                            f"(b,d,h,w)={tuple(int(i) for i in diff.nonzero()[0])}")


def _clone(out):
    if torch.is_tensor(out):
        return out.clone()
    if isinstance(out, (tuple, list)):
        return type(out)(_clone(t) for t in out)
    return out


def _same_bits(x, y):
    if torch.is_tensor(x):
        return torch.is_tensor(y) and x.shape == y.shape and torch.equal(
            x.contiguous().view(torch.int32), y.contiguous().view(torch.int32))
    if isinstance(x, (tuple, list)):
        return len(x) == len(y) and all(_same_bits(a, b) for a, b in zip(x, y))
    return x == y


def check_costreg_call(tag, a, k, out, fb, G, worst, elements=True):
    x, params, cin = a[:3]
    prec = a[3] if len(a) > 3 else k.get("precision", ops.FP32)
    blocked_in = k.get("blocked", False)
    tf32 = prec == ops.TF32
    kernels = costreg_kernels(cin, tf32)
    direct = {i for i, kern in enumerate(kernels) if kern == "direct"}
    # only conv0 of a 4-channel input lacks a tensor-core kernel
    want = set(range(11)) if not tf32 else {0} if cin == 4 else set()
    assert direct == want, f"{tag}: CUDA-core layers {sorted(direct)}, want {sorted(want)}"
    assert fb == (len(direct) if tf32 else 0), f"{tag}: {fb} fallback launches"
    ws_blocked = ops.costreg_blocked_supported(cin, prec)
    assert ws_blocked == (tf32 and not direct)
    assert ws_blocked or not blocked_in
    xs = x if blocked_in else ops.volume_storage(x)
    B, D, h, w = out.shape
    if G == 2:
        # the padding leaves the function unchanged: zero input channels, zero weight rows
        xl = R.from_blocked(xs) if blocked_in else xs
        assert cin == 4 and not xl[..., 2:].any(), f"{tag}: padded channels are not zero"
        L0 = ops.costreg_layer_info(cin, 0)
        w0 = params[L0["w_off"]:L0["w_off"] + 27 * 4 * 8].view(27, 4, 8)
        assert not w0[:, 2:].any() and w0[:, :2].any(), f"{tag}: conv0's padded weight rows"
    ws, logits, fb2 = rerun_costreg(xs, params, cin, prec, blocked_in, B, D, h, w)
    assert fb2 == fb, f"{tag}: re-run made {fb2} fallback launches, the cascade {fb}"
    tail = bool(_lib.load().casmvs_costreg_tail_supported(cin, prec))
    _assert_bits(f"{tag} {'fused tail' if tail else 'logits'} vs two-layer re-run", out, logits)
    if not elements:
        return tail
    # the driver stores its activations blocked wherever every layer has a tensor-core kernel,
    # whatever the input's layout
    xb = R.to_blocked(xs) if ws_blocked and not blocked_in else xs
    need =CFG5.check_costreg_elements(tag, xb, ws, logits, costreg_layers(params, cin, kernels),
                                       B, D, h, w, range(B), blocked=ws_blocked, kernels=kernels,
                                       tf32=tf32)
    for fam, v in need.items():
        _note(worst, fam, v)
    return tail


# ------------------------------------------------------------------------------- GPU: cascade
@pytest.mark.gpu
@pytest.mark.parametrize("case,precision", RUNS, ids=[f"{n}-{p}" for n, p in RUNS])
def test_cascade_calls_vs_fp64(case, precision, sweep_rec, monkeypatch):
    c = CASES[case]
    monkeypatch.setattr(FEAT_T, "WORST", {})
    monkeypatch.setattr(REG_T, "WORST", {})
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    model = _model(c, precision)
    imgs, pm, dmin, dint = synth.make_inputs(B=c["B"], V=c["V"], W=c["W"], H=c["H"], seed=c["B"])
    inverse = c.get("sampling") == "inverse"
    dmin, dint = c.get("depth", (dmin, dint))
    if inverse and c["B"] > 1:           # per-item ranges: the ladders' first_b / step_b
        dmin = torch.tensor([[dmin + 2.5 * i] for i in range(c["B"])], device=DEV)
        dint = torch.tensor([[dint * (1.0 + 0.05 * i)] for i in range(c["B"])], device=DEV)
    f0 = _lib.fallback_count()
    model(imgs.to(DEV), pm.to(DEV), dmin, dint)
    torch.cuda.synchronize()
    n_fb = _lib.fallback_count() - f0
    calls = list(sweep_rec.calls)
    sweep_rec.calls.clear()
    names = [cl[0] for cl in calls]
    counts = {n: names.count(n) for n in FEAT_T.RECORDED if n in names}
    assert counts == FEAT_T.CHAIN[precision], counts
    # FeatureNet level l has 8 << l channels
    ladder = {l: ops.ladder_supported(c["V"], 8 << l, c["G"]) for l in range(3)}
    k1 =[n for n in names if n in ("warp_cost", "warp_cost_ladder")]
    assert k1 == ["warp_cost_ladder" if ladder[l] else "warp_cost" for l in (2, 1, 0)], k1
    assert names.count("costreg") == 3
    tag = f"{case} {precision}"
    worst = {}
    tails = 0
    if inverse:
        # the same images through FeatureNet: the uniform run's calls, bit for bit
        feat = [(n, _clone(out)) for n, _, _, out, _ in calls if n in FEAT_T.RECORDED]
        model.set_depth_sampling("uniform")
        model(imgs.to(DEV), pm.to(DEV), dmin, dint)
        torch.cuda.synchronize()
        uni = [(n, out) for n, _, _, out, _ in sweep_rec.calls if n in FEAT_T.RECORDED]
        sweep_rec.calls.clear()
        assert [n for n, _ in feat] == [n for n, _ in uni], tag
        for i, ((n, x), (_, y)) in enumerate(zip(feat, uni)):
            assert _same_bits(x, y), f"{tag}: FeatureNet call {i} ({n}) differs from the uniform run"
    for name, a, k, out, fb in calls:
        if name in FEAT_T.RECORDED:
            if not inverse:
                FEAT_T.check_call(sweep_rec, name, a, k, out, tag)
                torch.cuda.empty_cache()
        elif name in REG_T.RECORDED:
            REG_T.check_call(name, a, k, out, tag)
        elif name == "costreg":
            D = out.shape[1]
            tails += check_costreg_call(f"{tag} costreg D={D} {tuple(out.shape[2:])} B={c['B']}",
                                        a, k, out, fb, c["G"], worst,
                                        elements=c.get("costreg_fp64", not inverse))
            torch.cuda.empty_cache()
        else:
            check_k1_call(f"{tag} {name} D={a[2].D if name == 'warp_cost_ladder' else a[2].shape[1]}"
                          f" {tuple(a[0].shape[3:])}", sweep_rec, name, a, k, out, worst)
    want_fb = 3 if precision == "tf32" and c["G"] in (2, 4) else 0
    assert n_fb == want_fb, f"{tag}: {n_fb} fallback launches in the forward, want {want_fb}"
    if precision == "tf32" and c["G"] in (1, 8):
        assert tails == 3, f"{tag}: the fused tail ran at {tails} of 3 stages"
    for fam, v in list(FEAT_T.WORST.items()) + list(REG_T.WORST.items()):
        _note(worst, fam, v)
    SUMMARY[(case, precision)] = worst
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"[sweep] {tag}: {len(calls)} calls checked in {time.time() - t0:.1f} s, peak "
          f"allocated {peak:.1f} GiB; worst eps needed: "
          + ", ".join(f"{f} {v:.2e}" for f, v in sorted(worst.items())))


@pytest.mark.gpu
@pytest.mark.parametrize("case", BATCH_CASES)
def test_batch_equals_single_forwards(case, monkeypatch):
    c = CASES[case]
    B = c["B"]
    model = _model(c, "tf32")
    # each view with its own (1, 1) depth range tensors
    views = [CFG5._view(c, i) for i in range(B)]
    rec_ = CFG5._CallDigests(monkeypatch)
    singles, records = [], []
    for v in views:
        rec_.record()
        singles.append(model(*v))
        records.append(rec_.stop())
    inputs = [torch.cat([v[j] for v in views]) for j in range(4)]
    rec_.record(records)
    batched = model(*inputs)
    calls = rec_.stop()
    torch.cuda.synchronize()
    assert not torch.equal(singles[0]["depth_0"], singles[-1]["depth_0"])   # distinct views
    for i in range(B):
        for l in (0, 1, 2):
            for key in (f"depth_{l}", f"confidence_{l}"):
                got, want = batched[key][i], singles[i][key][0]
                if not torch.equal(got, want):
                    diff = got != want
                    pytest.fail(f"{case}: view {i} {key} differs from the single-view forward at "
                                f"{int(diff.sum())} of {diff.numel()} pixels; "
                                f"{CFG5._first_difference(records[i], calls, i)}")
        assert CFG5._first_difference(records[i], calls, i) == "every recorded library call agrees"


# ------------------------------------------------------------------------------- GPU: chunkings
# odd-D stage shapes of the table, blocked (G = 1 or 8): Cin, B, D, h, w
DCHUNK_SHAPES = {
    "1184x800_stage1_d40": (32, 1, 40, 200, 296),
    "640x512_g8_stage2_d40": (8, 1, 40, 256, 320),
    "32x32_g8_stage1_d24_b3": (8, 3, 24, 8, 8),
}


def dchunk_child():
    """In a child process under CASMVS_TMA_DCHUNK: each shape's layers within eps and the fused
    tail bit-identical to the two-layer path."""
    for name, (cin, B, D, h, w) in DCHUNK_SHAPES.items():
        x = CFG5._blocked_input(cin * 1000 + D + B, cin, B, D, h, w)
        params = CONV_T._net_params(cin)
        ws, logits, fb = rerun_costreg(x, params, cin, ops.TF32, True, B, D, h, w)
        assert fb == 0
        fused = ops.costreg(x, params, cin, ops.TF32, blocked=True, fused_tail=True)
        torch.cuda.synchronize()
        assert torch.isfinite(logits).all() and logits.std() > 0
        _assert_bits(f"{name} fused tail", fused, logits)
        need = CFG5.check_costreg_elements(name, x, ws, logits, CFG5.costreg_layers(params, cin),
                                           B, D, h, w, range(B))
        print(f"[sweep] dchunk {os.environ.get('CASMVS_TMA_DCHUNK')} {name}: worst eps needed "
              + ", ".join(f"{f} {v:.2e}" for f, v in sorted(need.items())), flush=True)


@pytest.mark.gpu
@pytest.mark.parametrize("dchunk", [1, 2, 3])
def test_odd_depths_under_every_chunking(dchunk):
    code = ("import sys, torch\n"
            "sys.path.insert(0, %r)\n"
            "sys.path.insert(0, %r)\n"
            "import test_gpu_shape_sweep_fp64 as T\n"
            "with torch.no_grad():\n"
            "    T.dchunk_child()\n" % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, CASMVS_TMA_DCHUNK=str(dchunk))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True,
                       timeout=900)
    print("\n".join(ln for ln in r.stdout.splitlines() if "worst" in ln or "sweep" in ln))
    assert r.returncode == 0, f"CASMVS_TMA_DCHUNK={dchunk}:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"


# ------------------------------------------------------------------------------- GPU: training
TRAIN_CASES = {   # name: W, H, V, G, n_depths
    "dtu_g2": (640, 512, 3, 2, (8, 32, 48)),
    "dtu_g4": (640, 512, 3, 4, (8, 32, 48)),
    "blendedmvs_v4_d8_24_56": (768, 576, 4, 1, (8, 24, 56)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(TRAIN_CASES))
def test_training_step_vs_fp64(case, rec):  # noqa: F811
    from casmvsnet_pl_b200 import train
    W_, H, V, G, Ds = TRAIN_CASES[case]
    a = train.build_parser().parse_args(["--precision", "tf32", "--optimizer", "sgd",
                                         "--num_groups", str(G), "--n_views", str(V),
                                         "--n_depths", *map(str, Ds)])
    with torch.enable_grad():
        torch.manual_seed(0)
        model = train.build_model(a, DEV)
        tr = train.Trainer(a, model, DEV)
        f0 = _lib.fallback_count()
        loss, _ = tr.train_step(TS._sample(1, W_, H, seed=3, V=V))
        torch.cuda.synchronize()
    n_fb = _lib.fallback_count() - f0
    assert torch.isfinite(loss).item()
    print(f"[sweep] train {case}: {W_}x{H} V={V} G={G} D={Ds}: loss {loss.item():.5f}")
    fallbacks = TS._check_conv_calls(case, rec, True)
    want = TS._expected_fallbacks(True, G)
    assert fallbacks == want, f"{case}: fallback layers {sorted(fallbacks)}, want {sorted(want)}"
    assert n_fb == len(want), f"{case}: {n_fb} fallback launches in the step, want {len(want)}"
    TS._check_k1_k3(case, rec)


@pytest.mark.gpu
def test_train_cli_runs_with_two_groups(tmp_path, monkeypatch):
    """A short train.py run with --num_groups 2 on the synthetic DTU fixture: finite losses, and
    the checkpoint holds the reference's (8, 2, 3, 3, 3) conv0 and loads for evaluation."""
    from casmvsnet_pl_b200 import InPlaceABN, eval_pipeline, train
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    from casmvsnet_pl_b200.synth_scenes import make_dtu_train
    from oracle.make_golden_train import FIXTURE_SEED
    import json
    root = make_dtu_train(str(tmp_path / "dtu"), seed=FIXTURE_SEED)
    monkeypatch.chdir(tmp_path)
    with torch.enable_grad():
        train.main(["--root_dir", root, "--train_list", os.path.join(root, "lists", "train.txt"),
                    "--val_list", os.path.join(root, "lists", "val.txt"), "--num_groups", "2",
                    "--num_epochs", "1", "--precision", "tf32", "--optimizer", "adam",
                    "--num_workers", "2", "--seed", "0", "--exp_name", "g2"])
    recs = [json.loads(ln) for ln in open(tmp_path / "logs" / "g2" / "metrics.jsonl")]
    losses = [r["train/loss"] for r in recs if "train/loss" in r]
    assert losses and all(l == l and abs(l) < float("inf") for l in losses), losses
    ckpts = sorted((tmp_path / "ckpts" / "g2").glob("*.ckpt"))
    assert ckpts
    model = CascadeMVSNet(num_groups=2, norm_act=InPlaceABN, precision="tf32")
    model = eval_pipeline.load_checkpoint(model, str(ckpts[0]))
    for l in range(3):
        assert tuple(getattr(model, f"cost_reg_{l}").conv0.conv.weight.shape) == (8, 2, 3, 3, 3)
    model = model.eval().to(DEV)
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=3, W=640, H=512, seed=1)
    out = model(imgs.to(DEV), pm.to(DEV), dmin, dint)
    assert all(bool(torch.isfinite(out[f"depth_{l}"]).all()) for l in range(3))


@pytest.mark.gpu
def test_eval_pipeline_colmap_runs_with_two_groups(tmp_path):
    from casmvsnet_pl_b200 import eval_pipeline as ep
    from casmvsnet_pl_b200 import synth_scenes
    root = tmp_path / "capture"
    synth_scenes.make_colmap(str(root), n_views=6, image_wh=(160, 120), depth=3.0,
                             n_points=3000, seed=7, fmt="both")
    out = tmp_path / "out"
    ep.main(["--dataset_name", "colmap", "--root_dir", str(root), "--out", str(out),
             "--img_wh", "128", "96", "--n_views", "3", "--conf", "0", "--min_geo_consistent",
             "0", "--num_groups", "2", "--n_depths", "8", "24", "40"])
    assert os.path.getsize(out / "points" / "capture.ply") > 0


@pytest.mark.gpu
def test_zz_print_worst():
    """Worst eps needed per kernel family and case (runs last in file order)."""
    eps = {**{f"k1_{k}": v for k, v in K1_T.EPS.items()}, **CONV_T.EPS, **REG_T.EPS}
    eps.update({f: v for f, v in FEAT_T.EPS.items() if f not in ("tma", "tma2", "direct")})
    for (case, prec), worst in sorted(SUMMARY.items()):
        print(f"[sweep] {case} {prec}: " + ", ".join(
            f"{f} {v:.2e} (eps {eps.get(f, float('nan')):.1e})" for f, v in sorted(worst.items())))


# ------------------------------------------------------------------------------- CPU
def test_case_table_edges():
    """Every edge a case names holds by construction, and the table covers the ranges."""
    for name, c in CASES.items():
        assert c["W"] % 32 == 0 and c["H"] % 32 == 0, name
        assert all(D > 0 and D % 8 == 0 for D in c["Ds"]), name
        for e in c["edges"]:
            assert EDGES[e](c), f"{name}: edge {e} does not hold"
    cs = list(CASES.values())
    assert {c["G"] for c in cs} == {1, 2, 4, 8}
    assert {c["V"] for c in cs} >= {2, 3, 4, 9}
    assert {c["B"] for c in cs} == {1, 3} and sum(c["B"] == 3 for c in cs) >= 2
    assert {D for c in cs for D in c["Ds"] if D // 8 % 2 and D > 8} >= {24, 40, 56}
    assert {c["Ds"][2] for c in cs} >= {96, 128, 192}
    assert any(c["Ds"][2] == 192 and (c["W"], c["H"]) == (1152, 864) for c in cs)
    assert {(c["W"], c["H"]) for c in cs} >= {(32, 32), (1184, 800), (800, 608), (1600, 1184),
                                              (2048, 96), (2560, 1440)}
    assert conv5_dims(CASES["1184x800_d24_d40"]) == (37, 25)
    assert conv5_dims(CASES["800x608_g4_v4_d56"]) == (25, 19)
    assert conv5_dims(CASES["32x32_d8"]) == (1, 1) and stages(CASES["32x32_d8"])[2][2:] == (8, 8)
    assert 3 <= len([r for r in RUNS if r[1] == "fp32"]) <= 4
    for name, (cin, B, D, h, w) in DCHUNK_SHAPES.items():
        assert D // 8 % 2 == 1 and D > 8 and h % 8 == 0 and w % 8 == 0, name
    assert TRAIN_CASES["blendedmvs_v4_d8_24_56"][4][1] // 8 % 2 == 1
    inv = [CASES[n] for n in INV_CASES]
    assert {c["G"] for c in inv} == {1, 2, 4, 8} and {c["V"] for c in inv} >= {2, 3, 4, 9}
    assert any(D // 8 % 2 and D > 8 for c in inv for D in c["Ds"])
    assert any(c["Ds"][2] == 192 for c in inv) and any(c["B"] == 3 for c in inv)
    assert {(c["W"], c["H"]) for c in inv} >= {(32, 32), (2048, 96)}
    assert any(c.get("ratios") == (1, 2.5, 5.5) for c in inv)
    assert any("wide_range" in c["edges"] for c in inv)
    assert any(c.get("costreg_fp64") for c in inv)


_ODD = (8, 1, 24, 16, 16)        # Cin, B, D, h, w: D/8 = 3


def _check_odd(acts, layers, blocked):
    x, ws, logits = CFG5._pack(acts, _ODD, blocked)
    cin, B, D, h, w = _ODD
    kernels = ["direct"] + ["tma" if L["stride"] == 1 else "tma2" for L in layers[1:]]
    return CFG5.check_costreg_elements("simulated odd D", x, ws, logits, layers, B, D, h, w,
                                       range(B), blocked=blocked,
                                       kernels=None if blocked else kernels)


@pytest.mark.parametrize("blocked", [True, False])
def test_simulated_odd_depth_workspace_passes(blocked):
    acts, layers = CFG5._small_net(_ODD)
    need = _check_odd(acts, layers, blocked)
    assert need and all(v <= CONV_T.EPS[f] for f, v in need.items())


# (activation, layer index, plane) in the last depth chunk of an odd-D layer
_LAST_PLANES = [("c0", 0, _ODD[2] - 1), ("c6", 6, _ODD[2] // 8 - 1), ("u7", 7, _ODD[2] // 4 - 1),
                ("u9", 8, _ODD[2] // 2 - 1), ("logits", 10, _ODD[2] - 1)]


@pytest.mark.parametrize("blocked", [True, False])
@pytest.mark.parametrize("act,layer,plane", _LAST_PLANES)
def test_check_catches_a_wrong_last_plane(act, layer, plane, blocked):
    """One plane of the last depth chunk holds the previous plane's values."""
    acts, layers = CFG5._small_net(_ODD)
    acts[act][:, plane] = acts[act][:, plane - 1]
    with pytest.raises(AssertionError) as e:
        _check_odd(acts, layers, blocked)
    msg = str(e.value)
    print(msg)
    assert f"layer {layer} ({act})" in msg and f"(b,d,h,w,c)=(0, {plane}," in msg


@pytest.mark.parametrize("act,layer,plane", _LAST_PLANES)
def test_check_catches_an_unwritten_last_plane(act, layer, plane):
    """The last plane was never written: it keeps the workspace's NaN fill."""
    acts, layers = CFG5._small_net(_ODD)
    acts[act][:, plane] = float("nan")
    with pytest.raises(AssertionError) as e:
        _check_odd(acts, layers, True)
    msg = str(e.value)
    print(msg)
    assert f"layer {layer} ({act})" in msg and f"(b,d,h,w,c)=(0, {plane}," in msg


def test_two_groups_pad_to_four_channels_and_keep_the_reference_shape():
    from casmvsnet_pl_b200.models.mvsnet import CostRegNet
    torch.manual_seed(0)
    net = CostRegNet(2, ABN)
    assert tuple(net.conv0.conv.weight.shape) == (8, 2, 3, 3, 3) and net.kernel_channels == 4
    w = net._conv0_weight()
    assert tuple(w.shape) == (8, 4, 3, 3, 3)
    assert torch.equal(w[:, :2], net.conv0.conv.weight) and not w[:, 2:].any()
    x = ops.as_volume_view(torch.randn(2, 8, 4, 6, 2))              # logical (B, 2, D, h, w)
    xp = net._pad_channels(x)
    assert tuple(xp.shape) == (2, 4, 8, 4, 6)
    assert torch.equal(xp[:, :2], x) and not xp[:, 2:].any()
    assert ops.volume_storage(xp).is_contiguous()
    # conv0 of the padded pair is conv0 of the original pair
    y = torch.nn.functional.conv3d(x.double(), net.conv0.conv.weight.double(), padding=1)
    yp = torch.nn.functional.conv3d(xp.double(), w.double(), padding=1)
    assert torch.equal(y, yp)
    for cin in (1, 4, 8, 16, 32):
        assert CostRegNet(cin, ABN).kernel_channels == -(-cin // 4) * 4
