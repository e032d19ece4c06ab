"""Depth regression (K3), its backward and the depth hypotheses (K4) element by element against
float64 (oracle/regress_fp64.py):

  * inside the cascade: the forward with return_index=True at cfg2, cfg3 (G = 8), cfg4 view and
    cfg5 view (D = 64 at level 2), tf32 and fp32, and cfg2 at B = 2 with (B, 1) tensor depth
    parameters; cfg2, cfg4 view and cfg2 at B = 2 (distinct per-item ranges) again with the
    inverse-depth sweep, whose K4 calls (inverse_hypotheses) must equal the float32 restatement
    of oracle/inverse_depth_fp64.py bit for bit, clamped pixels the far-clamp rung.  A fixture records every K3 / K4 call; each is checked against float64 applied
    to its own inputs.  The ladder entry points run where ops.ladder_supported holds (V - 1 <= 2:
    cfg2, cfg3); cfg4 and cfg5 materialise their hypotheses and call regress;
  * K3 directly: synthetic logits at scales 1, 4 and 30 at every stage shape, every hypothesis
    form ((B, D, h, w), (D,), ladders with a float, (B,) or (B, h, w) first), input_is_prob and
    want_prob, and the generic kernel (with its 32-thread small-map branch) in a child process
    with CASMVS_K3_REG=0; all of it in the uniform and in the inverse mode (inverse ladders:
    their depths from INV.ladder_f32, which ladder.materialize() must equal bit for bit, and
    regress_ladder must equal regress on them bit for bit);
  * known answers, exact: one plane far above the rest, uniform logits, logits of magnitude 1e3,
    depth_first == depth_hypotheses[:, 0], and first rungs that straddle the 1e-7 clamp;
  * casmvs_regress_bwd at the 640x512 and 768x576 training crops, uniform and inverse, tensor
    and vector hypotheses;
  * a profiler test that every K3 / K4 / FeatureNet kernel instantiation was launched.

The index is compared with clamp(trunc(fidx64), 0, D-1); within the bound of fidx from an
integer either neighbour is accepted, and the number of such pixels must stay below
AMBIGUOUS_MAX of the pixels.  Peaked logits (scale 30, magnitude 1e3) are exempt from that
limit: a near one-hot softmax puts fidx within rounding of an integer by construction, so most
of their pixels are ambiguous; their index must still be one of the two neighbours.  EPS is the
largest power of two within 4x of the worst eps needed over this file on an H100 (it prints
them), never above EPS_CEIL."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import ABN, _lib, ops, synth
from oracle import inverse_depth_fp64 as INV
from oracle import regress_fp64 as RG

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS_CEIL = 2.0 ** -17
# Worst eps needed over every case of this file, measured on an H100 80GB HBM3 at a 700 W power
# limit; each eps is the largest power of two within 4x of it.
EPS = {
    "k3": 2.0 ** -19,            # regress_kernel / regress_par_kernel reductions: 5.7e-7
    "k3_bwd": 2.0 ** -20,        # regress_bwd_kernel: 2.9e-7
    "k3_inv": 2.0 ** -19,        # the inverse-mode K3 kernels (regress_inv / regress_par_inv): 6.2e-7
    "k3_inv_bwd": 2.0 ** -20,    # regress_inv_bwd_kernel: 3.8e-7
}
# Share of pixels whose index is ambiguous, worst 4.8e-4 over the non-peaked cases on the same
# H100 (D = 8 at 512x640, logits x4); the limit is the power of two above twice that.
AMBIGUOUS_MAX = 2.0 ** -10
WORST = {}

CASCADE = {   # name: W, H, V, G, n_depths, B, depth sampling
    "cfg2": (640, 512, 3, 1, (8, 32, 48), 1, "uniform"),
    "cfg3": (640, 512, 3, 8, (8, 32, 48), 1, "uniform"),
    "cfg4_view": (1152, 864, 5, 1, (8, 32, 48), 1, "uniform"),
    "cfg5_view": (1920, 1056, 7, 1, (8, 32, 64), 1, "uniform"),
    "cfg2_B2": (640, 512, 3, 1, (8, 32, 48), 2, "uniform"),
    "cfg2_inv": (640, 512, 3, 1, (8, 32, 48), 1, "inverse"),
    "cfg4_view_inv": (1152, 864, 5, 1, (8, 32, 48), 1, "inverse"),
    "cfg2_B2_inv": (640, 512, 3, 1, (8, 32, 48), 2, "inverse"),
}
RECORDED = ("regress", "regress_ladder", "depth_first", "depth_hypotheses", "uniform_hypotheses",
            "inverse_hypotheses")


@pytest.fixture
def recorder(monkeypatch):
    calls = []
    orig = {n: getattr(ops, n) for n in RECORDED}

    def wrap(name):
        def f(*a, **k):
            out = orig[name](*a, **k)
            calls.append((name, a, k, out))
            return out
        return f
    for n in RECORDED:
        monkeypatch.setattr(ops, n, wrap(n))
    return calls


def _report(tag, fam, rep):
    WORST[fam] = max(WORST.get(fam, 0.0), rep.eps_needed)
    print(f"[fp64] {tag} [{fam}]: {rep.describe()}")
    assert rep.ok, f"{tag} [{fam}]: {rep.describe()}"


def _check_k3(tag, logits, hyp, depth, conf, index, prob=None, is_prob=False, peaked=False,
              inverse=False):
    fam = "k3_inv" if inverse else "k3"
    reps = RG.check_regress(logits, hyp, depth, conf, index, prob, is_prob, EPS[fam], inverse)
    for k in ("prob", "depth", "conf"):
        if k in reps:
            _report(f"{tag} {k}", fam, reps[k])
    if index is not None:
        wrong, amb, first = reps["index"]
        print(f"[fp64] {tag} index: {wrong} wrong, {amb} ambiguous of {index.numel()} "
              f"({amb / index.numel():.2e})")
        assert wrong == 0, f"{tag}: {wrong} wrong indices, first at (b, y, x) = {first}"
        if not peaked:
            assert amb <= AMBIGUOUS_MAX * index.numel(), f"{tag}: {amb} ambiguous indices"


def _step32(v, B):
    """The float32 step value(s) the kernel uses."""
    if torch.is_tensor(v):
        return v.reshape(-1).float().to(DEV)
    return float(torch.tensor(float(v), dtype=torch.float32))


def _check_k4(tag, out, want, bound, clamped=None, first_only=False):
    if first_only:
        want, bound = want[:, :1], bound[:, :1]
        out = out.unsqueeze(1)
    rep = RG.check(out, want, bound, torch.zeros_like(bound), 0.0, ("b", "d", "y", "x"),
                   scale=want.abs())
    print(f"[fp64] {tag} [k4]: {rep.describe()}")
    assert rep.ok, f"{tag} [k4]: {rep.describe()}"
    if clamped is not None and bool(clamped.any()):
        assert bool((out[:, 0][clamped] == RG.THRESH).all()), f"{tag}: clamped rung != 1e-7f"


def ladder_hyp(lad):
    """The hypotheses of a Ladder for the float64 checks: an inverse ladder's from the float32
    restatement INV.ladder_f32, which materialize() must equal bit for bit; a uniform ladder's
    materialised (the same two roundings as the kernels)."""
    m = lad.materialize()
    if not lad.inverse:
        return m
    want = torch.from_numpy(INV.ladder_f32(lad.first, lad.step, lad.D, lad.B, lad.h, lad.w))
    assert torch.equal(m.cpu(), want), "inverse Ladder.materialize() != INV.ladder_f32"
    return want.to(m.device)


def inverse_steps_f32(st):
    """ops.InverseSteps -> the (u_near, u_far, [s_l]) float32 (B,) arrays of INV.steps_f32."""
    def arr(x):
        return np.broadcast_to(INV._np32(x).reshape(-1), (st.B,)).copy()
    return arr(st.u_near), arr(st.u_far), [arr(s) for s in st.step]


def _check_inverse_k4(tag, a, k, out):
    """inverse_hypotheses bit for bit against rules 3-4 restated in float32 on the call's own
    current_depth; where rule 4's far clamp holds by a clear margin in float64 the first rung
    is exactly the clamp u_far + (D-1) s."""
    st, level, D, h, w = a[:5]
    cur = k.get("current_depth", a[6] if len(a) > 6 else None)
    first_only = k.get("first_only", a[7] if len(a) > 7 else False)
    ref = inverse_steps_f32(st)
    c = None if cur is None else cur.cpu().numpy()
    want = INV.first_rung_f32(ref, level, D, c) if first_only else INV.hypotheses_f32(ref, level, D, h, w, c)
    assert torch.equal(out.cpu(), torch.from_numpy(np.ascontiguousarray(want))), \
        f"{tag} inverse_hypotheses L{level} D={D} first_only={first_only}: differs from INV"
    if cur is None:
        return
    s, uf = ref[2][level].reshape(-1, 1, 1), ref[1].reshape(-1, 1, 1)
    up = torch.nn.functional.interpolate(cur.double().cpu().unsqueeze(1), scale_factor=2,
                                         mode="bilinear", align_corners=True)[:, 0].numpy()
    clamped = 1 / up + D / 2 * s.astype(np.float64) < (uf + (D - 1) * s.astype(np.float64)) * (1 - 1e-5)
    rung = (uf + (np.float32(D - 1) * s).astype(np.float32)).astype(np.float32)
    got = out.cpu().numpy() if first_only else out[:, 0].cpu().numpy()
    rung = np.broadcast_to(rung if first_only else INV._rcp(rung), got.shape)
    assert (got == rung)[clamped].all(), f"{tag}: a clamped pixel's first plane is not the far clamp"
    print(f"[fp64] {tag} inverse_hypotheses L{level} D={D} first_only={first_only}: bit-exact, "
          f"{int(clamped.sum())} clamped pixels")
    return int(clamped.sum())


def check_call(name, a, k, out, tag):
    if name == "regress":
        logits, dv = a[0], a[1]
        is_prob = k.get("input_is_prob", False)
        inverse = k.get("inverse", a[5] if len(a) > 5 else False)
        depth, conf, index, prob = out
        _check_k3(f"{tag} regress D={logits.shape[1]} {tuple(logits.shape[2:])}", logits, dv,
                  depth, conf, index, prob, is_prob, inverse=inverse)
    elif name == "regress_ladder":
        logits, lad = a[0], a[1]
        depth, conf, index = out
        _check_k3(f"{tag} regress_ladder D={logits.shape[1]} {tuple(logits.shape[2:])}", logits,
                  ladder_hyp(lad), depth, conf, index, inverse=lad.inverse)
    elif name == "inverse_hypotheses":
        _check_inverse_k4(tag, a, k, out)
    elif name in ("depth_first", "depth_hypotheses"):
        cur, D, interval = a[:3]
        up = name == "depth_first" or k.get("upsample", a[3] if len(a) > 3 else False)
        want, bound, clamped = RG.hypotheses_ref(cur, D, _step32(interval, cur.shape[0]), up)
        _check_k4(f"{tag} {name} D={D} up={up}", out, want, bound, clamped,
                  first_only=name == "depth_first")
    elif name == "uniform_hypotheses":
        dmin, interval, D, B, h, w = a[:6]
        want, bound = RG.uniform_ref(_step32(dmin, B), _step32(interval, B), B, D, h, w, DEV)
        _check_k4(f"{tag} uniform D={D}", out, want, bound)
    else:
        raise AssertionError(name)


# ------------------------------------------------------------------------------- in the cascade
@pytest.mark.parametrize("precision", ["tf32", "fp32"])
@pytest.mark.parametrize("cfg", list(CASCADE))
def test_cascade_k3_k4_calls_vs_fp64(cfg, precision, recorder):
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    W, H, V, G, Ds, B, sampling = CASCADE[cfg]
    torch.manual_seed(0)
    model = CascadeMVSNet(n_depths=list(Ds), num_groups=G, norm_act=ABN, precision=precision,
                          depth_sampling=sampling)
    synth.randomize_model_(model, 0)
    model = model.eval().to(DEV)
    model.return_index = True
    imgs, pm, dmin, dint = synth.make_inputs(B=B, V=V, W=W, H=H, seed=B)
    if B > 1:         # per-item depth ranges: the ladder's first_b / step_b and first_map
        dmin = torch.tensor([[425.0], [451.5]])
        dint = torch.tensor([[2.65], [3.05]])
    model(imgs.to(DEV), pm.to(DEV), dmin, dint)
    torch.cuda.synchronize()
    names = [n for n, *_ in recorder]
    ladder = ops.ladder_supported(V, 8, G)
    assert ladder == (V - 1 <= 2)
    if sampling == "inverse":
        assert sorted(names) == (["inverse_hypotheses"] * (2 if ladder else 3) +
                                 ["regress" if not ladder else "regress_ladder"] * 3), names
    elif ladder:
        assert sorted(names) == ["depth_first"] * 2 + ["regress_ladder"] * 3, names
    else:
        assert sorted(names) == (["depth_hypotheses"] * 2 + ["regress"] * 3 +
                                 ["uniform_hypotheses"]), names
    for name, a, k, out in list(recorder):
        check_call(name, a, k, out, f"{cfg} {precision}")


# ------------------------------------------------------------------------------- K3 directly
STAGES = [(8, 512, 640), (32, 256, 320), (48, 128, 160), (64, 264, 480), (8, 37, 53)]
FORMS = ["tensor", "vector", "ladder_float", "ladder_batch", "ladder_map"]


def _hyp(form, g, B, D, h, w, inverse=False):
    if inverse:
        return _hyp_inverse(form, g, B, D, h, w)
    step = 2.65 * (1 + D / 16)
    if form == "tensor":
        return torch.rand(B, D, h, w, generator=g, device=DEV) * 500 + 400
    if form == "vector":
        return 425.0 + step * torch.arange(D, device=DEV, dtype=torch.float32)
    if form == "ladder_float":
        return ops.Ladder(425.0, step, D, B, h, w, DEV)
    if form == "ladder_batch":
        fb = torch.tensor([425.0 + 17.3 * b for b in range(B)], device=DEV)
        sb = torch.tensor([step * (1 + 0.13 * b) for b in range(B)], device=DEV)
        return ops.Ladder(fb, sb, D, B, h, w, DEV)
    first = 500 + 60 * torch.rand(B, h, w, generator=g, device=DEV)
    return ops.Ladder(first, step, D, B, h, w, DEV)


def _hyp_inverse(form, g, B, D, h, w):
    """The FORMS in the inverse mode over a wide range (near 0.5 .. far 6, per item 0.5 + 0.04 b
    .. 6 + 0.7 b): ladders in 1/depth, the vector and tensor forms their depths."""
    un = [1 / (0.5 + 0.04 * b) for b in range(B)]
    s = [(un[b] - 1 / (6.0 + 0.7 * b)) / (D - 1) for b in range(B)]
    if form == "tensor":
        return 1 / (un[0] - (un[0] - 1 / 6.0) * torch.rand(B, D, h, w, generator=g, device=DEV))
    if form == "vector":
        return torch.from_numpy(INV.ladder_f32(un[0], s[0], D, 1, 1, 1).reshape(D)).to(DEV)
    if form == "ladder_float":
        return ops.Ladder(un[0], s[0], D, B, h, w, DEV, inverse=True)
    if form == "ladder_batch":
        return ops.Ladder(torch.tensor(un, device=DEV), torch.tensor(s, device=DEV), D, B, h, w,
                          DEV, inverse=True)
    # a per-pixel first rung between the far clamp and u_near
    sb = torch.tensor(s, device=DEV).view(B, 1, 1)
    lo = 1 / torch.tensor([6.0 + 0.7 * b for b in range(B)], device=DEV).view(B, 1, 1) + (D - 1) * sb
    hi = torch.tensor(un, device=DEV).view(B, 1, 1)
    first = lo + (hi - lo) * torch.rand(B, h, w, generator=g, device=DEV)
    return ops.Ladder(first, sb.reshape(B), D, B, h, w, DEV, inverse=True)


def _direct_cases():
    for inverse in (False, True):
        i = 0
        for D, h, w in STAGES:
            for scale in (1.0, 4.0, 30.0):
                yield D, h, w, scale, FORMS[i % len(FORMS)], inverse
                i += 1


def _direct_id(c):
    return "D%d_%dx%d_x%g_%s" % c[:5] + ("_inv" if c[5] else "")


def _run_direct(D, h, w, scale, form, inverse=False, B=2):
    g = torch.Generator(device=DEV).manual_seed(D * 1000 + h + int(scale) + (7 if inverse else 0))
    logits = torch.randn(B, D, h, w, generator=g, device=DEV) * scale
    hyp = _hyp(form, g, B, D, h, w, inverse)
    out = {}
    lad = None
    if isinstance(hyp, ops.Ladder):
        out["ladder"] = ops.regress_ladder(logits, hyp, want_index=True) + (None,)
        lad, hyp = hyp, ladder_hyp(hyp)
    out["logits"] = ops.regress(logits, hyp, want_index=True, want_prob=True, inverse=inverse)
    prob = torch.softmax(logits.double(), 1).float()
    out["prob_in"] = ops.regress(prob, hyp, input_is_prob=True, want_index=True, inverse=inverse)
    if lad is not None and inverse:
        # the ladder generates the same planes as the tensor it materialises: the same bits
        for a, b in zip(out["ladder"][:3], out["logits"][:3]):
            assert torch.equal(a, b), f"D={D} {h}x{w} {form}: regress_ladder != regress"
    return logits, hyp, prob, out


def _check_direct(tag, logits, hyp, prob, out, peaked, inverse=False):
    for k, (depth, conf, index, p) in out.items():
        if k == "prob_in":
            _check_k3(f"{tag} {k}", prob, hyp, depth, conf, index, None, True, peaked, inverse)
        else:
            _check_k3(f"{tag} {k}", logits, hyp, depth, conf, index, p, False, peaked, inverse)


@pytest.mark.parametrize("case", list(_direct_cases()), ids=_direct_id)
def test_regress_direct_vs_fp64(case):
    D, h, w, scale, form, inverse = case
    logits, hyp, prob, out = _run_direct(D, h, w, scale, form, inverse)
    _check_direct(f"D={D} {h}x{w} x{scale} {form}" + (" inverse" if inverse else ""), logits, hyp,
                  prob, out, scale > 4, inverse)


GENERIC = [(8, 512, 640, 4.0, "tensor", False), (48, 128, 160, 30.0, "ladder_map", False),
           (32, 37, 53, 1.0, "vector", False), (64, 264, 480, 4.0, "ladder_batch", False),
           (8, 512, 640, 4.0, "ladder_map", True), (48, 128, 160, 30.0, "tensor", True),
           (32, 37, 53, 1.0, "ladder_float", True), (64, 264, 480, 4.0, "vector", True)]


def _generic_outputs():
    res = []
    for c in GENERIC:
        _, _, _, out = _run_direct(*c)
        res.append({k: [t.cpu() if t is not None else None for t in v] for k, v in out.items()})
    return res


def test_regress_generic_kernel_vs_fp64(tmp_path):
    """CASMVS_K3_REG=0: every D runs the one-thread-per-pixel generic kernel, with 32-thread
    blocks where the map is small (37x53, 128x160)."""
    code = ("import sys, torch\n"
            "sys.path.insert(0, %r)\n"
            "sys.path.insert(0, %r)\n"
            "import test_gpu_regress_fp64 as T\n"
            "with torch.no_grad():\n"
            "    torch.save(T._generic_outputs(), sys.argv[1])\n"
            % (ROOT, os.path.join(ROOT, "tests")))
    path = str(tmp_path / "k3_generic.pt")
    subprocess.run([sys.executable, "-c", code, path], check=True,
                   env=dict(os.environ, CASMVS_K3_REG="0"), timeout=600)
    got = torch.load(path)
    for c, res in zip(GENERIC, got):
        D, h, w, scale, form, inverse = c
        g = torch.Generator(device=DEV).manual_seed(D * 1000 + h + int(scale) + (7 if inverse else 0))
        logits = torch.randn(2, D, h, w, generator=g, device=DEV) * scale
        hyp = _hyp(form, g, 2, D, h, w, inverse)
        hyp = ladder_hyp(hyp) if isinstance(hyp, ops.Ladder) else hyp
        prob = torch.softmax(logits.double(), 1).float()
        out = {k: tuple(t.to(DEV) if t is not None else None for t in v) for k, v in res.items()}
        _check_direct(f"generic D={D} {h}x{w} x{scale} {form}" + (" inverse" if inverse else ""),
                      logits, hyp, prob, out, scale > 4, inverse)


# ------------------------------------------------------------------------------- known answers
@pytest.mark.parametrize("D,h,w", [(8, 512, 640), (32, 256, 320), (48, 128, 160), (64, 33, 47)])
def test_regress_known_answers(D, h, w):
    g = torch.Generator(device=DEV).manual_seed(D)
    B = 2
    hyp = torch.rand(B, D, h, w, generator=g, device=DEV) * 500 + 400
    for k in (0, 1, D - 2, D - 1):
        logits = torch.randn(B, D, h, w, generator=g, device=DEV)
        logits[:, k] += 40.0
        depth, conf, index, _ = ops.regress(logits, hyp, want_index=True)
        assert torch.equal(index, torch.full_like(index, k)), f"D={D} peak {k}: index"
        assert torch.equal(depth, hyp[:, k]), f"D={D} peak {k}: depth"
        assert torch.equal(conf, torch.ones_like(conf)), f"D={D} peak {k}: confidence"
    flat = torch.full((B, D, h, w), 0.5, device=DEV)
    depth, conf, index, prob = ops.regress(flat, hyp, want_index=True, want_prob=True)
    _check_k3(f"uniform D={D}", flat, hyp, depth, conf, index, prob)
    assert torch.equal(index, torch.full_like(index, (D - 1) // 2))
    big = torch.randn(B, D, h, w, generator=g, device=DEV) * 1e3
    depth, conf, index, prob = ops.regress(big, hyp, want_index=True, want_prob=True)
    assert all(bool(torch.isfinite(t).all()) for t in (depth, conf, prob))
    _check_k3(f"magnitude 1e3 D={D}", big, hyp, depth, conf, index, prob, peaked=True)


def test_hypotheses_known_answers():
    g = torch.Generator(device=DEV).manual_seed(3)
    for (D, hi, wi), step in (((32, 64, 80), 5.3), ((48, 32, 40), 10.6), ((8, 256, 320), 2.65),
                              ((64, 132, 240), 10.6)):
        cur = 425 + 500 * torch.rand(2, hi, wi, generator=g, device=DEV)
        full = ops.depth_hypotheses(cur, D, step, upsample=True)
        first = ops.depth_first(cur, D, step)
        assert torch.equal(first, full[:, 0]), f"D={D}: depth_first != depth_hypotheses[:, 0]"
        st = torch.tensor([[step], [step * 1.1]], device=DEV)
        assert torch.equal(ops.depth_first(cur, D, st), ops.depth_hypotheses(cur, D, st, True)[:, 0])
    # first rungs straddling the clamp: cur - D/2 step around 1e-7 (and far below, far above)
    D, step = 32, 2.65
    half = float(torch.tensor(D / 2 * step, dtype=torch.float32))
    base = torch.tensor([half - 1.0, half - 1e-5, half, half + 1e-7, half + 2e-7, half + 1e-4,
                         half + 1.0, 0.0], device=DEV)
    cur = base[torch.randint(0, 8, (2, 24, 40), generator=g, device=DEV)]
    for name, fn in (("depth_first", lambda: ops.depth_first(cur, D, step)),
                     ("depth_hypotheses", lambda: ops.depth_hypotheses(cur, D, step, True))):
        out = fn()
        want, bound, clamped = RG.hypotheses_ref(cur, D, _step32(step, 2), True)
        assert bool(clamped.any()) and bool((~clamped).any())
        _check_k4(f"clamp {name}", out, want, bound, clamped, first_only=name == "depth_first")
    plain = ops.depth_hypotheses(cur.unsqueeze(1), D, step, upsample=False)
    want, bound, clamped = RG.hypotheses_ref(cur.unsqueeze(1), D, _step32(step, 2), False)
    _check_k4("clamp no upsample", plain, want, bound, clamped)
    uni = ops.uniform_hypotheses(torch.tensor([[425.0], [1e-3]]), torch.tensor([[10.6], [0.1]]),
                                 48, 2, 7, 9, DEV)
    want, bound = RG.uniform_ref(torch.tensor([425.0, 1e-3]), torch.tensor([10.6, 0.1]), 2, 48, 7,
                                 9, DEV)
    _check_k4("uniform tensor", uni, want, bound)


def test_inverse_hypotheses_far_clamp():
    """A current depth map with pixels beyond the far plane: K4's inverse planes bit for bit,
    the far clamp held at those pixels, per-item (B,) and float steps."""
    g = torch.Generator(device=DEV).manual_seed(8)
    for dmin, dint in ((425.0, 2.65), (torch.tensor([[425.0], [451.5]]), torch.tensor([[2.65], [3.05]]))):
        st = ops.inverse_steps(dmin, dint, (8, 32, 48), (1, 2, 4), 2, DEV)
        for level, D, h, w in ((1, 32, 256, 320), (0, 8, 512, 640)):
            cur = 425.0 + 500.0 * torch.rand(2, h // 2, w // 2, generator=g, device=DEV)
            cur[:, : h // 8] = 5000.0                       # far beyond the far plane (about 925)
            for first_only in (True, False):
                a = (st, level, D, h, w, DEV)
                k = dict(current_depth=cur, first_only=first_only)
                n = _check_inverse_k4(f"far clamp {'tensor' if torch.is_tensor(dmin) else 'float'}",
                                      a, k, ops.inverse_hypotheses(*a, **k))
                assert n >= 2 * (h // 4 - 1) * w, n


# ------------------------------------------------------------------------------- backward
BWD = {   # name: B, D, h, w, hypotheses
    "dtu_L0": (2, 8, 512, 640, "tensor"), "dtu_L1": (2, 32, 256, 320, "tensor"),
    "dtu_L2": (2, 48, 128, 160, "tensor"), "blended_L0": (2, 8, 576, 768, "tensor"),
    "blended_L1": (2, 32, 288, 384, "tensor"), "blended_L2": (2, 48, 144, 192, "tensor"),
    "dtu_L2_vector": (2, 48, 128, 160, "vector"),
}
# the inverse regression's backward at both training crops (hypotheses over a wide range)
for _name in list(BWD):
    BWD[_name + "_inv"] = BWD[_name]
BWD["blended_L2_vector_inv"] = (2, 48, 144, 192, "vector")


@pytest.mark.parametrize("name", list(BWD))
def test_regress_bwd_vs_fp64(name):
    B, D, h, w, form = BWD[name]
    inverse = name.endswith("_inv")
    g = torch.Generator(device=DEV).manual_seed(D + h)
    logits = torch.randn(B, D, h, w, generator=g, device=DEV) * 4
    hyp = _hyp(form, g, B, D, h, w, inverse)
    gd = torch.randn(B, h, w, generator=g, device=DEV)
    gl = torch.full_like(logits, float("nan"))
    flags = int(hyp.dim() == 1) | (ops.INVERSE_DEPTH if inverse else 0)
    _lib.check(_lib.load().casmvs_regress_bwd(ops._ptr(logits), ops._ptr(hyp), flags,
                                              ops._ptr(gd), ops._ptr(gl), B, D, h, w,
                                              ops._stream()), "regress_bwd")
    g64, b0, A = RG.regress_bwd_ref(logits, hyp, gd, inverse)
    fam = "k3_inv_bwd" if inverse else "k3_bwd"
    _report(f"bwd {name} {(B, D, h, w)}", fam, RG.check(gl, g64, b0, A, EPS[fam], ("b", "d", "y", "x")))


# ------------------------------------------------------------------------------- coverage
KERNELS = [r"regress_kernel<true, 8>", r"regress_kernel<false, 8>", r"regress_par_kernel<true>",
           r"regress_par_kernel<false>", r"fpn_level_kernel<8>", r"fpn_level_kernel<16>",
           r"fpn_merge_kernel", r"conv2d_rgb8_kernel", r"conv2d_rgb8_x4_kernel",
           r"conv2d_5x5s2_fp32_kernel<8, 16>", r"conv2d_5x5s2_fp32_kernel<16, 32>",
           r"hypotheses_kernel", r"uniform_hypotheses_kernel", r"regress_bwd_kernel",
           r"regress_kernel<true, 0>", r"regress_kernel<false, 0>",
           r"regress_inv_kernel<true, 8>", r"regress_inv_kernel<false, 8>",
           r"regress_par_inv_kernel<true>", r"regress_par_inv_kernel<false>",
           r"regress_inv_kernel<true, 0>", r"regress_inv_kernel<false, 0>",
           r"inverse_hypotheses_kernel", r"regress_inv_bwd_kernel"]


def _launched(k, names):
    """k names a kernel, not the tail of a longer one (hypotheses_kernel in
    inverse_hypotheses_kernel)."""
    return any(re.search(r"(?<![A-Za-z0-9_])" + re.escape(k), n) for n in names)


def test_kernel_coverage():
    from torch.profiler import ProfilerActivity, profile
    g = torch.Generator(device=DEV).manual_seed(0)

    def rn(*s):
        return torch.randn(*s, generator=g, device=DEV)

    def cl(t):
        return t.contiguous(memory_format=torch.channels_last)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        # D = 256: the plane-parallel kernel's shared memory exceeds 96 KB, the generic one runs
        for D in (8, 32, 256):
            lg, dv = rn(1, D, 16, 24), rn(1, D, 16, 24) + 500
            for inverse in (False, True):
                ops.regress(lg, dv, inverse=inverse)
                ops.regress(torch.softmax(lg, 1), dv, input_is_prob=True, inverse=inverse)
        for cout in (8, 16):
            ops.fpn_level(cl(rn(1, 32, 8, 10)), cl(rn(1, 8, 16, 20)), rn(32, 8, 1, 1), rn(32),
                          rn(cout, 32, 3, 3), rn(cout), want_feat=False)
        ops.fpn_merge(None, cl(rn(1, 8, 16, 20)), rn(32, 8, 1, 1), rn(32))
        for W_ in (20, 21):
            ops.conv2d_rgb8(rn(1, 3, 8, W_), rn(8, 3, 3, 3), rn(8), 0.01)
        for cin, cout in ((8, 16), (16, 32)):
            ops.conv2d_5x5s2_fp32(cl(rn(1, cin, 9, 11)), rn(cout, cin, 5, 5).contiguous(), rn(cout),
                                  0.01)
        ops.depth_hypotheses(rn(1, 4, 5) + 500, 8, 2.65, upsample=True)
        ops.uniform_hypotheses(425.0, 2.65, 8, 1, 4, 5, DEV)
        ops.inverse_hypotheses(ops.inverse_steps(425.0, 2.65, (8, 32, 48), (1, 2, 4), 1), 1, 32, 8,
                               10, DEV, current_depth=rn(1, 4, 5).abs() + 500)
        lg, dv, gd = rn(1, 8, 4, 5), rn(1, 8, 4, 5) + 500, rn(1, 4, 5)
        gl = torch.empty_like(lg)
        for flags in (0, ops.INVERSE_DEPTH):
            _lib.check(_lib.load().casmvs_regress_bwd(ops._ptr(lg), ops._ptr(dv), flags, ops._ptr(gd),
                                                      ops._ptr(gl), 1, 8, 4, 5, ops._stream()),
                       "regress_bwd")
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    missing = [k for k in KERNELS if not _launched(k, names)]
    for k in KERNELS:
        print(f"[coverage] {k}: {'launched' if k not in missing else 'MISSING'}")
    assert not missing, (missing, sorted(n for n in names if re.search("casmvs", n)))


def test_zz_print_worst():
    for fam, v in sorted(WORST.items()):
        print(f"[fp64] worst eps needed [{fam}]: {v:.3e} (eps {EPS[fam]:.3e})")
    assert all(e <= EPS_CEIL for e in EPS.values())
