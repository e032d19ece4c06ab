"""CostRegNet at the 1920x1056 / V=7 cascade stages (D = 64 / 32 / 8) and at the batch sizes
the benchmark runs, element by element against float64, and the whole cascade's batch
independence at full size:

  * casmvs_costreg_fwd (TF32 | BLOCKED input, caller-owned NaN-filled workspace) at the three
    stage shapes for B = 1 and B = 4, and at stage 1 for B = 5, whose 5.2 GB blocked input is
    the first shape past 2^32 bytes (a 32-bit byte offset or TMA coordinate would wrap there).
    Each of the 11 layers of every batch element is checked against float64 applied to the
    kernel's own input activation and skip of that element, at the committed per-kernel eps of
    test_gpu_conv_fp64.EPS.  The layers do not mix batch elements, so the float64 reference of
    one element alone is exact and keeps float64 memory at the B = 1 size;
  * the fused conv11 + prob tail gives the logits of the two-layer path, bit for bit, at the
    same batched shapes;
  * the tf32 cascade (eager) at 1920x1056, V=7, D=(8,32,64) and at 640x512, V=3: a forward of
    four distinct views, with per-view (B,1) depth parameters, equals four single-view forwards
    bit for bit, and at 640x512 the CUDA-graph replay equals the eager forward.  Every library
    call of the forwards is recorded, so a difference is reported at the first library call
    whose outputs differ (or at the torch op between library calls that introduced it).

The CPU part checks the per-element reference against the whole-batch one, and that the
per-element check of a workspace catches a batch-offset defect at the element that has it."""
import pytest
import torch

import test_gpu_conv_fp64 as CONV_T
from casmvsnet_pl_b200 import ABN, _lib, ops, synth
from oracle import conv3d_fp64 as R

DEV = "cuda:0"

STAGES = {   # cfg5 (1920x1056, V=7) stages: Cin, D, h, w
    "stage1": (32, 64, 264, 480),
    "stage2": (16, 32, 528, 960),
    "stage3": (8, 8, 1056, 1920),
}
DRIVER_SHAPES = {f"1920x1056_{s}_B{B}": (cin, B, D, h, w)
                 for B in (1, 4) for s, (cin, D, h, w) in STAGES.items()}
# a single-GPU sharded_depth_inference call runs every view of its batch on one GPU
DRIVER_SHAPES["1920x1056_stage1_B5"] = (32, 5, 64, 264, 480)
TAIL_SHAPES = {k: v for k, v in DRIVER_SHAPES.items() if v[1] > 1}


# ------------------------------------------------------------------------------- float64 reference
def layer_fp64(x, w64, kind, stride, scale, shift, slope, skip):
    """One layer in float64: (y64, A, |shift| + |skip|) for channels-last x (B, D, h, w, Cin)."""
    acc = R.conv3d_ref(x, w64, kind, stride)
    y64 = R.epilogue(acc, scale, shift, slope, skip)
    del acc
    A = R.magnitude(x, w64, kind, stride, scale)
    return y64, A, R.epilogue_magnitude(y64, shift, skip)


def costreg_layers(params, cin):
    """The 11 layers of a casmvs_costreg_fwd parameter blob: kind, stride, channels, the weights
    the operand images hold (RNA-rounded to TF32) and the folded scale / shift."""
    out = []
    for i in range(11):
        L = ops.costreg_layer_info(cin, i)
        n = 27 * L["cin"] * L["cout"]
        w = params[L["w_off"]:L["w_off"] + n].view(27, L["cin"], L["cout"])
        out.append(dict(L, w=R.tf32_rna(w.contiguous()),
                        scale=params[L["scale_off"]:L["scale_off"] + L["cout"]],
                        shift=params[L["shift_off"]:L["shift_off"] + L["cout"]]))
    return out


def check_costreg_elements(tag, x, ws, logits, layers, B, D, h, w, elements, blocked=True,
                           kernels=None, tf32=True):
    """Check every layer of batch elements `elements` of a casmvs_costreg_fwd call: x the blocked
    input (B, Cin/4, D, h, w, 4), ws the workspace it left (blocked activations at the offsets
    the driver slices it at), logits (B, D, h, w).  The float64 reference of element b is
    computed from element b's activations alone.

    blocked=False: x and the activations are channels-last (B, D, h, w, C), as the driver leaves
    them where some layer has no tensor-core kernel or in the fp32 precision.  kernels: the eps
    family of each layer's kernel (default: the wgmma kernel of its stride).  tf32=False: the
    fp32 precision, whose stores and inputs are not TF32-rounded.  -> {family: worst eps needed}."""
    n = B * D * h * w
    acts, off = {"x": x}, 0
    for name, c, s in CONV_T._ACTS:
        size = c * n // s ** 3
        dims = (D // s, h // s, w // s)
        buf = ws[off:off + size]
        acts[name] = buf.view(B, c // 4, *dims, 4) if blocked else buf.view(B, *dims, c)
        off += size
    assert (off + 64) == ws.numel()         # every float but the 64-float alignment slack

    def element(name, b):
        if name == "logits":
            return logits[b:b + 1].unsqueeze(-1)
        return R.from_blocked(acts[name][b:b + 1]) if blocked else acts[name][b:b + 1]

    worst = {}
    for b in elements:
        for i, L in enumerate(layers):
            xin = element(CONV_T._IN[i], b)
            if tf32:
                assert CONV_T._is_tf32(xin), f"{tag} b={b}: input of layer {i} is not TF32-exact"
            skip = element(CONV_T._SKIP[i], b) if i in CONV_T._SKIP else None
            slope = 1.0 if i == 10 else CONV_T.SLOPE
            y64, A, extra = layer_fp64(xin, L["w"], L["kind"], L["stride"], L["scale"],
                                       L["shift"], slope, skip)
            kernel = kernels[i] if kernels else "tma" if L["stride"] == 1 else "tma2"
            need = CONV_T._check(f"{tag} b={b} layer {i} ({CONV_T._OUT[i]})", kernel,
                                 element(CONV_T._OUT[i], b), y64, A,
                                 R.R_TF32 if tf32 and L["cout"] > 1 else 0.0, extra)
            worst[kernel] = max(worst.get(kernel, 0.0), need)
            del xin, skip, y64, A, extra
    print(f"[fp64] {tag}: checked batch elements {list(elements)} of B={B}")
    return worst


def _blocked_input(seed, cin, B, D, h, w):
    """A TF32-exact blocked cost volume (B, Cin/4, D, h, w, 4), filled one element at a time."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.empty(B, cin // 4, D, h, w, 4, device=DEV)
    for b in range(B):
        x[b] = R.tf32_rna(torch.randn(cin // 4, D, h, w, 4, generator=g, device=DEV))
    return x


# ------------------------------------------------------------------------------- GPU: CostRegNet
@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(DRIVER_SHAPES))
def test_costreg_driver_layers_vs_fp64_per_element(shape):
    cin, B, D, h, w = DRIVER_SHAPES[shape]
    torch.cuda.reset_peak_memory_stats()
    lib = _lib.load()
    x = _blocked_input(cin * 1000 + D + B, cin, B, D, h, w)
    params = CONV_T._net_params(cin)
    ws_bytes = lib.casmvs_costreg_workspace_bytes(B, cin, D, h, w)
    ws = torch.full((ws_bytes // 4,), float("nan"), device=DEV)
    logits = torch.empty(B, D, h, w, device=DEV)
    f0 = _lib.fallback_count()
    _lib.check(lib.casmvs_costreg_fwd(ops._ptr(x), ops._ptr(params), ops._ptr(logits), B, cin, D,
                                      h, w, ops.TF32 | ops.BLOCKED, ops._ptr(ws), ws_bytes,
                                      ops._stream()), "costreg")
    torch.cuda.synchronize()
    assert _lib.fallback_count() == f0
    check_costreg_elements(f"costreg tf32 {shape}", x, ws, logits, costreg_layers(params, cin),
                           B, D, h, w, range(B))
    print(f"[fp64] {shape}: peak allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(TAIL_SHAPES))
def test_fused_tail_logits_are_bit_identical_batched(shape):
    cin, B, D, h, w = TAIL_SHAPES[shape]
    x = _blocked_input(cin * 1000 + D + B + 1, cin, B, D, h, w)
    params = CONV_T._net_params(cin)
    f0 = _lib.fallback_count()
    fused = ops.costreg(x, params, cin, ops.TF32, blocked=True, fused_tail=True)
    unfused = ops.costreg(x, params, cin, ops.TF32, blocked=True, fused_tail=False)
    torch.cuda.synchronize()
    assert _lib.fallback_count() == f0
    assert torch.isfinite(unfused).all()
    for b in range(B):
        assert unfused[b].std() > 0
        diff = fused[b] != unfused[b]
        assert not diff.any(), (
            f"{shape}: batch element {b}: {int(diff.sum())} of {diff.numel()} logits differ, "
            f"first at (d,h,w)={tuple(int(i) for i in diff.nonzero()[0])}")


# ------------------------------------------------------------------------------- GPU: cascade
CASCADES = {
    "cfg5": dict(W=1920, H=1056, V=7, n_depths=(8, 32, 64)),
    "cfg2": dict(W=640, H=512, V=3, n_depths=(8, 32, 48)),
}
RECORDED = ("conv2d_rgb8", "conv2d_planar", "conv2d_5x5s2", "conv2d_5x5s2_fp32", "fpn_merge",
            "fpn_level", "uniform_hypotheses", "depth_hypotheses", "depth_first", "warp_cost",
            "warp_cost_ladder", "costreg", "regress", "regress_ladder", "inverse_hypotheses")
_CHUNK = 1 << 26


def _digest(t):
    """Checksum of a tensor's bits: the raw bit patterns times odd position weights, summed
    modulo 2^64.  Any single changed element changes it (|bits delta| * weight < 2^64)."""
    v = t.detach().contiguous().view(-1)
    if v.dtype == torch.float32:
        v = v.view(torch.int32)
    total = 0
    for s in range(0, v.numel(), _CHUNK):
        c = v[s:s + _CHUNK].long()
        wgt = torch.arange(2 * s + 1, 2 * (s + c.numel()), 2, device=c.device)
        total = (total + int((c * wgt).sum())) % (1 << 64)
    return total


def _leaves(obj):
    """The values of a call's arguments or result that carry data: tensors and floats (a Ladder
    by its first rung and step, InverseSteps by u_near, u_far and the steps).  Ints and flags are shapes and modes, equal by construction."""
    if torch.is_tensor(obj) or isinstance(obj, float):
        return [obj]
    if isinstance(obj, ops.Ladder):
        return _leaves(obj.first) + _leaves(obj.step)
    if isinstance(obj, ops.InverseSteps):
        return _leaves(obj.u_near) + _leaves(obj.u_far) + _leaves(list(obj.step))
    if isinstance(obj, (tuple, list)):
        return [x for o in obj for x in _leaves(o)]
    if isinstance(obj, dict):
        return [x for k in sorted(obj) for x in _leaves(obj[k])]
    return []


class _CallDigests:
    """Wraps the library calls of the inference path.  While recording, each call appends
    (name, inputs, outputs), every leaf as ("t", shape, digest) or ("f", value).  Given the
    records of the single-view forwards, a batched forward's leaves are digested per view: the
    rows of view i of a tensor whose first dimension is B times the single-view one, the whole
    tensor where the shapes agree (weights)."""

    def __init__(self, monkeypatch):
        self.calls, self.single = None, None
        for name in RECORDED:
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name)))

    def _wrap(self, name, fn):
        def f(*a, **k):
            out = fn(*a, **k)
            if self.calls is not None:
                self.calls.append(self._entry(name, _leaves((a, k)), _leaves(out)))
            return out
        return f

    def _entry(self, name, ins, outs):
        if self.single is None:
            return name, [self._desc(x) for x in ins], [self._desc(x) for x in outs]
        k, n = len(self.calls), len(self.single)
        ref = self.single[0]
        if k >= len(ref) or ref[k][0] != name or len(ref[k][1]) != len(ins) or \
                len(ref[k][2]) != len(outs):
            return name, None, None
        return (name, [[self._desc(x, r, i, n) for x, r in zip(ins, ref[k][1])] for i in range(n)],
                [[self._desc(x, r, i, n) for x, r in zip(outs, ref[k][2])] for i in range(n)])

    @staticmethod
    def _desc(x, ref=None, i=0, n=1):
        if not torch.is_tensor(x):
            return ("f", x)
        shape = tuple(x.shape)
        if ref is not None and ref[0] == "t" and shape != ref[1]:
            if shape[0] != n * ref[1][0] or shape[1:] != ref[1][1:]:
                return ("t", shape, None)
            m = ref[1][0]
            x, shape = x[i * m:(i + 1) * m], ref[1]
        return ("t", shape, _digest(x))

    def record(self, single=None):
        self.calls, self.single = [], single

    def stop(self):
        calls, self.calls, self.single = self.calls, None, None
        return calls


def _first_difference(single, batched, i):
    """Where the batched forward's view i first departs from its single-view forward."""
    torch_op = None
    for k, (s, b) in enumerate(zip(single, batched)):
        if b[1] is None:
            return f"library call {k}: the single-view forward ran {s[0]}, the batched one {b[0]}"
        if b[1][i] != s[1]:
            # the earlier library calls agree: an op between them and this call differs; keep
            # comparing the library calls whose inputs agree
            torch_op = torch_op or (f"the inputs of library call {k} ({s[0]}) differ while every "
                                    f"earlier library call's outputs agree: the first difference "
                                    f"is in a torch op, not in this library")
            continue
        if b[2][i] != s[2]:
            return "; ".join(x for x in (torch_op, f"library call {k} ({s[0]}) gives different "
                                         f"outputs from the same inputs") if x)
    if len(single) != len(batched):
        return (torch_op or "") + f" the forwards made {len(single)} and {len(batched)} library calls"
    return torch_op or "every recorded library call agrees"


def _cascade(c):
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(0)
    m = CascadeMVSNet(n_depths=list(c["n_depths"]), norm_act=ABN, precision="tf32")
    synth.randomize_model_(m, 0)
    return m.eval().to(DEV)


def _view(c, i):
    """View i: its own images, its baseline scaled by 1 + 0.05 i (the translation column of
    every projection matrix) and its own depth range, as (1,1) tensors."""
    imgs, pm, dmin, dint = synth.make_inputs(B=1, V=c["V"], W=c["W"], H=c["H"], seed=i)
    pm = pm.clone()
    pm[..., 3] *= 1.0 + 0.05 * i
    return (imgs.to(DEV), pm.to(DEV), torch.tensor([[dmin + 2.5 * i]], device=DEV),
            torch.tensor([[dint * (1.0 + 0.05 * i)]], device=DEV))


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", list(CASCADES))
def test_cascade_batch_of_four_equals_four_single_views(cfg, monkeypatch):
    c, B = CASCADES[cfg], 4
    torch.cuda.reset_peak_memory_stats()
    model = _cascade(c)
    views = [_view(c, i) for i in range(B)]
    rec = _CallDigests(monkeypatch)
    f0 = _lib.fallback_count()
    singles, records = [], []
    for v in views:
        rec.record()
        singles.append(model(*v))
        records.append(rec.stop())
    inputs = [torch.cat([v[j] for v in views]) for j in range(4)]
    rec.record(records)
    batched = model(*inputs)
    calls = rec.stop()
    torch.cuda.synchronize()
    assert _lib.fallback_count() == f0
    assert not torch.equal(singles[0]["depth_0"], singles[-1]["depth_0"])   # distinct views
    print(f"{cfg}: {len(calls)} library calls per forward")
    for i in range(B):
        for l in (0, 1, 2):
            for key in (f"depth_{l}", f"confidence_{l}"):
                got, want = batched[key][i], singles[i][key][0]
                if not torch.equal(got, want):
                    diff = got != want
                    pytest.fail(f"{cfg} B={B}: view {i} {key} differs from the single-view forward "
                                f"at {int(diff.sum())} of {diff.numel()} pixels, first at (h,w)="
                                f"{tuple(int(j) for j in diff.nonzero()[0])}; "
                                f"{_first_difference(records[i], calls, i)}")
        assert _first_difference(records[i], calls, i) == "every recorded library call agrees"
    if cfg == "cfg2":
        from casmvsnet_pl_b200.graph import GraphedCascade
        g = GraphedCascade(model, *inputs, warmup=1)
        out = g()
        torch.cuda.synchronize()
        for key in batched:
            assert torch.equal(out[key], batched[key]), f"graph replay != eager: {key}"
    print(f"{cfg}: peak allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


# ------------------------------------------------------------------------------- CPU
def test_per_element_reference_equals_whole_batch():
    """Every layer kind at ragged shapes, B = 3, with and without skip and at Cout = 1: the
    float64 reference of each batch element alone is the whole-batch reference's slice."""
    g = torch.Generator().manual_seed(3)
    B = 3
    for (kind, stride), dims in CONV_T.RAGGED.items():
        for cin, cout, with_skip in ((8, 16, True), (16, 1, False)):
            x = torch.randn(B, *dims, cin, generator=g)
            w64 = torch.randn(27, cin, cout, generator=g, dtype=torch.float64) * (27 * cin) ** -0.5
            scale = torch.rand(cout, generator=g) + 0.5
            shift = torch.randn(cout, generator=g) * 0.1
            out = R.out_dims(kind, stride, *dims)
            skip = torch.randn(B, *out, cout, generator=g) if with_skip else None
            slope = CONV_T.SLOPE if cout > 1 else 1.0
            whole = layer_fp64(x, w64, kind, stride, scale, shift, slope, skip)
            parts = [layer_fp64(x[b:b + 1], w64, kind, stride, scale, shift, slope,
                                None if skip is None else skip[b:b + 1]) for b in range(B)]
            for j, name in enumerate(("y64", "A", "extra")):
                if whole[j].dim() == 5:
                    got = torch.cat([p[j] for p in parts])
                else:                                   # |shift| only: broadcast per channel
                    assert all(torch.equal(p[j], whole[j]) for p in parts)
                    continue
                assert got.shape == whole[j].shape
                assert torch.equal(got, whole[j]), (kind, stride, cin, cout, name)


_SMALL = (8, 3, 8, 16, 24)     # Cin, B, D, h, w


def _small_net(shape=_SMALL):
    """A CostRegNet driver call simulated in float64 on the CPU at `shape` (Cin, B, D, h, w):
    random layers of the driver's shapes; each activation is its float64 layer, TF32-rounded like
    the kernels' stores (the logits unrounded), laid out as casmvs_costreg_fwd leaves its
    workspace.  -> x, acts, layers, with acts channels-last by name."""
    cin, B, D, h, w = shape
    g = torch.Generator().manual_seed(5)
    layers = []
    for i in range(11):
        L = ops.costreg_layer_info(cin, i)
        wt = torch.randn(27, L["cin"], L["cout"], generator=g) * (27 * L["cin"]) ** -0.5
        scale = torch.ones(L["cout"]) if i == 10 else torch.rand(L["cout"], generator=g) + 0.5
        layers.append(dict(L, w=R.tf32_rna(wt), scale=scale,
                           shift=torch.randn(L["cout"], generator=g) * 0.1))
    acts = {"x": R.tf32_rna(torch.randn(B, D, h, w, cin, generator=g))}
    for i, L in enumerate(layers):
        skip = acts[CONV_T._SKIP[i]] if i in CONV_T._SKIP else None
        y64, _, _ = layer_fp64(acts[CONV_T._IN[i]], L["w"], L["kind"], L["stride"], L["scale"],
                               L["shift"], 1.0 if i == 10 else CONV_T.SLOPE, skip)
        acts[CONV_T._OUT[i]] = R.tf32_rna(y64.float()) if L["cout"] > 1 else y64.float()
    return acts, layers


def _pack(acts, shape=_SMALL, blocked=True):
    """-> x, workspace, logits (B, D, h, w) in casmvs_costreg_fwd's layout: blocked, or with
    blocked=False channels-last."""
    cin, B, D, h, w = shape
    lay = R.to_blocked if blocked else (lambda t: t.contiguous())
    ws = torch.cat([lay(acts[name]).reshape(-1) for name, _, _ in CONV_T._ACTS] +
                   [torch.full((64,), float("nan"))])
    assert ws.numel() * 4 == _lib.load().casmvs_costreg_workspace_bytes(B, cin, D, h, w)
    return lay(acts["x"]), ws, acts["logits"][..., 0].contiguous()


def _check_small(acts, layers):
    cin, B, D, h, w = _SMALL
    x, ws, logits = _pack(acts)
    check_costreg_elements("simulated costreg", x, ws, logits, layers, B, D, h, w, range(B))


def test_simulated_costreg_workspace_passes():
    _check_small(*_small_net())


def test_check_catches_the_last_element_reading_element_0():
    """u9 of the last batch element is element 0's (a batch offset dropped in conv9)."""
    acts, layers = _small_net()
    B = _SMALL[1]
    acts["u9"][B - 1] = acts["u9"][0]
    with pytest.raises(AssertionError) as e:
        _check_small(acts, layers)
    print(e.value)
    assert f"b={B - 1} layer 8 (u9)" in str(e.value)


@pytest.mark.parametrize("plane", [0, 5])
def test_check_catches_one_depth_plane_of_the_last_element(plane):
    """One depth plane of the last element's c0 holds element 0's values (a depth chunk
    stored at the wrong batch offset): the check fails at that element, layer and plane."""
    acts, layers = _small_net()
    B = _SMALL[1]
    acts["c0"][B - 1, plane] = acts["c0"][0, plane]
    with pytest.raises(AssertionError) as e:
        _check_small(acts, layers)
    print(e.value)
    msg = str(e.value)
    assert f"b={B - 1} layer 0 (c0)" in msg and f"(b,d,h,w,c)=(0, {plane}," in msg
