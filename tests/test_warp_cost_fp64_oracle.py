"""The float64 cost-volume reference (oracle/warp_cost_fp64.py) and the per-element bound the GPU
tests hold the K1 kernels and their backward to: the reference against F.grid_sample applied to
the reference formula in float64, an fp32 restatement of the kernels inside the bound at every
element (stress poses included), and -- without a GPU -- proof that the bound, at the loosest
setting a GPU test may commit, flags the subtle ways a cost-volume kernel goes wrong."""
import pytest
import torch
import torch.nn.functional as F

from casmvsnet_pl_b200 import synth
from oracle import casmvs_oracle as O
from oracle import warp_cost_fp64 as W
import test_gpu_warp_cost_fp64 as G

torch.set_default_dtype(torch.float32)


def _inputs(V, C, h, w, D, stress, seed, B=2):
    """Features (B, V, C, h, w) ~ N(0,1), projections and hypotheses that differ per batch item;
    stress: rolled / pitched views and view 1 crossing q_z = 0 inside the sweep."""
    g = torch.Generator().manual_seed(seed)
    feats = torch.randn(B, V, C, h, w, generator=g)
    pm = synth.projection_matrices(V, W=4 * w, H=4 * h, stress=stress,
                                   behind_view=1 if stress else None)[:, 2]
    pm = pm.unsqueeze(0).repeat(B, 1, 1, 1)
    for b in range(1, B):
        pm[b, :, 0, 2] += 1.37 * b
        pm[b, :, 1, 2] -= 0.71 * b
    dv = (560.0 + 15 * torch.arange(D).float().reshape(1, D, 1, 1)
          + torch.rand(B, D, h, w, generator=g) + 7.0 * torch.arange(B).float().reshape(B, 1, 1, 1))
    return feats, pm, dv


def _cl(feats):
    """(B, V, C, h, w) -> (B, V, h, w, C)."""
    return feats.permute(0, 1, 3, 4, 2).contiguous()


def _vol(y):
    """(B, C, D, h, w) -> (B, D, h, w, C)."""
    return y.permute(0, 2, 3, 4, 1)


# ------------------------------------------------------------------------------- float64 formula
def _warp_grid_sample64(src, P, dv):
    """O.plane_sweep_warp's formula in float64 (normalise, F.grid_sample, zeros, align_corners)."""
    B, C, h, w = src.shape
    D = dv.shape[1]
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float64),
                            torch.arange(w, dtype=torch.float64), indexing="ij")
    pix = torch.stack([xs.reshape(-1), ys.reshape(-1), torch.ones(h * w, dtype=torch.float64)], 0)
    pix = pix.unsqueeze(0).expand(B, -1, -1).repeat(1, 1, D)
    q = P[:, :, :3] @ pix + P[:, :, 3:] / dv.reshape(B, 1, D * h * w)
    behind = q[:, 2:] <= W.THRESH
    q[:, 0:1][behind] = w
    q[:, 1:2][behind] = h
    q[:, 2:3][behind] = 1
    uv = q[:, :2] / q[:, 2:]
    uv[:, 0] = uv[:, 0] / ((w - 1) / 2) - 1
    uv[:, 1] = uv[:, 1] / ((h - 1) / 2) - 1
    grid = uv.reshape(B, 2, D, h * w).permute(0, 2, 3, 1)
    out = F.grid_sample(src, grid, mode="bilinear", padding_mode="zeros", align_corners=True)
    return out.reshape(B, C, D, h, w)


def _cost_from_warps(ref, warps, G_):
    """Reductions of mvsnet.py in the dtype of the inputs: ref (B, C, h, w), warps of the source
    views (B, C, D, h, w) -> (B, Cout, D, h, w)."""
    V = len(warps) + 1
    r = ref.unsqueeze(2)
    if G_ == 1:
        S = r + sum(warps)
        Q = r * r + sum(x * x for x in warps)
        return Q / V - (S / V) ** 2
    B, C, D, h, w = warps[0].shape
    S = sum(warps)
    return (S * r).reshape(B, G_, C // G_, D, h, w).mean(2) / (V - 1)


@pytest.mark.parametrize("stress", [False, True])
@pytest.mark.parametrize("V,C,G_", [(3, 8, 1), (4, 16, 8), (3, 32, 8), (5, 8, 2)])
def test_reference_equals_grid_sample_float64(V, C, G_, stress):
    feats, pm, dv = _inputs(V, C, 11, 19, 6, stress, seed=V + C)
    f64, P64, d64 = feats.double(), pm.double(), dv.double()
    warps = [_warp_grid_sample64(f64[:, v], P64[:, v - 1], d64) for v in range(1, V)]
    want = _vol(_cost_from_warps(f64[:, 0], warps, G_))
    y64, b0, A = W.cost_ref(_cl(feats), pm, dv, G_)
    assert ((y64 - want).abs().max() / want.abs().max()).item() < 1e-12
    assert (b0 >= 0).all() and (A >= y64.abs() * (1 - 1e-12)).all()
    for v in range(1, V):
        w64, _, _ = W.homo_warp_ref(_cl(feats)[:, v], pm[:, v - 1], dv)
        x = _vol(warps[v - 1])
        assert ((w64 - x).abs().max() / x.abs().max().clamp_min(1e-300)).item() < 1e-12
    if stress:      # view 1 crosses q_z = 0 inside the sweep: both branches are taken
        qz = (pm[:, 0, 2, :3] @ torch.tensor([9.0, 5.0, 1.0])).reshape(-1, 1, 1, 1) + \
            pm[:, 0, 2, 3].reshape(-1, 1, 1, 1) / dv
        assert (qz <= W.THRESH).any() and (qz > W.THRESH).any()


def test_backward_reference_equals_autograd_float64():
    for G_ in (1, 8):
        feats, pm, dv = _inputs(3, 16, 9, 13, 5, True, seed=3 + G_)
        f64 = feats.double().requires_grad_(True)
        warps = [_warp_grid_sample64(f64[:, v], pm[:, v - 1].double(), dv.double()) for v in (1, 2)]
        cost = _cost_from_warps(f64[:, 0], warps, G_)
        up = torch.randn(cost.shape, generator=torch.Generator().manual_seed(G_)).double()
        (cost * up).sum().backward()
        g64, b0, M, _ = W.warp_cost_bwd_ref(_cl(feats), pm, dv, _vol(up).float().contiguous(), G_)
        want = _cl(f64.grad)
        assert ((g64 - want).abs().max() / want.abs().max()).item() < 1e-12
        assert (b0 >= 0).all() and (M >= g64.abs() * (1 - 1e-12)).all()


# ------------------------------------------------------------------------------- fp32 restatement
def _warp32(src, P, dv, defect=None):
    """O.plane_sweep_warp_direct in fp32, written out so that a defect can be injected:
    "nw_sw" / "ne_sw" swap two tap weights, "border" reads column w-2 for u in [w-1, w),
    "bwd_ne_right" scatters the ne tap's gradient one column to the right."""
    B, C, h, w = src.shape
    D = dv.shape[1]
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32),
                            torch.arange(w, dtype=torch.float32), indexing="ij")
    out = []
    for b in range(B):
        p = P[b]
        inv_d = 1.0 / dv[b]
        qx = p[0, 0] * xs + p[0, 1] * ys + p[0, 2] + p[0, 3] * inv_d
        qy = p[1, 0] * xs + p[1, 1] * ys + p[1, 2] + p[1, 3] * inv_d
        qz = p[2, 0] * xs + p[2, 1] * ys + p[2, 2] + p[2, 3] * inv_d
        behind = qz <= 1e-7
        u = torch.where(behind, torch.full_like(qx, float(w)), qx / qz)
        v = torch.where(behind, torch.full_like(qy, float(h)), qy / qz)
        x0, y0 = torch.floor(u), torch.floor(v)
        fx, fy = u - x0, v - y0
        wts = [(1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy]
        if defect == "nw_sw":
            wts[0], wts[2] = wts[2], wts[0]
        if defect == "ne_sw":
            wts[1], wts[2] = wts[2], wts[1]
        acc = torch.zeros(C, D, h, w)
        for i, ((dy, dx), wgt) in enumerate(zip(((0, 0), (0, 1), (1, 0), (1, 1)), wts)):
            xi, yi = x0 + dx, y0 + dy
            ok = (xi >= 0) & (xi <= w - 1) & (yi >= 0) & (yi <= h - 1)
            xc = xi.clamp(0, w - 1).long()
            if defect == "border" and dx == 0:
                xc = torch.where(x0 == w - 1, xc - 1, xc)
            yc = yi.clamp(0, h - 1).long()
            tap = src[b][:, yc, xc]
            if defect == "bwd_ne_right" and i == 1:
                xr = (xc + 1).clamp(max=w - 1)
                tap = src[b][:, yc, xr] + (tap - src[b][:, yc, xr]).detach()
            acc = acc + tap * (wgt * ok)
        out.append(acc)
    return torch.stack(out)


def _cost32(feats, pm, dv, G_, defect=None, warp_defect=None):
    V = feats.shape[1]
    warps = []
    for v in range(1, V):
        P, d = pm[:, v - 1], dv
        if defect == "batch_proj":
            P = P.clone()
            P[1] = P[0]
        if defect == "prev_plane":
            d = torch.cat([dv[:, :1], dv[:, :-1]], 1)
        x = _warp32(feats[:, v], P, d, warp_defect)
        if defect == "drop_view_run_end" and v == V - 1:
            x = x.clone()
            x[:, :, 15::16] = 0
        warps.append(x)
    if defect == "var_mean_vm1":
        r = feats[:, 0].unsqueeze(2)
        S = r + sum(warps)
        Q = r * r + sum(x * x for x in warps)
        return _vol(Q / V - (S / (V - 1)) ** 2)
    y = _vol(_cost_from_warps(feats[:, 0], warps, G_))
    if defect == "group_shift":
        y = y.clone()
        y[..., 3] = y[..., 4]
    return y


def test_restatement_matches_oracle_direct():
    feats, pm, dv = _inputs(3, 8, 10, 14, 4, True, seed=1)
    for v in (1, 2):
        assert torch.equal(_warp32(feats[:, v], pm[:, v - 1], dv),
                           O.plane_sweep_warp_direct(feats[:, v], pm[:, v - 1], dv))


CASES = [(3, 8, 1, 7, 23, 6), (3, 16, 8, 6, 35, 5), (4, 32, 8, 5, 21, 4), (3, 32, 4, 9, 10, 5),
         (8, 8, 1, 6, 12, 3)]


@pytest.mark.parametrize("stress", [False, True])
@pytest.mark.parametrize("V,C,G_,h,w,D", CASES)
def test_fp32_restatement_within_bound(V, C, G_, h, w, D, stress):
    """Every element, no quantile: K_Q, C_DIV, EPS_BLEND and the committed eps are not too tight
    for fp32 arithmetic with more roundings than the kernels (IEEE division, unfused sums)."""
    feats, pm, dv = _inputs(V, C, h, w, D, stress, seed=h * w + C)
    y = _cost32(feats, pm, dv, G_)
    fam = "gather"
    rep = W.check_cost(y, _cl(feats), pm, dv, G_, G.EPS[fam])
    print(f"fp32 restatement V={V} C={C} G={G_} stress={stress}: {rep.describe()}")
    assert rep.ok, rep.describe()
    if not stress:
        assert rep.loose == 0, rep.describe()
    else:
        assert rep.loose_share <= G.LOOSE_CEIL["cost"], rep.describe()
    hw = O.plane_sweep_warp_direct(feats[:, 1], pm[:, 0], dv)
    rep = W.check_homo_warp(_vol(hw), _cl(feats)[:, 1], pm[:, 0], dv, G.EPS["homo"])
    assert rep.ok, rep.describe()


@pytest.mark.parametrize("stress", [False, True])
@pytest.mark.parametrize("G_", [1, 8])
def test_fp32_backward_within_bound(G_, stress):
    feats, pm, dv = _inputs(3, 16, 12, 17, 6, stress, seed=G_ + 40)
    with torch.enable_grad():
        f = feats.clone().requires_grad_(True)
        y = _cost32(f, pm, dv, G_)
        up = torch.randn(y.shape, generator=torch.Generator().manual_seed(9))
        (y * up).sum().backward()
    rep = W.check_warp_cost_bwd(_cl(f.grad), _cl(feats), pm, dv, up, G_, G.EPS["bwd"])
    print(f"fp32 backward G={G_} stress={stress}: {rep.describe()}")
    assert rep.ok, rep.describe()
    assert rep.loose_share <= (G.LOOSE_CEIL["bwd"] if stress else 0.0), rep.describe()


# ------------------------------------------------------------------------------- discrimination
def test_committed_tolerances_within_ceilings():
    for fam, eps in G.EPS.items():
        assert 0 < eps <= G.EPS_CEIL[fam], fam
    for fam, c in G.LOOSE_CEIL.items():
        assert 0 <= c <= G.LOOSE_CEIL_MAX, fam


def _flags(y, feats, pm, dv, G_, fam="gather"):
    rep = W.check_cost(y, _cl(feats), pm, dv, G_, G.EPS_CEIL[fam])
    return not rep.ok, rep


@pytest.mark.parametrize("defect", ["nw_sw", "ne_sw", "border"])
def test_flags_wrong_tap(defect):
    feats, pm, dv = _inputs(3, 8, 9, 21, 5, False, seed=5)
    if defect == "border":
        # pure translations: u = x + 0.25 + 2/d lands in [w-1, w) for the last two columns
        pm = torch.zeros_like(pm)
        pm[:, :, 0, 0] = pm[:, :, 1, 1] = pm[:, :, 2, 2] = 1
        pm[:, :, 0, 2] = 0.25
        pm[:, :, 0, 3] = 2.0
        dv = torch.full_like(dv, 4.0)
    for G_ in (1, 8):
        y = _cost32(feats, pm, dv, G_, warp_defect=defect)
        flagged, rep = _flags(y, feats, pm, dv, G_)
        assert flagged, (defect, rep.describe())
        if defect == "border":
            assert rep.worst["at"][3] >= 21 - 2, rep.describe()


def test_flags_plane_sampled_at_previous_hypothesis():
    feats, pm, dv = _inputs(3, 16, 8, 12, 7, False, seed=6)
    y = _cost32(feats, pm, dv, 1, defect="prev_plane")
    flagged, rep = _flags(y, feats, pm, dv, 1)
    assert flagged and rep.worst["at"][1] >= 1, rep.describe()


def test_flags_view_dropped_at_run_end():
    feats, pm, dv = _inputs(3, 8, 6, 10, 20, False, seed=7)
    for G_ in (1, 8):
        y = _cost32(feats, pm, dv, G_, defect="drop_view_run_end")
        flagged, rep = _flags(y, feats, pm, dv, G_)
        assert flagged and rep.worst["at"][1] == 15, rep.describe()


def test_flags_batch_item_with_item0_projection():
    feats, pm, dv = _inputs(3, 8, 8, 14, 4, False, seed=8)
    y = _cost32(feats, pm, dv, 1, defect="batch_proj")
    flagged, rep = _flags(y, feats, pm, dv, 1)
    assert flagged and rep.worst["at"][0] == 1, rep.describe()


def test_flags_group_written_with_next_group():
    feats, pm, dv = _inputs(3, 32, 7, 11, 4, False, seed=9)
    y = _cost32(feats, pm, dv, 8, defect="group_shift")
    flagged, rep = _flags(y, feats, pm, dv, 8)
    assert flagged and rep.worst["at"][4] == 3, rep.describe()


def test_flags_variance_mean_over_v_minus_1():
    feats, pm, dv = _inputs(3, 8, 7, 11, 4, False, seed=10)
    y = _cost32(feats, pm, dv, 1, defect="var_mean_vm1")
    assert _flags(y, feats, pm, dv, 1)[0]


def test_flags_backward_tap_scattered_one_column_right():
    feats, pm, dv = _inputs(3, 16, 10, 15, 5, False, seed=11)
    for G_ in (1, 8):
        with torch.enable_grad():
            f = feats.clone().requires_grad_(True)
            y = _cost32(f, pm, dv, G_, warp_defect="bwd_ne_right")
            up = torch.randn(y.shape, generator=torch.Generator().manual_seed(2))
            (y * up).sum().backward()
        rep = W.check_warp_cost_bwd(_cl(f.grad), _cl(feats), pm, dv, up, G_, G.EPS_CEIL["bwd"])
        assert not rep.ok and rep.worst["at"][1] >= 1, rep.describe()
