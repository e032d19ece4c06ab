"""Screened Poisson on the GPU (poisson.py's point_weight, the casmvs_poisson_screen_* kernels):
each kernel call per element against float64 (oracle/poisson_screen_oracle.py) on every level at
depths 6-8, the reductions against fsum, then end to end: convergence at depths 6-10, closed
meshes, the cube's fidelity against the unscreened mesh, identical bytes, eval_pipeline and the
memory refusal.  Admissible errors: moments 1e-12 relative (double sums); each float32 result
within EPS * sum of |terms| (plus one rounding of the result)."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, mesh, poisson, synth_dtu, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import mesh_oracle as M
from oracle import poisson_oracle as O
from oracle import poisson_screen_oracle as Q

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = 1e-6                 # float32 stencil updates: a few roundings of the sum of |terms|
U = 2.0 ** -24


def _cuda(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dtu():
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        p = synth_dtu.make_scene(d, n_stl=2000, n_data=40_000, seed=2)
    cams = synth_dtu.CENTER + np.array([[0, 0, -500.0], [80, 0, -480], [-80, 40, -490]])
    return p, cams


def _run(depth, cloud="sphere", alpha=4.0, keep_fields=True):
    if cloud == "sphere":
        p, n = O.sphere(200_000, seed=0, noise=0.001)
        kw = dict(normals=_cuda(n))
    elif cloud == "cube":
        p, n, _ = Q.cube(300_000, seed=0)
        kw = dict(normals=_cuda(n))
    else:
        p, cams = _dtu()
        kw = dict(cam_centres=cams)
    fields = {} if keep_fields else None                  # depth 10's fields fill most of the card
    out = poisson.poisson_mesh(_cuda(p), depth=depth, point_weight=alpha, fields=fields, **kw)
    return fields, out


def _layout(x, n, level):
    """A level's n^3 array -> the oracle layout ((n + 1)^3 on coarse levels)."""
    x = np.asarray(x, np.float64).reshape(n, n, n)
    return x if level == 0 else np.pad(x, ((0, 1),) * 3)


@pytest.fixture(scope="module", params=[6, 7, 8])
def screened(request):
    fields, out = _run(request.param)
    return request.param, fields, out


def test_moments_and_coarsened_moments(screened):
    depth, f, (_, _, _, st) = screened
    N = 1 << depth
    idx = f["index"].cpu().numpy()
    p, _ = O.sphere(200_000, seed=0, noise=0.001)
    g = O.grid(p, depth)
    pk = p[idx]                                           # the kept points in sorted order
    levels = [(k.cpu().numpy(), m.cpu().numpy()) for k, m in f["levels"]]
    assert len(levels) == depth - 2
    want = Q.moments(pk, g, 0)
    assert np.array_equal(levels[0][0], want[0])
    assert np.abs(levels[0][1] - want[1]).max() <= 1e-12 * np.abs(want[1]).max()
    n = N
    for l in range(1, len(levels)):
        ck, cm = Q.coarsen(*levels[l - 1], n)
        assert np.array_equal(levels[l][0], ck), l
        assert np.abs(levels[l][1] - cm).max() <= 1e-12 * np.abs(cm).max(), l
        direct = Q.moments(pk, g, l)
        assert np.abs(levels[l][1] - direct[1]).max() <= 1e-12 * np.abs(direct[1]).max(), l
        n //= 2
    assert f["g"] == 4.0 * len(levels[0][0]) / st["points"]


def test_screened_rhs(screened):
    depth, f, (_, _, _, st) = screened
    N, h = 1 << depth, st["h"]
    keys, mom = (x.cpu().numpy() for x in f["levels"][0])
    _, Phi = Q.screen_matrix(keys, mom, N, N)           # moments are >= 0, and so is Phi
    b = f["b"].cpu().numpy().astype(np.float64).reshape(N, N, N)
    gt = f["g"] / (h * h) * st["target"]
    want = np.where(O._interior(N), b - gt * Phi, 0.0)
    got = f["b_s"].cpu().numpy().reshape(N, N, N)
    bound = U * np.abs(want) + 1e-12 * (np.abs(b) + abs(gt) * (Phi + 8 * mom[:, 0].max()))
    assert (np.abs(got - want) <= bound).all()
    total = math.fsum((got.astype(np.float64).reshape(-1) ** 2).tolist())
    assert abs(f["bb_s"] - total) <= 1e-12 * total


def _level(f, st, l):
    n = st["N"] >> l
    keys, mom = (x.cpu().numpy() for x in f["levels"][l])
    S, _ = Q.screen_matrix(keys, mom, n, n if l == 0 else n + 1)
    k, m = f["levels"][l]
    cmap, mask = poisson._cell_map(k, n), poisson._corner_mask(k, n)
    srow, s32, s64 = poisson._stencils(cmap, mask, m, n, l == 0)
    return n, S, abs(S), mask, srow, s32, s64


def _random_field(n, level, seed):
    rng = np.random.default_rng(seed)
    e = rng.normal(size=(n, n, n)).astype(np.float32)
    inner = O._interior(n + (level > 0))[:n, :n, :n] if level else O._interior(n)
    return np.where(inner, e, 0).astype(np.float32)


def test_residuals_and_smoother_on_every_level(screened):
    depth, f, (_, _, _, st) = screened
    lib, N = _lib.load(), st["N"]
    h, g = st["h"], f["g"]
    for l in range(depth - 2):
        n, S, Sabs, mask, srow, s32, _ = _level(f, st, l)
        hl = float(np.float32(h * (1 << l)))
        gl = g / 2 ** l
        e = _random_field(n, l, 10 + l)
        r = _random_field(n, l, 20 + l) / np.float32(hl * hl)
        et, rt = _cuda(e.reshape(-1)), _cuda(r.reshape(-1))
        E, R = _layout(e, n, l), _layout(r, n, l)
        inner = O._interior(len(E))
        # float32 multigrid residual
        out = torch.empty_like(et)
        _lib.check(lib.casmvs_poisson_screen_mg_residual(_p(et), _p(rt), _p(mask), _p(srow), _p(s32),
                                                         n, l, hl, g, _p(out), _st()), "mg_residual")
        want = np.where(inner, R - Q.apply_screened(E, hl, S, gl), 0.0)
        absE = np.abs(E)
        terms = np.abs(R) + (O._nbsum(absE) + 6 * absE + gl * (Sabs @ absE.reshape(-1)).reshape(E.shape)) / hl ** 2
        got = _layout(out.cpu().numpy(), n, l)
        assert (np.abs(got - want) <= EPS * terms + 1e-30).all(), ("mg_residual", l)
        # one 8-colour sweep: each colour reads this call's earlier colours
        e2 = et.clone()
        _lib.check(lib.casmvs_poisson_screen_smooth(_p(e2), _p(rt), _p(mask), _p(srow), _p(s32), n, l,
                                                    hl, g, 1, 0, _st()), "smooth")
        want = Q.smooth(E.copy(), R, hl, S, gl, 1)
        aw = np.abs(want)
        terms = (O._nbsum(aw) + hl * hl * np.abs(R) + gl * (Sabs @ aw.reshape(-1)).reshape(E.shape)) / 6
        got = _layout(e2.cpu().numpy(), n, l)
        # a colour's rounding reaches the later colours of the sweep: up to 8 updates in a chain
        worst = float((np.abs(got - want) / (terms + 1e-30)).max())
        assert worst <= 8 * EPS, ("smooth", l, worst)
        if n == 8:                                           # the one-block coarsest kernel
            e3 = torch.empty_like(et)
            _lib.check(lib.casmvs_poisson_screen_smooth(_p(e3), _p(rt), _p(mask), _p(srow), _p(s32),
                                                        n, l, hl, g, 50, 1, _st()), "smooth")
            want = Q.smooth(np.zeros_like(E), R, hl, S, gl, 50)
            got = _layout(e3.cpu().numpy(), n, l)
            assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max(), "coarsest"
    # the double residual on level 0 and its ||r||^2 against fsum
    n, S, Sabs, mask, srow, _, s64 = _level(f, st, 0)
    chi = f["chi"]
    bs = f["b_s"]
    ws = torch.empty(lib.casmvs_poisson_workspace_bytes(N ** 3) // 8, dtype=torch.float64, device=DEV)
    rr = torch.zeros(1, dtype=torch.float64, device=DEV)
    r = torch.empty(N ** 3, dtype=torch.float32, device=DEV)
    _lib.check(lib.casmvs_poisson_screen_residual(_p(chi), _p(bs), _p(mask), _p(srow), _p(s64), N, h,
                                                  g, _p(r), _p(ws), _p(rr), _st()), "residual")
    C = chi.cpu().numpy().reshape(N, N, N)
    B = bs.cpu().numpy().astype(np.float64).reshape(N, N, N)
    want = np.where(O._interior(N), B - Q.apply_screened(C, h, S, g), 0.0)
    aC = np.abs(C)
    terms = np.abs(B) + (O._nbsum(aC) + 6 * aC + g * (Sabs @ aC.reshape(-1)).reshape(C.shape)) / (h * h)
    got = r.cpu().numpy().reshape(N, N, N)
    assert (np.abs(got - want) <= U * np.abs(want) + 1e-13 * terms + 1e-300).all()
    total = math.fsum((want.reshape(-1) ** 2).tolist())
    assert abs(float(rr.item()) - total) <= 1e-9 * total + 1e-300
    # the screened iso level: the mean of chi at the kept points
    p, _ = O.sphere(200_000, seed=0, noise=0.001)
    pk = p[f["index"].cpu().numpy()]
    base, frac = O._corners(pk, O.grid(p, depth))
    c = C.reshape(-1)
    terms = [float(w) * c[i] for d in O.CORNERS
             for w, i in zip(O.trilinear(frac, d).astype(np.float64), O.flat(base + np.array(d), N))]
    want = math.fsum(terms) / len(pk)
    assert abs(f["iso"] - want) <= 1e-10 * max(abs(want), np.abs(C).max())


@pytest.mark.parametrize("cloud", ["sphere", "dtu", "cube"])
def test_screened_solve_converges_at_every_depth(cloud):
    cycles = []
    for depth in range(6, 11):
        _, (_, _, f, st) = _run(depth, cloud, keep_fields=False)
        assert st["screened_ratios"][-1] <= 1e-5 and st["screened_cycles"] <= 40, (cloud, depth)
        assert len(f) > 0
        cycles.append(st["screened_cycles"])
        torch.cuda.empty_cache()
    print(f"screened cycles, {cloud}, depths 6-10 at alpha 4: {cycles}")


def test_screened_sphere_and_cube_meshes_are_closed_and_outward():
    for cloud in ("sphere", "cube"):
        _, (v, _, f, st) = _run(8, cloud)
        v, f = v.cpu().numpy(), f.cpu().numpy()
        assert M.is_closed_oriented(f) and M.euler_characteristic(len(v), f) == 2, cloud
        assert M.signed_volume(v, f) > 0, cloud
        if cloud == "sphere":
            d = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 1.0)
            assert d.max() < 1.0 * st["h"]


def test_screening_brings_the_cube_mesh_closer_to_the_cube():
    p, n, q = Q.cube(1_000_000, side=1.0, seed=3)
    res = {}
    for alpha in (0.0, 4.0):
        v, _, f, st = poisson.poisson_mesh(_cuda(p), normals=_cuda(n), depth=8, point_weight=alpha)
        d = Q.cube_distance(v.cpu().numpy(), q)
        res[alpha] = (d.mean(), np.percentile(d, 95), st["h"])
    print("cube side 1, depth 8: mean / p95 distance (h = %.5f): alpha 0: %.3e / %.3e, "
          "alpha 4: %.3e / %.3e" % (res[0][2], res[0][0], res[0][1], res[4][0], res[4][1]))
    assert res[4.0][0] < res[0.0][0] and res[4.0][1] < res[0.0][1]


def test_screened_bytes_are_reproducible_and_alpha_zero_is_the_unscreened_path(tmp_path):
    views = synth_scenes.sphere_scene(8, (320, 240), seed=1, device=DEV)
    p = torch.cat([v["points"] for v in views])
    rgb = torch.cat([v["image"][v["depth"] > 0] for v in views]).to(torch.uint8)
    cams = np.stack([-np.linalg.inv(v["P"][:3, :3].astype(np.float64)) @ v["P"][:3, 3] for v in views])
    out = {}
    for tag, kw in (("s1", dict(point_weight=4.0)), ("s2", dict(point_weight=4.0)),
                    ("z", dict(point_weight=0.0)), ("plain", {})):
        v, c, f, st = poisson.poisson_mesh(p, rgb, cam_centres=cams, depth=8, **kw)
        mesh.write_mesh_ply(tmp_path / f"{tag}.ply", v, c, f)
        out[tag] = (tmp_path / f"{tag}.ply").read_bytes()
    assert out["s1"] == out["s2"] and out["z"] == out["plain"] and out["s1"] != out["plain"]


def _tree_bytes(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


def test_eval_pipeline_screened_mesh_changes_only_the_mesh(tmp_path):
    from casmvsnet_pl_b200 import ABN, synth
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    root = tmp_path / "capture"
    synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), n_points=3000, seed=7)
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(model, 0)
    ckpt = tmp_path / "weights.pt"
    torch.save(model.state_dict(), ckpt)
    common = ["--dataset_name", "colmap", "--root_dir", str(root), "--img_wh", "128", "96",
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt),
              "--mesh", "--mesh_method", "poisson", "--poisson_depth", "7"]
    ep.main(common + ["--out", str(tmp_path / "p")])
    ep.main(common + ["--out", str(tmp_path / "s"), "--poisson_point_weight", "4"])
    plain, scr = _tree_bytes(tmp_path / "p"), _tree_bytes(tmp_path / "s")
    mesh_file = os.path.join("mesh", "capture.ply")
    assert scr.keys() == plain.keys()
    assert {k: v for k, v in scr.items() if k != mesh_file} == \
        {k: v for k, v in plain.items() if k != mesh_file}
    assert scr[mesh_file] != plain[mesh_file]


def test_a_screened_grid_that_does_not_fit_is_refused_with_a_depth_that_would():
    p, n = O.sphere(10_000, seed=6)
    budget = poisson._bytes_needed(8, len(p), screen=True) - 1
    with pytest.raises(_lib.CasMVSError, match="screening.*depth 7 would fit"):
        poisson.poisson_mesh(_cuda(p), normals=_cuda(n), depth=8, max_bytes=budget, point_weight=4)
    _, _, f, st = poisson.poisson_mesh(_cuda(p), normals=_cuda(n), depth=7, max_bytes=budget,
                                       point_weight=4)
    assert len(f) > 0 and st["screened_ratios"][-1] <= 1e-5


def _box(t, n, w, margin=0):
    """The window w = (x0, y0, z0, x1, y1, z1) of a level's n^3 device array grown by `margin`
    and clipped to the grid -> (host float64 box, origin)."""
    lo = [max(v - margin, 0) for v in w[:3]]
    hi = [min(v + margin, n) for v in w[3:]]
    a = t.reshape(n, n, n)[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
    return a.double().cpu().numpy(), np.array(lo)


def _nodes(shape, origin):
    return np.indices(shape).reshape(3, -1).T + origin


@pytest.mark.parametrize("depth", [9, 10])
def test_kernels_in_windows_at_depths_9_and_10(depth):
    """Every screening kernel call per element in the windows of oracle/poisson_fp64.windows
    (corners, face centres, boxes around surface nodes, the last x-slabs) on every level."""
    from oracle import poisson_fp64 as F
    lib = _lib.load()
    p, _ = O.sphere(200_000, seed=0, noise=0.001)
    g = O.grid(p, depth)
    N, h, lo = g["N"], g["h"], [int(v) for v in g["lo"]]
    levels = poisson._screen_levels(_cuda(p), N, h, lo)
    n_s = len(levels[0]["keys"])
    gg = 4.0 * n_s / len(p)
    gen = torch.Generator(device=DEV).manual_seed(depth)
    prev = None
    for l, lv in enumerate(levels):
        n = N >> l
        keys, mom = lv["keys"].cpu().numpy(), lv["moments"].cpu().numpy()
        # moments: level 0 from the points, coarser levels from their children and the points
        want_k, want_m = Q.moments(p, g, l)
        assert np.array_equal(keys, want_k), l
        assert np.abs(mom - want_m).max() <= 1e-12 * np.abs(want_m).max(), l
        if prev is not None:
            ck, cm = Q.coarsen(*prev, 2 * n)
            assert np.array_equal(keys, ck) and np.abs(mom - cm).max() <= 1e-12 * np.abs(cm).max()
        prev = (keys, mom)
        top = n if l else n - 1
        idx = torch.arange(n, device=DEV)
        inner1 = (idx > 0) & (idx < top)
        inner = (inner1[:, None, None] & inner1[None, :, None] & inner1[None, None, :]).reshape(-1)
        hl = float(np.float32(h * (1 << l)))
        gl = gg / 2 ** l
        e = torch.randn(n ** 3, generator=gen, device=DEV) * inner
        r = torch.randn(n ** 3, generator=gen, device=DEV) * inner / (hl * hl)
        surf = [tuple(int(v) for v in keys[len(keys) // k] // np.array([n * n, n, 1]) % n)
                for k in (2, 3, 5)]
        wins = F.windows(n, surface=surf)
        ops = (_p(lv["mask"]), _p(lv["srow"]), _p(lv["stencil"]), n, l, hl, gg)
        out = torch.empty_like(e)
        _lib.check(lib.casmvs_poisson_screen_mg_residual(_p(e), _p(r), *ops, _p(out), _st()), "mg_res")
        e2 = e.clone()
        _lib.check(lib.casmvs_poisson_screen_smooth(_p(e2), _p(r), *ops, 1, 0, _st()), "smooth")
        for w in wins:
            E, o = _box(e, n, w, 9)
            R, _ = _box(r, n, w, 9)
            rows, _ = Q.stencil_rows(_nodes(E.shape, o), keys, mom, n)
            # the float32 multigrid residual, on the box's interior
            Ep = np.pad(E, 1)                            # outside the grid reads 0
            c = (slice(1, -1),) * 3
            nb = sum(np.roll(Ep, s, a)[c] for a in range(3) for s in (1, -1))
            shifted = [np.roll(Ep, tuple(-d for d in Q.OFFSETS[k]), (0, 1, 2))[c].reshape(-1)
                       for k in range(27)]
            se = sum(rows[:, k] * shifted[k] for k in range(27)).reshape(E.shape)
            sabs = sum(np.abs(rows[:, k] * shifted[k]) for k in range(27)).reshape(E.shape)
            gidx = _nodes(E.shape, o).reshape(E.shape + (3,))
            gin = ((gidx > 0) & (gidx < top)).all(-1)
            want = np.where(gin, R - (nb - 6 * E - gl * se) / hl ** 2, 0.0)
            terms = np.abs(R) + (sum(np.abs(np.roll(Ep, s, a)[c]) for a in range(3) for s in (1, -1))
                                 + 6 * np.abs(E) + gl * sabs) / hl ** 2
            got, _ = _box(out, n, w, 9)
            edge = ((gidx >= o + 1) & (gidx < o + np.array(E.shape) - 1)).all(-1)
            bad = edge & (np.abs(got - want) > EPS * terms + 1e-30)
            assert not bad.any(), ("mg_residual", depth, l, w)
            # one 8-colour sweep, exact 8 or more nodes inside the grown box
            Ew, Rw = np.pad(E, 1), np.pad(R, 1)          # so that a node at n - 1 is updated
            roww, _ = Q.stencil_rows(_nodes(Ew.shape, o - 1), keys, mom, n)
            want = Q.window_sweep(Ew, Rw, o - 1, n, l, hl, gl, roww)[1:-1, 1:-1, 1:-1]
            got, _ = _box(e2, n, w, 9)
            core = ((gidx >= np.asarray(w[:3])) & (gidx < np.asarray(w[3:]))).all(-1)
            aw = np.abs(want)
            nbw = O._nbsum(np.pad(aw, 1))[1:-1, 1:-1, 1:-1]  # the box's outer layer has neighbours too
            terms = (nbw + hl * hl * np.abs(R) + gl * sabs) / 6 + np.abs(want)
            assert (np.abs(got - want)[core] <= (8 * EPS * terms + 1e-30)[core]).all(), \
                ("smooth", depth, l, w)
        del e, r, out, e2
        torch.cuda.empty_cache()
    # level 0: the screened right-hand side and the double residual in the same windows
    lv = levels[0]
    keys, mom = lv["keys"].cpu().numpy(), lv["moments"].cpu().numpy()
    b = torch.randn(N ** 3, generator=gen, device=DEV)
    gt = 3.0 / (h * h)
    bs = torch.empty_like(b)
    ws = torch.empty(lib.casmvs_poisson_workspace_bytes(N ** 3) // 8, dtype=torch.float64, device=DEV)
    bb = torch.zeros(1, dtype=torch.float64, device=DEV)
    _lib.check(lib.casmvs_poisson_screen_rhs(_p(b), _p(lv["mask"]), _p(lv["map"]), _p(lv["moments"]),
                                             N, gt, _p(bs), _p(ws), _p(bb), _st()), "rhs")
    total = float((bs.double() ** 2).sum())
    assert abs(float(bb.item()) - total) <= 1e-10 * total
    chi = torch.randn(N ** 3, generator=gen, device=DEV, dtype=torch.float64)
    idx = torch.arange(N, device=DEV)
    i1 = (idx > 0) & (idx < N - 1)
    chi *= (i1[:, None, None] & i1[None, :, None] & i1[None, None, :]).reshape(-1)
    rr = torch.zeros(1, dtype=torch.float64, device=DEV)
    r = torch.empty_like(b)
    _lib.check(lib.casmvs_poisson_screen_residual(_p(chi), _p(bs), _p(lv["mask"]), _p(lv["srow"]),
                                                  _p(lv["stencil64"]), N, h, gg, _p(r), _p(ws),
                                                  _p(rr), _st()), "residual")
    surf = [tuple(int(v) for v in keys[len(keys) // k] // np.array([N * N, N, 1]) % N) for k in (2, 3)]
    for w in F.windows(N, surface=surf):
        B, o = _box(b, N, w)
        C, _ = _box(chi, N, w, 1)
        nodes = _nodes(B.shape, o)
        rows, phi = Q.stencil_rows(nodes, keys, mom, N)
        gin = ((nodes > 0) & (nodes < N - 1)).all(1).reshape(B.shape)
        want = np.where(gin, B - gt * phi.reshape(B.shape), 0.0)
        got, _ = _box(bs, N, w)
        bound = U * np.abs(want) + 1e-12 * (np.abs(B) + gt * (phi.reshape(B.shape) + 8 * mom[:, 0].max()))
        assert (np.abs(got - want) <= bound).all(), ("rhs", depth, w)
        Cp = np.pad(C, 1)
        s0 = np.array(o) - np.maximum(np.array(w[:3]) - 1, 0) + 1      # offset of the box in Cp
        def at(d):
            sl = tuple(slice(s0[a] + d[a], s0[a] + d[a] + B.shape[a]) for a in range(3))
            return Cp[sl]
        Bs, _ = _box(bs, N, w)
        nb = sum(at(d) for d in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)))
        sc = sum(rows[:, k].reshape(B.shape) * at(Q.OFFSETS[k]) for k in range(27))
        sabs = sum(np.abs(rows[:, k].reshape(B.shape) * at(Q.OFFSETS[k])) for k in range(27))
        want = np.where(gin, Bs - (nb - 6 * at((0, 0, 0)) - gg * sc) / (h * h), 0.0)
        terms = np.abs(Bs) + (np.abs(nb) + 6 * np.abs(at((0, 0, 0))) + gg * sabs) / (h * h)
        got, _ = _box(r, N, w)
        assert (np.abs(got - want) <= U * np.abs(want) + 1e-12 * terms + 1e-300).all(), \
            ("residual", depth, w)
