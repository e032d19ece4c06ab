"""Dynamic consistency fusion (geo_fuse_kernel<kDynamic>, casmvs_geo_fuse_dynamic_fwd) element by
element against float64 (oracle/fusion_dynamic_fp64.py), with no statistical slack:

  * fusion.refine_ref_view(rule="dynamic", debug=True) on the noisy sphere-and-plane scenes of
    test_gpu_fusion_fp64.py at 1152x864, 1600x1200 and 1920x1056 with 10 and 16 sources, and
    with 0, 1, 2 and 3 sources: every level in its admissible set, every reprojection within
    the bound of an admissible candidate, geo_count, mask_final, depth_refined, image_refined
    and points; the non-debug outputs bitwise those of the debug call, and two runs alike;
  * the raw entry on the known-answer cases (bin ties, borders, saturation, qz = 0, NaN / zero /
    negative depths, errors on the level thresholds), and S = 17 refused before device work;
  * fusion.fuse_scan(rule="dynamic") on a ring of 8 views: each call checked on its own inputs,
    those inputs bitwise what the refined-view cache prescribes, and the output the
    concatenation of the calls' outputs;
  * eval_pipeline --fusion dynamic end to end on a Tanks scan, with and without --mesh.
"""
import ctypes

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, eval_pipeline as ep, fusion, io, synth_scenes
from oracle import fusion_dynamic_fp64 as FD
from oracle import fusion_fp64 as FF

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
# Share of (source, pixel) pairs with more than one admissible level.  It depends only on the
# oracle and the data: at most 1.07e-2 over these scenes (1152x864, 2 sources; 9.1e-3 at
# 1920x1056 with 10), about nine times the fixed rule's share, since nine levels put eighteen
# thresholds in the way where that rule has two; the ceiling is the power of two above the worst.
AMBIGUOUS_MAX = 2.0 ** -6

SHAPES = [  # W, H, S
    (1152, 864, 10),
    (1600, 1200, 10),
    (1920, 1056, 10),
    (1152, 864, 16),
    (1152, 864, 3),
    (1152, 864, 2),
    (1152, 864, 1),
    (1152, 864, 0),
]


def _gpu(v):
    return None if v is None else v.to(DEV)


def _refine(inp, debug):
    return fusion.refine_ref_view(_gpu(inp["depth_ref"]), inp["P_ref"],
                                  [_gpu(d) for d in inp["depth_srcs"]], list(inp["P_srcs"]),
                                  _gpu(inp["image_ref"]), [_gpu(i) for i in inp["image_srcs"]],
                                  _gpu(inp["proba_ref"]), conf=inp["conf"], debug=debug,
                                  rule="dynamic")


def _report(tag, inp, out, exact=False):
    rep = FD.check_fuse_dynamic(inp, out, exact=exact, device=DEV)
    print(f"[fp64] dynamic {tag}{' exact' if exact else ''}: {rep.describe()}")
    assert rep.ok, f"{tag}: {rep.describe()}"
    assert rep.ambiguous <= AMBIGUOUS_MAX * max(rep.pairs, 1), f"{tag}: {rep.describe()}"
    return rep


def _scene(W, H, S):
    views = synth_scenes.sphere_scene(max(S + 1, 12), (W, H), seed=W + S, radius=150, device=DEV)
    C = [-np.linalg.solve(v["P"][:3, :3].astype(np.float64), v["P"][:3, 3]) for v in views]
    near = sorted(range(1, len(views)), key=lambda i: np.linalg.norm(C[i] - C[0]))[:S]
    return FF.scene_inputs([views[0]] + [views[i] for i in near], S, seed=W + S)


@pytest.mark.parametrize("W,H,S", SHAPES, ids=[f"{w}x{h}_S{s}" for w, h, s in SHAPES])
def test_refine_ref_view_dynamic_fp64(W, H, S):
    inp = _scene(W, H, S)
    got = _refine(inp, debug=True)
    assert "mask" not in got and got["level"].shape == (S, H, W) and got["level"].dtype == torch.uint8
    rep = _report(f"{W}x{H} S={S}", inp, got)
    plain = _refine(inp, debug=False)
    again = _refine(inp, debug=True)
    for k in ("depth_refined", "image_refined", "geo_count", "mask_final", "points"):
        assert torch.equal(plain[k], got[k]), f"{k} differs with debug"
    for k in ("level", "reproj", "depth_refined", "image_refined", "geo_count", "mask_final", "points"):
        assert torch.equal(again[k], got[k]), f"{k} differs between two runs"
    lv = got["level"].long()
    if S < 2:
        assert not bool(got["mask_final"].any())
    if S >= 10:
        assert rep.certain_true > 0.02 * rep.pairs and rep.certain_false > 0.02 * rep.pairs, rep.describe()
        hist = torch.bincount(lv.reshape(-1), minlength=11).cpu()
        assert bool((hist[2:] > 0).all()), hist          # every level occurs
        # the rules differ: the dynamic mask keeps pixels the fixed rule (5 sources) drops
        ref = fusion.refine_ref_view(_gpu(inp["depth_ref"]), inp["P_ref"],
                                     [_gpu(d) for d in inp["depth_srcs"]], list(inp["P_srcs"]),
                                     _gpu(inp["image_ref"]), [_gpu(i) for i in inp["image_srcs"]],
                                     _gpu(inp["proba_ref"]), conf=inp["conf"], min_geo_consistent=5)
        assert bool((got["mask_final"] & ~ref["mask_final"]).any())


# ------------------------------------------------------------------------------- raw entry
def _raw(inp, S=None, outputs=None):
    """casmvs_geo_fuse_dynamic_fwd with the inputs' own rows -> (status, outputs)."""
    lib = _lib.load()
    d = _gpu(inp["depth_ref"]).contiguous()
    H, W = d.shape
    srcs = [_gpu(x).contiguous() for x in inp["depth_srcs"]]
    imgs = [_gpu(x).contiguous() for x in inp["image_srcs"]]
    n = len(srcs) if S is None else S
    img_ref = _gpu(inp["image_ref"]).contiguous()
    proba = _gpu(inp["proba_ref"])
    rs = np.ascontiguousarray(np.asarray(inp["rs"], np.float32).reshape(-1))
    sr = np.ascontiguousarray(np.asarray(inp["sr"], np.float32).reshape(-1))
    r2w = torch.from_numpy(np.asarray(inp["ref2world"], np.float32)).to(DEV).contiguous()
    f32 = dict(device=DEV, dtype=torch.float32)
    out = outputs or dict(depth_refined=torch.empty(H, W, **f32), image_refined=torch.empty(H, W, 3, **f32),
                          geo_count=torch.empty(H, W, device=DEV, dtype=torch.int32),
                          mask_final=torch.empty(H, W, device=DEV, dtype=torch.uint8),
                          points=torch.empty(H, W, 3, **f32), reproj=torch.empty(max(n, 1), H, W, **f32),
                          level=torch.empty(max(n, 1), H, W, device=DEV, dtype=torch.uint8))
    arr = ctypes.c_void_p * max(len(srcs), 1)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None      # noqa: E731
    fp = ctypes.POINTER(ctypes.c_float)
    rc = lib.casmvs_geo_fuse_dynamic_fwd(
        p(d), p(img_ref), p(proba.contiguous() if proba is not None else None),
        arr(*[x.data_ptr() for x in srcs]), arr(*[x.data_ptr() for x in imgs]),
        rs.ctypes.data_as(fp), sr.ctypes.data_as(fp), p(r2w), n, H, W, float(inp["conf"]),
        p(out["depth_refined"]), p(out["image_refined"]), p(out["geo_count"]), p(out["mask_final"]),
        p(out["points"]), p(out["reproj"]), p(out["level"]),
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, out


@pytest.mark.parametrize("name", [c[0] for c in FD.edge_cases()])
def test_edge_cases_raw_entry(name):
    inp = dict(FD.edge_cases())[name]
    rc, out = _raw(inp)
    _lib.check(rc, "geo_fuse_dynamic")
    S = len(inp["depth_srcs"])
    out = dict(out, level=out["level"][:S], reproj=out["reproj"][:S], mask_final=out["mask_final"].bool())
    for exact in (True, False):
        rep = FD.check_fuse_dynamic(inp, out, exact=exact, device=DEV)
        print(f"[fp64] dynamic edge {name}{' exact' if exact else ''}: {rep.describe()}")
        assert rep.ok, f"{name}: {rep.describe()}"
    if name == "levels":
        # dx = 1/8, 3/8, 1/2, 5/8, 7/8, 1, 11/8, 9/4, 5/2, 3 px: on and between the thresholds
        assert out["level"][:, 5, 5].tolist() == [2, 2, 3, 3, 4, 5, 6, 10, 0, 0]
        assert bool(out["mask_final"][5, 5]) and int(out["geo_count"][5, 5]) == 8
    if name == "confidence":
        assert not bool(out["mask_final"].any())         # S = 0 keeps nothing


def test_seventeen_sources_refused():
    name, inp = FD.edge_cases()[0]
    inp = dict(inp)
    reps = 17 // len(inp["depth_srcs"]) + 1
    for k in ("depth_srcs", "image_srcs"):
        inp[k] = (list(inp[k]) * reps)[:17]
    inp["rs"] = np.concatenate([inp["rs"]] * reps)[:17]
    inp["sr"] = np.concatenate([inp["sr"]] * reps)[:17]
    H, W = inp["depth_ref"].shape
    f32 = dict(device=DEV, dtype=torch.float32)
    sentinel = dict(depth_refined=torch.full((H, W), -7.0, **f32), image_refined=torch.full((H, W, 3), -7.0, **f32),
                    geo_count=torch.full((H, W), -7, device=DEV, dtype=torch.int32),
                    mask_final=torch.full((H, W), 7, device=DEV, dtype=torch.uint8),
                    points=torch.full((H, W, 3), -7.0, **f32), reproj=torch.full((17, H, W), -7.0, **f32),
                    level=torch.full((17, H, W), 77, device=DEV, dtype=torch.uint8))
    before = {k: v.clone() for k, v in sentinel.items()}
    n0 = _lib.launch_count()
    rc, out = _raw(inp, S=17, outputs=sentinel)
    assert rc != 0 and b"at most 16" in _lib.load().casmvs_last_error()
    assert _lib.launch_count() == n0
    for k, v in before.items():
        assert torch.equal(out[k], v), f"{k} written"


# ------------------------------------------------------------------------------- fuse_scan
@pytest.fixture
def recorder(monkeypatch):
    calls = []
    orig = fusion.refine_ref_view

    def f(*a, **k):
        out = orig(*a, **dict(k, debug=True))
        calls.append((a, k, out))
        return out
    monkeypatch.setattr(fusion, "refine_ref_view", f)
    return calls


def _ring(W=400, H=304):
    views = synth_scenes.sphere_scene(8, (W, H), seed=5, radius=150, device=DEV)
    g = torch.Generator().manual_seed(5)
    rng = np.random.default_rng(5)
    depths = {v: (views[v]["depth"].cpu() * (1 + 0.002 * torch.randn(H, W, generator=g))).to(DEV)
              for v in range(8)}
    images = {v: torch.from_numpy(rng.integers(0, 256, (H, W, 3)).astype(np.float32)).to(DEV) for v in range(8)}
    probas = {v: torch.from_numpy(rng.uniform(0.3, 1.0, (H // 4, W // 4)).astype(np.float32)).to(DEV)
              for v in range(8)}
    proj = {v: views[v]["P"] for v in range(8)}
    proj[9] = views[0]["P"]
    return depths, images, probas, proj


METAS = [(0, [1, 7, 2, 6]),
         (1, [0, 2, 7, 3, 6, 4, 5]),      # view 1 was view 0's source; view 0 is refined
         (3, [4, 9, 2]),                  # 9 has no prediction: skipped after caching 4 raw
         (2, [1, 3, 0, 4]),
         (9, [0, 1]),                     # no prediction for the reference itself
         (4, [3, 5, 2]),
         (5, [4, 6, 3, 7]),
         (6, [5, 7, 4, 0]),
         (7, [6, 0, 5, 1])]               # cut by max_ref_views


def test_fuse_scan_dynamic_fp64(recorder):
    depths, images, probas, proj = _ring()
    max_ref, skip, conf = 8, 3, 0.5
    collect = []
    xyz, rgb = fusion.fuse_scan(METAS, depths, probas, images, proj, conf=conf, skip=skip,
                                max_ref_views=max_ref, collect=collect, rule="dynamic")
    refined, k = {}, 0
    for ref, srcs in METAS[:max_ref]:
        if ref not in depths or any(sv not in depths for sv in srcs):
            continue
        a, kw, out = recorder[k]
        assert kw["rule"] == "dynamic"
        dref, iref = refined.get(ref, (depths[ref], images[ref]))
        assert torch.equal(a[0], dref) and torch.equal(a[4], iref), f"call {k} (ref {ref}): reference input"
        assert np.array_equal(np.asarray(a[1], np.float32), proj[ref])
        assert len(a[2]) == len(srcs) and torch.equal(a[6], probas[ref])
        for j, sv in enumerate(srcs):
            ds, im = refined.get(sv, (depths[sv], images[sv]))
            assert torch.equal(a[2][j], ds) and torch.equal(a[5][j], im), f"call {k} (ref {ref}): source {sv}"
            assert np.array_equal(np.asarray(a[3][j], np.float32), proj[sv])
        refined[ref] = (out["depth_refined"], torch.round(out["image_refined"]).clamp(0, 255))
        k += 1
    assert k == len(recorder) and set(refined) == {0, 1, 2, 4, 5, 6}

    for k, (a, kw, out) in enumerate(recorder):
        P_ref, P_srcs = np.asarray(a[1], np.float32), [np.asarray(P, np.float32) for P in a[3]]
        inp = dict(depth_ref=a[0], image_ref=a[4], proba_ref=a[6], depth_srcs=a[2], image_srcs=a[5],
                   rs=np.stack([FF.rel(P, P_ref) for P in P_srcs]).reshape(-1, 12),
                   sr=np.stack([FF.rel(P_ref, P) for P in P_srcs]).reshape(-1, 12),
                   ref2world=np.linalg.inv(P_ref).astype(np.float32), conf=a[7])
        _report(f"fuse_scan call {k}", inp, out)

    want_xyz = torch.cat([o["points"][o["mask_final"]][::skip] for _, _, o in recorder])
    want_rgb = torch.cat([o["image_refined"][o["mask_final"]][::skip] for _, _, o in recorder]).to(torch.uint8)
    assert len(want_xyz) > 1000
    assert torch.equal(xyz, want_xyz) and torch.equal(rgb, want_rgb)
    assert len(collect) == len(recorder)
    for c, (a, _, o) in zip(collect, recorder):
        m = o["mask_final"]
        assert torch.equal(c["depth"], torch.where(m, o["depth_refined"], 0.0))
        assert torch.equal(c["image"], o["image_refined"]) and torch.equal(c["points"], o["points"][m])


def test_fuse_scan_dynamic_is_reproducible():
    depths, images, probas, proj = _ring()
    runs = [fusion.fuse_scan(METAS, depths, probas, images, proj, conf=0.5, rule="dynamic")
            for _ in range(2)]
    assert len(runs[0][0]) > 1000
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    # min_geo_consistent is ignored by the dynamic rule
    other = fusion.fuse_scan(METAS, depths, probas, images, proj, conf=0.5, min_geo_consistent=1,
                             rule="dynamic")
    assert torch.equal(runs[0][0], other[0])


# ------------------------------------------------------------------------------- eval_pipeline
class _PlaneModel(torch.nn.Module):
    """Stands in for CascadeMVSNet: each reference view's depth is that of the world plane
    z = Z0 the synthetic Tanks cameras look at, with confidence 1, so every rule has consistent
    pixels to keep whatever the weights."""

    def __init__(self, depths):
        super().__init__()
        self.depths = depths                   # in the order the scan yields its views
        self.calls = 0

    def forward(self, imgs, pm, dmin, dint):
        d = self.depths[self.calls % len(self.depths)].to(imgs.device)
        self.calls += 1
        H, W = d.shape
        return {"depth_0": d[None], "confidence_2": torch.ones(1, H // 4, W // 4, device=imgs.device)}


def _plane_depths(scan, Z0):
    depths = []
    for ref in [m[0] for m in scan.metas]:
        P = scan.proj_mats[ref][0].numpy().astype(np.float64)
        W, H = scan.img_wh
        yy, xx = np.mgrid[:H, :W].astype(np.float64)
        Minv = np.linalg.inv(P[:3, :3])
        ray = np.einsum("ij,hwj->hwi", Minv, np.stack([xx, yy, np.ones_like(xx)], -1))
        off = Minv @ P[:3, 3]
        depths.append(torch.from_numpy(((Z0 + off[2]) / ray[..., 2]).astype(np.float32)))
    return depths


def test_eval_pipeline_dynamic_end_to_end(tmp_path, monkeypatch, capsys):
    from casmvsnet_pl_b200.models import mvsnet
    root = tmp_path / "tnt"
    synth_scenes.make_tanks(str(root), "intermediate", "Horse", n_views=6, image_wh=(200, 120), seed=3)
    wh, n_views = (128, 96), 5
    scan = ep.TanksTestScan(str(root), "intermediate", "Horse", wh, n_views)
    depths = _plane_depths(scan, 3.0)
    monkeypatch.setattr(mvsnet, "CascadeMVSNet", lambda **kw: _PlaneModel(depths))
    common = ["--dataset_name", "tanks", "--split", "intermediate", "--scan", "Horse",
              "--root_dir", str(root), "--img_wh", str(wh[0]), str(wh[1]), "--n_views", str(n_views)]
    ep.main(common + ["--fusion", "dynamic", "--out", str(tmp_path / "dyn")])
    ep.main(common + ["--fusion", "dynamic", "--mesh", "--out", str(tmp_path / "dyn_mesh")])
    ep.main(common + ["--out", str(tmp_path / "plain")])
    ep.main(common + ["--fusion", "reference", "--out", str(tmp_path / "ref")])
    log = capsys.readouterr().out
    ply = lambda d: (tmp_path / d / "points" / "Horse.ply").read_bytes()      # noqa: E731
    n = len(io.read_ply(tmp_path / "dyn" / "points" / "Horse.ply"))
    assert n > 1000 and f"Horse: dynamic fusion kept {n} points" in log
    assert ply("dyn") == ply("dyn_mesh")
    v, _, f = io.read_mesh_ply(tmp_path / "dyn_mesh" / "mesh" / "Horse.ply")
    assert len(v) > 0 and len(f) > 0
    # --fusion reference is the run without the flag, byte for byte; neither logs a rule
    assert ply("plain") == ply("ref") and "reference fusion kept" not in log
    # the dynamic cloud is its own: the plain run keeps only pixels 4 of the 4 sources agree on
    assert len(io.read_ply(tmp_path / "plain" / "points" / "Horse.ply")) <= n
