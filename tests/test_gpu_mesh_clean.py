"""Mesh cleaning on the GPU (mesh_clean.py, csrc/mesh_clean.cu): every step and the whole call bit
for bit against the numpy restatement (oracle/mesh_clean_oracle.py) on a TSDF mesh, a Poisson mesh
of a cloud with outliers and a mesh with degenerate faces, a non-manifold edge and a bow tie; then
byte reproducibility, the command line, the refusals, floaters removed exactly, and
eval_pipeline --mesh_clean end to end."""
import os

import numpy as np
import pytest
import torch

import test_mesh_clean as C
from casmvsnet_pl_b200 import _lib, io, mesh, mesh_clean, poisson, simplify, synth_dtu, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import mesh_clean_oracle as O
from oracle import mesh_oracle as M
from oracle import simplify_oracle as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _host(t):
    return t.cpu().numpy()


def _tsdf_scene():
    views = synth_scenes.sphere_scene(12, (240, 180), seed=3, device=DEV)
    v, c, f, _ = mesh.mesh_views([x["points"] for x in views], [x["depth"] for x in views],
                                 [x["image"] for x in views], [x["P"] for x in views], voxel=0.05)
    return _host(v), _host(c), _host(f)


def _poisson_dtu():
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        p = synth_dtu.make_scene(d, n_stl=2000, n_data=40_000, seed=2, outlier_frac=0.02)
    cams = synth_dtu.CENTER + np.array([[0, 0, -500.0], [80, 0, -480], [-80, 40, -490]])
    rgb = np.random.default_rng(0).integers(0, 256, (len(p), 3)).astype(np.uint8)
    v, c, f, _ = poisson.poisson_mesh(_cuda(p.astype(np.float32)), _cuda(rgb), cam_centres=cams,
                                      depth=10, log=lambda m: None)
    return _host(v), _host(c), _host(f)


def _degenerate():
    v, f = C.grid_without(12, [(5, 5), (5, 6), (6, 5), (6, 6)])
    n = len(v)
    extra_v = np.array([[0.5, 0.5, 0.3], [1.3, 1.3, 0.0], [1.3, 1.1, 0.0], [1.1, 1.3, 0.1]],
                       np.float32)
    a, b = 3 * 13 + 3, 3 * 13 + 4                         # an interior edge of the grid
    corner = 12 * 13 + 12                                 # the grid corner (1, 1, 0)
    extra_f = np.array([[a, b, n],                        # third face on edge ab: non-manifold
                        [corner, n + 1, n + 2],           # a second fan at the corner: bow tie
                        [n + 1, n + 3, n + 2],
                        [5, 5, 6],                        # repeated index
                        [0, 1, 2]], np.int32)             # collinear: zero area
    v = np.concatenate([v, extra_v])
    return v, (np.arange(len(v) * 3) % 251).astype(np.uint8).reshape(-1, 3), np.concatenate([f, extra_f])


def _sphere_fans():
    v, c, f, _ = C.sphere_with_fans_removed(40)
    return v, c, f


MESHES = {
    "tsdf_scene": (_tsdf_scene, dict(max_hole=128)),
    "poisson_dtu": (_poisson_dtu, dict(max_hole=128)),
    "degenerate": (_degenerate, dict(min_ratio=0.0, max_hole=32)),
    "sphere_fans": (_sphere_fans, dict(max_hole=16)),
}


@pytest.fixture(scope="module", params=list(MESHES))
def case(request):
    make, kw = MESHES[request.param]
    v, c, f = make()
    return request.param, v, np.asarray(c, np.uint8), np.asarray(f, np.int32), kw


def test_every_step_is_bit_identical_to_the_oracle(case):
    name, v, c, f, kw = case
    trace = {}
    O.clean_mesh(v, c, f, trace=trace, **kw)
    P = _cuda(v)
    fg, dropped = mesh_clean.cleanup(P, _cuda(f))
    assert np.array_equal(_host(fg), trace["cleaned"])
    pc = mesh_clean.pieces(P, fg)
    po = trace["pieces"]
    assert np.array_equal(_host(pc["face_area"]).view(np.uint64), po["face_area"].view(np.uint64))
    assert np.array_equal(_host(pc["comp"]), po["comp"])
    assert np.array_equal(_host(pc["roots"]), po["roots"])
    assert np.array_equal(_host(pc["count"]), po["count"])
    assert np.array_equal(_host(pc["area"]).view(np.uint64), po["area"].view(np.uint64))
    assert np.array_equal(_host(pc["piece"]), po["piece"])
    kept = _cuda(trace["kept"])
    lp = mesh_clean.boundary_loops(kept, len(v))
    lo = trace["loops"]
    for k in ("edge_keys", "out_deg", "in_deg", "next", "next_face", "comp", "size", "open",
              "owners", "sizes"):
        assert np.array_equal(_host(lp[k]), lo[k]), k
    assert lp["not_simple"] == lo["not_simple"]
    small = lp["sizes"] <= kw["max_hole"]
    owners, sizes = lp["owners"][small], lp["sizes"][small]
    assert np.array_equal(_host(owners), trace["owners"])
    thr = mesh_clean.piece_threshold(pc["count"], kw.get("min_faces", 0), kw.get("min_ratio", 0.01))
    keep_face = (pc["count"] >= thr)[pc["piece"]]
    piece_area = pc["area"][pc["piece"][keep_face]]
    status, area, tris, _ = mesh_clean.fill_holes(P, lp, owners, sizes, piece_area)
    assert np.array_equal(_host(status), trace["status"])
    assert np.array_equal(_host(area).view(np.uint64), trace["area"].view(np.uint64))
    assert np.array_equal(_host(tris), trace["tris"])
    print(f"{name}: {len(f)} faces, {len(lo['owners'])} loops, sizes up to "
          f"{int(lo['sizes'].max()) if len(lo['sizes']) else 0}, status counts "
          f"{np.bincount(trace['status'], minlength=4).tolist()}")


def test_the_whole_call_is_bit_identical_to_the_oracle(case):
    name, v, c, f, kw = case
    V, Cc, F, st = mesh_clean.clean_mesh(_cuda(v), _cuda(c), _cuda(f), **kw)
    Vo, Co, Fo, sto = O.clean_mesh(v, c, f, **kw)
    assert st == sto
    assert np.array_equal(_host(V).view(np.uint32), Vo.view(np.uint32))
    assert np.array_equal(_host(Cc), Co) and np.array_equal(_host(F), Fo)
    print(name, st)
    if name == "degenerate":
        assert st["degenerate"] == 2 and st["holes_filled"] == 1 and st["loops_not_simple"] >= 1
    if name == "sphere_fans":
        assert st["holes_filled"] == 3
        assert M.is_closed_oriented(_host(F)) and M.euler_characteristic(len(V), _host(F)) == 2


def test_two_runs_write_the_same_bytes_and_the_cli_agrees(tmp_path):
    v, c, f = _tsdf_scene()
    out = []
    for i in range(2):
        V, Cc, F, _ = mesh_clean.clean_mesh(_cuda(v), _cuda(c), _cuda(f), min_ratio=0.02,
                                            max_hole=100)
        mesh.write_mesh_ply(tmp_path / f"{i}.ply", V, Cc, F)
        out.append((tmp_path / f"{i}.ply").read_bytes())
    assert out[0] == out[1]
    mesh.write_mesh_ply(tmp_path / "in.ply", v, c, f)
    mesh_clean.main(["--ply", str(tmp_path / "in.ply"), "--out", str(tmp_path / "cli.ply"),
                     "--min_ratio", "0.02", "--max_hole", "100"])
    assert (tmp_path / "cli.ply").read_bytes() == out[0]


def test_injected_floaters_are_removed_exactly():
    v, c, f = S.sphere_mesh(40)
    rng = np.random.default_rng(5)
    fv, fc, ff = [], [], []
    n = 0
    for k in range(6):
        sv, sc, sf = S.sphere_mesh(6)
        sv = (sv * 0.02 + rng.uniform(-2, 2, 3)).astype(np.float32)
        fv.append(sv), fc.append(sc), ff.append(sf + n)
        n += len(sv)
    tri = np.array([[3.0, 3, 3], [3.01, 3, 3], [3, 3.01, 3]], np.float32)
    fv.append(tri), fc.append(np.zeros((3, 3), np.uint8)), ff.append(np.array([[n, n + 1, n + 2]]))
    n += 3
    # floater vertices first, floater faces scattered among the sphere's
    verts = np.concatenate(fv + [v])
    cols = np.concatenate(fc + [c])
    floats = np.concatenate(ff)
    faces = f + n
    at = np.sort(rng.choice(len(faces) + 1, len(floats)))
    faces = np.insert(faces, at, floats, axis=0).astype(np.int32)
    V, Cc, F, st = mesh_clean.clean_mesh(_cuda(verts), _cuda(cols), _cuda(faces), min_ratio=0.05,
                                         max_hole=128)
    assert st["pieces_removed"] == 7 and st["faces_added"] == 0 and st["loops"] == 0
    assert np.array_equal(_host(V), v) and np.array_equal(_host(Cc), c)
    assert np.array_equal(_host(F), f)


def test_bad_inputs_empty_results_and_oversized_work_are_refused():
    v, f = S.grid_mesh(4)
    c = np.zeros_like(v, np.uint8)
    bad_v = v.copy()
    bad_v[3, 1] = np.inf
    with pytest.raises(ValueError, match="non-finite"):
        mesh_clean.clean_mesh(_cuda(bad_v), _cuda(c), _cuda(f))
    bad_f = f.copy()
    bad_f[2, 0] = len(v)
    with pytest.raises(ValueError, match="outside"):
        mesh_clean.clean_mesh(_cuda(v), _cuda(c), _cuda(bad_f))
    bad_f[2, 0] = -1
    with pytest.raises(ValueError, match="outside"):
        mesh_clean.clean_mesh(_cuda(v), _cuda(c), _cuda(bad_f))
    for bad_c in (c.astype(np.float32), c[:, :2], c[:-1]):
        with pytest.raises(ValueError, match="colours"):
            mesh_clean.clean_mesh(_cuda(v), _cuda(np.ascontiguousarray(bad_c)), _cuda(f))
    with pytest.raises(ValueError, match="no faces"):
        mesh_clean.clean_mesh(_cuda(v), _cuda(c), _cuda(np.zeros((0, 3), np.int32)))
    with pytest.raises(ValueError, match="every face is degenerate"):
        mesh_clean.clean_mesh(_cuda(v), _cuda(c), _cuda(np.array([[0, 0, 1], [0, 1, 2]], np.int32)))
    with pytest.raises(ValueError, match="exceeds the largest piece"):
        mesh_clean.clean_mesh(_cuda(v), _cuda(c), _cuda(f), min_faces=len(f) + 1)
    with pytest.raises(_lib.CasMVSError, match="needs .* bytes .* but 1000 bytes"):
        mesh_clean.clean_mesh(_cuda(v), _cuda(c), _cuda(f), max_bytes=1000)
    need = len(f) * mesh_clean.BYTES_PER_FACE + len(v) * mesh_clean.BYTES_PER_VERTEX
    mesh_clean.clean_mesh(_cuda(v), _cuda(c), _cuda(f), max_bytes=need)


def _tree_bytes(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


@pytest.mark.parametrize("method", ["tsdf", "poisson"])
def test_eval_pipeline_mesh_clean_end_to_end(tmp_path, method):
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
              "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0", "--ckpt", str(ckpt)]
    meshing = ["--mesh", "--mesh_method", method] + (["--poisson_depth", "7"] if method == "poisson" else [])
    cleaning = ["--mesh_clean", "--mesh_clean_ratio", "0.05", "--mesh_max_hole", "64"]
    N = 300
    ep.main(common + meshing + ["--out", str(tmp_path / "full")])
    ep.main(common + meshing + cleaning + ["--out", str(tmp_path / "c")])
    ep.main(common + meshing + cleaning + ["--mesh_faces", str(N), "--mesh_texture",
                                           "--out", str(tmp_path / "cst")])
    full, cl, cst = (_tree_bytes(tmp_path / d) for d in ("full", "c", "cst"))
    mesh_file = os.path.join("mesh", "capture.ply")
    assert {k: v for k, v in cl.items() if k != mesh_file} == \
        {k: v for k, v in full.items() if k != mesh_file}
    assert {k: v for k, v in cst.items() if not k.startswith("mesh")} == \
        {k: v for k, v in full.items() if not k.startswith("mesh")}
    mesh_clean.main(["--ply", str(tmp_path / "full" / mesh_file), "--out", str(tmp_path / "cli.ply"),
                     "--min_ratio", "0.05", "--max_hole", "64"])
    assert (tmp_path / "cli.ply").read_bytes() == cl[mesh_file]
    simplify.main(["--ply", str(tmp_path / "cli.ply"), "--out", str(tmp_path / "s.ply"),
                   "--faces", str(N)])
    assert (tmp_path / "s.ply").read_bytes() == cst[mesh_file]
    assert os.path.join("mesh", "capture.obj") in cst
    v_obj = sum(1 for line in cst[os.path.join("mesh", "capture.obj")].splitlines()
                if line.startswith(b"v "))
    assert v_obj == len(io.read_mesh_ply(tmp_path / "s.ply")[0])
