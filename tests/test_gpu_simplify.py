"""Quadric edge-collapse decimation on the GPU (simplify.py, csrc/simplify.cu): the whole
decimation and every kernel's first-round state bit for bit against the numpy restatement
(oracle/simplify_oracle.py), then the properties a user relies on — closed meshes stay closed,
flat grids stay flat with their corners, a cube keeps its edges and corners, fidelity against a
serial greedy decimation, byte reproducibility, and eval_pipeline --mesh_faces end to end."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, io, mesh, simplify, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import mesh_oracle as M
from oracle import simplify_oracle as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _host(t):
    return t.cpu().numpy()


def _plane_scene():
    views = synth_scenes.sphere_scene(12, (240, 180), seed=3, device=DEV)
    v, c, f, _ = mesh.mesh_views([x["points"] for x in views], [x["depth"] for x in views],
                                 [x["image"] for x in views], [x["P"] for x in views], voxel=0.05)
    return _host(v), _host(c), _host(f)


def _degenerate():
    v, f = S.grid_mesh(12)
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
    return (np.concatenate([v, extra_v]), np.zeros((n + 4, 3), np.uint8) + 7,
            np.concatenate([f, extra_f]))


MESHES = {
    "plane_scene": (_plane_scene, 0.10),
    "closed_sphere": (lambda: S.sphere_mesh(60), 0.02),
    "degenerate": (_degenerate, 0.10),
}


@pytest.mark.parametrize("name", list(MESHES))
def test_decimation_is_bit_identical_to_the_oracle(name):
    make, ratio = MESHES[name]
    v, c, f = make()
    c = np.asarray(c, np.uint8)
    if name == "plane_scene":
        assert 10_000 < len(f) < 150_000, len(f)
    target = max(1, round(ratio * len(f)))
    V, C, F, st = simplify.simplify_mesh(_cuda(v), _cuda(c), _cuda(f), target)
    Vo, Co, Fo, sto = S.simplify(v, c, f, target)
    assert st == sto
    assert np.array_equal(_host(V).view(np.uint32), Vo.view(np.uint32))
    assert np.array_equal(_host(C), Co) and np.array_equal(_host(F), Fo)
    if name == "degenerate":
        assert st["dropped_faces"] == 2 and st["frozen_vertices"] >= 3


@pytest.mark.parametrize("name", list(MESHES))
def test_first_round_kernels_match_the_oracle(name):
    make, ratio = MESHES[name]
    v, c, f = make()
    c = np.asarray(c, np.uint8)
    target = max(1, round(ratio * len(f)))
    P, C, fg, frozen, Q, dropped = simplify._prepare(_cuda(v), _cuda(c), _cuda(f).int())
    Po, Co, fo, frozen_o, Qo, dropped_o = S.prepare(v, c, f)
    assert dropped == dropped_o and np.array_equal(_host(fg), fo)
    assert np.array_equal(_host(frozen).astype(bool), frozen_o)
    assert np.array_equal(_host(Q).view(np.uint64), Qo.view(np.uint64))
    st = simplify._round_state(P, Q, fg, frozen)
    sto = S.round_state(Po, Qo, fo, frozen_o)
    assert np.array_equal(_host(st["ek"]), sto["ek"])
    assert np.array_equal(_host(st["deg"]), sto["deg"])
    assert np.array_equal(_host(st["bnd"]).astype(bool), sto["bnd"])
    assert np.array_equal(_host(st["v"]).view(np.uint32), sto["v"].view(np.uint32))
    assert np.array_equal(_host(st["cost"]).view(np.uint32), sto["cost"].view(np.uint32))
    assert np.array_equal(_host(st["valid0"]).astype(bool), sto["valid0"])
    assert np.array_equal(_host(st["key"]), sto["key"])
    sel, thr = simplify._select(st, fg, len(v))
    sel_o, thr_o = S.select(sto, fo, len(v))
    assert thr == thr_o and np.array_equal(_host(sel), sel_o) and sel_o.any()
    idx = simplify._budget(st, sel, len(fg), target)
    assert np.array_equal(_host(idx), S.budget(sto, sel_o, len(fo), target))


def test_a_closed_sphere_to_one_percent_stays_closed_and_outward():
    v, c, f = S.sphere_mesh(60)
    target = round(0.01 * len(f))
    V, C, F, st = simplify.simplify_mesh(_cuda(v), _cuda(c), _cuda(f), target)
    V, F = _host(V), _host(F)
    assert target - 1 <= len(F) <= target and st["stop"] == "target"
    assert M.is_closed_oriented(F) and M.euler_characteristic(len(V), F) == 2
    assert M.signed_volume(V, F) > 0


def test_a_flat_grid_stays_flat_and_keeps_its_corners():
    v, f = S.grid_mesh(100)
    V, C, F, st = simplify.simplify_mesh(_cuda(v), _cuda(np.zeros_like(v, np.uint8)), _cuda(f), 50)
    V = _host(V)
    assert len(F) <= 50 and st["stop"] == "target"
    assert np.abs(V[:, 2]).max() <= 1e-7
    for corner in ([0, 0], [1, 0], [0, 1], [1, 1]):
        assert np.abs(V[:, :2] - corner).max(1).min() <= 1e-6, corner


def test_a_cube_keeps_its_faces_edges_and_corners():
    v, f = S.cube_mesh(32)
    assert M.is_closed_oriented(f)
    V, C, F, st = simplify.simplify_mesh(_cuda(v), _cuda(np.zeros_like(v, np.uint8)), _cuda(f), 100)
    V, F = _host(V), _host(F)
    assert len(F) <= 100
    assert np.abs(np.abs(V).max(1) - 0.5).max() <= 1e-5          # on the cube's surface
    for s in np.array(np.meshgrid([-0.5, 0.5], [-0.5, 0.5], [-0.5, 0.5])).reshape(3, -1).T:
        assert np.abs(V - s).max(1).min() <= 1e-5, s
    assert M.is_closed_oriented(F) and M.euler_characteristic(len(V), F) == 2


def test_fidelity_is_within_twice_the_serial_greedy_decimation():
    v, c, f = S.sphere_mesh(60)                                   # about 20 k faces
    V, C, F, st = simplify.simplify_mesh(_cuda(v), _cuda(c), _cuda(f), 1000)
    Vs, Cs, Fs = S.serial_simplify(v, c, f, 1000)
    err = np.abs(np.linalg.norm(_host(V).astype(np.float64), axis=1) - 1).mean()
    err_s = np.abs(np.linalg.norm(Vs.astype(np.float64), axis=1) - 1).mean()
    print(f"mean | |v| - 1 |: parallel {err:.4e}, serial {err_s:.4e} ({len(F)} / {len(Fs)} faces)")
    assert len(F) <= 1000 and len(Fs) <= 1000
    assert err <= 2 * err_s


def test_two_runs_write_the_same_bytes_and_the_cli_agrees(tmp_path):
    v, c, f = _plane_scene()
    out = []
    for i in range(2):
        V, C, F, _ = simplify.simplify_mesh(_cuda(v), _cuda(c), _cuda(f), len(f) // 20)
        mesh.write_mesh_ply(tmp_path / f"{i}.ply", V, C, F)
        out.append((tmp_path / f"{i}.ply").read_bytes())
    assert out[0] == out[1]
    mesh.write_mesh_ply(tmp_path / "in.ply", v, c, f)
    simplify.main(["--ply", str(tmp_path / "in.ply"), "--out", str(tmp_path / "cli.ply"),
                   "--faces", str(len(f) // 20)])
    assert (tmp_path / "cli.ply").read_bytes() == out[0]
    simplify.main(["--ply", str(tmp_path / "in.ply"), "--out", str(tmp_path / "r.ply"),
                   "--ratio", "0.05"])
    assert len(io.read_mesh_ply(tmp_path / "r.ply")[2]) <= max(1, round(0.05 * len(f)))


def test_bad_inputs_and_oversized_work_are_refused():
    v, f = S.grid_mesh(4)
    c = np.zeros_like(v, np.uint8)
    bad_v = v.copy()
    bad_v[3, 1] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        simplify.simplify_mesh(_cuda(bad_v), _cuda(c), _cuda(f), 4)
    bad_f = f.copy()
    bad_f[2, 0] = len(v)
    with pytest.raises(ValueError, match="outside"):
        simplify.simplify_mesh(_cuda(v), _cuda(c), _cuda(bad_f), 4)
    with pytest.raises(_lib.CasMVSError, match="needs .* bytes .* but 1000 bytes"):
        simplify.simplify_mesh(_cuda(v), _cuda(c), _cuda(f), 4, max_bytes=1000)


def test_max_error_stops_early_and_says_so():
    v, c, f = S.sphere_mesh(24)
    logs = []
    V, C, F, st = simplify.simplify_mesh(_cuda(v), _cuda(c), _cuda(f), 10, max_error=1e-7,
                                         log=logs.append)
    Vo, Co, Fo, sto = S.simplify(v, c, f, 10, max_error=1e-7)
    assert st == sto and st["stop"] == "max_error" and len(F) > 10
    assert np.array_equal(_host(F), Fo) and st["max_cost"] <= 1e-7
    assert any("above the target" in m for m in logs)


def _tree_bytes(d):
    return {os.path.relpath(os.path.join(r, n), d): open(os.path.join(r, n), "rb").read()
            for r, _, files in os.walk(d) for n in files}


@pytest.mark.parametrize("method", ["tsdf", "poisson"])
def test_eval_pipeline_mesh_faces_end_to_end(tmp_path, method):
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
    N = 300
    ep.main(common + ["--out", str(tmp_path / "none")])
    ep.main(common + meshing + ["--out", str(tmp_path / "full")])
    ep.main(common + meshing + ["--mesh_faces", str(N), "--out", str(tmp_path / "s1")])
    ep.main(common + meshing + ["--mesh_faces", str(N), "--out", str(tmp_path / "s2")])
    none, full = _tree_bytes(tmp_path / "none"), _tree_bytes(tmp_path / "full")
    s1, s2 = _tree_bytes(tmp_path / "s1"), _tree_bytes(tmp_path / "s2")
    mesh_file = os.path.join("mesh", "capture.ply")
    assert s1 == s2
    assert {k: v for k, v in s1.items() if k != mesh_file} == none
    assert s1[mesh_file] != full[mesh_file] or len(io.read_mesh_ply(tmp_path / "full" / mesh_file)[2]) <= N
    assert len(io.read_mesh_ply(tmp_path / "s1" / mesh_file)[2]) <= N
    simplify.main(["--ply", str(tmp_path / "full" / mesh_file), "--out", str(tmp_path / "cli.ply"),
                   "--faces", str(N)])
    assert (tmp_path / "cli.ply").read_bytes() == s1[mesh_file]
