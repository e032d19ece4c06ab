"""Quadric edge-collapse decimation without a GPU: properties of the numpy restatement
(oracle/simplify_oracle.py) — planar quadrics, the link condition, the independence of one
round's collapses — the argument refusals of the CLI and of eval_pipeline, and a PLY round trip."""
import numpy as np
import pytest
from scipy import sparse

from casmvsnet_pl_b200 import eval_pipeline as ep
from casmvsnet_pl_b200 import io, mesh, simplify
from oracle import mesh_oracle as M
from oracle import simplify_oracle as S


def _state(verts, faces):
    P = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int32)
    frozen = S.frozen_flags(f, len(P))
    return S.round_state(P, S.vertex_quadrics(P, f, len(P)), f, frozen)


def test_a_planar_quadric_costs_nothing_in_its_plane():
    rng = np.random.default_rng(0)
    for tilt in (None, np.array([0.3, -0.2, 1.0])):
        v, f = S.grid_mesh(6)
        if tilt is not None:          # the plane z = 0.3 x - 0.2 y
            v[:, 2] = (0.3 * v[:, 0] - 0.2 * v[:, 1]).astype(np.float32)
        Q = S.vertex_quadrics(v, f, len(v))
        inner = 3 * 7 + 3                                 # an interior vertex: faces only
        xy = rng.uniform(-2, 2, (50, 2))
        z = np.zeros(50) if tilt is None else 0.3 * xy[:, 0] - 0.2 * xy[:, 1]
        c = S.qform(np.repeat(Q[inner][None], 50, 0), np.column_stack([xy, z]))
        assert np.abs(c).max() <= (0.0 if tilt is None else 1e-12)
        assert S.qform(Q[inner][None], np.array([[0.5, 0.5, 1.0]]))[0] > 0


def test_the_tetrahedron_edges_are_rejected():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)
    assert M.is_closed_oriented(f)
    st = _state(v, f)
    assert len(st["ek"]) == 6 and not st["valid"].any()


def test_the_link_condition_rejects_the_edge_that_would_pinch_a_strip():
    # a closed strip of 3 quads: bottom ring 0,1,2, top ring 3,4,5
    f = []
    for i in range(3):
        b0, b1, t0, t1 = i, (i + 1) % 3, 3 + i, 3 + (i + 1) % 3
        f += [[b0, b1, t1], [b0, t1, t0]]
    ang = np.arange(3) * 2 * np.pi / 3
    ring = np.column_stack([np.cos(ang), np.sin(ang), np.zeros(3)])
    v = np.concatenate([ring, ring + [0, 0, 1]]).astype(np.float32)
    f = np.array(f, np.int32)
    st = _state(v, f)
    adj = sparse.csr_matrix((np.ones(2 * len(st["a"])), (np.r_[st["a"], st["b"]], np.r_[st["b"], st["a"]])),
                            shape=(6, 6))
    common = np.asarray((adj @ adj)[st["a"], st["b"]]).ravel()
    bottom = (st["a"] < 3) & (st["b"] < 3)
    assert bottom.sum() == 3
    # a bottom edge has one face (one opposite vertex) but two common neighbours
    assert (st["cnt"][bottom] == 1).all() and (common[bottom] == 2).all()
    assert not st["valid"][bottom].any()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_no_two_collapses_of_a_round_touch_the_same_face(seed):
    rng = np.random.default_rng(seed)
    v, f = S.grid_mesh(14)
    v = v + rng.normal(0, 0.01, v.shape).astype(np.float32)
    v[:, 2] += rng.normal(0, 0.02, len(v)).astype(np.float32)
    s = S.sphere_mesh(16)
    verts = np.concatenate([v, s[0] + np.float32(3)])
    faces = np.concatenate([f, s[2] + len(v)])
    trace = []
    V, C, F, st = S.simplify(verts, np.zeros_like(verts, np.uint8), faces, len(faces) // 10,
                             trace=trace)
    assert st["rounds"] == len(trace) >= 3 and len(F) <= len(faces) // 10
    faces_now = S.prepare(verts, np.zeros_like(verts, np.uint8), faces)[2]
    for t in trace:
        fan = [set() for _ in range(len(verts))]        # faces at every vertex
        for i, x in enumerate(faces_now):
            for u in x:
                fan[u].add(i)
        seen = {}
        for e in np.nonzero(t["sel"])[0]:
            a, b = int(t["a"][e]), int(t["b"][e])
            for i in fan[a] | fan[b]:                     # every face the collapse rewrites
                assert i not in seen, f"collapses {seen[i]} and {(a, b)} both touch face {i}"
                seen[i] = (a, b)
        # the key-ordered prefix is a subset of the selection; replay it to follow the mesh
        P = np.zeros((len(verts), 3), np.float32)
        faces_now = S.collapse(P, np.zeros((len(verts), 3), np.uint8), np.zeros((len(verts), 10)),
                               faces_now, t, t["idx"])


def test_the_oracle_keeps_a_closed_sphere_closed():
    v, c, f = S.sphere_mesh(24)
    V, C, F, st = S.simplify(v, c, f, 200)
    assert 199 <= len(F) <= 200 and st["stop"] == "target"
    assert M.is_closed_oriented(F) and M.euler_characteristic(len(V), F) == 2
    assert M.signed_volume(V, F) > 0


def test_cli_arguments_are_refused():
    base = ["--ply", "in.ply", "--out", "out.ply"]
    for bad in ([], ["--faces", "10", "--ratio", "0.5"], ["--faces", "0"], ["--ratio", "0"],
                ["--ratio", "1.5"], ["--ratio", "nan"], ["--faces", "10", "--max_error", "-1"],
                ["--faces", "10", "--max_error", "inf"]):
        with pytest.raises(SystemExit):
            simplify.parse_args(base + bad)
    a = simplify.parse_args(base + ["--ratio", "0.25", "--max_error", "0.5"])
    assert a.ratio == 0.25 and a.faces is None and a.max_error == 0.5


def test_simplify_mesh_refuses_bad_targets_and_errors_before_any_gpu_work():
    v, f = S.grid_mesh(2)
    for kw, msg in ((dict(target_faces=0), "target_faces"), (dict(target_faces=2.5), "target_faces"),
                    (dict(target_faces=4, max_error=-1.0), "max_error"),
                    (dict(target_faces=4, max_error=float("nan")), "max_error")):
        with pytest.raises(ValueError, match=msg):
            simplify.simplify_mesh(v, np.zeros_like(v, np.uint8), f, **kw)


def test_eval_pipeline_mesh_faces_flag_is_checked():
    base = ["--dataset_name", "colmap", "--root_dir", "x"]
    for bad in (["--mesh_faces", "100"], ["--mesh", "--mesh_faces", "0"]):
        with pytest.raises(SystemExit):
            ep.parse_args(base + bad)
    assert ep.parse_args(base + ["--mesh", "--mesh_faces", "100"]).mesh_faces == 100
    assert ep.parse_args(base + ["--mesh"]).mesh_faces is None


def test_a_simplified_mesh_survives_a_ply_round_trip(tmp_path):
    v, c, f = S.sphere_mesh(16)
    V, C, F, _ = S.simplify(v, c, f, 100)
    mesh.write_mesh_ply(tmp_path / "m.ply", V, C, F)
    v2, c2, f2 = io.read_mesh_ply(tmp_path / "m.ply")
    assert np.array_equal(v2, V) and np.array_equal(c2, C) and np.array_equal(f2, F)
    assert f2.dtype == np.int32 and c2.dtype == np.uint8
