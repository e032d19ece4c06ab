"""COLMAP scene conversion on the GPU: casmvs_view_scores_fwd against the float64 oracle, its
determinism, the source lists, and eval_pipeline --dataset_name colmap end to end on the
synthetic capture of synth_scenes.make_colmap."""
import os

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import _lib, colmap, io as cio, synth_scenes
from casmvsnet_pl_b200 import eval_pipeline as ep
from oracle import view_select_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _within_bound(got, want):
    err = np.abs(got - want) - 1e-12 * (1 + want)
    return float(err.max()), bool((err <= 0).all())


@pytest.mark.parametrize("n_img,n_pts,seed", [(2, 50, 0), (17, 800, 1), (60, 4000, 2)])
def test_scores_match_oracle_on_ragged_tracks(n_img, n_pts, seed):
    c, xyz, ptr, img = synth_scenes.sparse_tracks(n_img, n_pts, (1, min(40, n_img)), seed)
    got = colmap.view_scores(c, xyz, ptr, img, DEV).cpu().numpy()
    # the loop restatement at the small sizes, the vectorised one (equal to it) at the largest
    want = (O.view_scores if n_pts <= 800 else O.view_scores_vec)(c, xyz, ptr, img, n_img)
    worst, ok = _within_bound(got, want)
    assert ok, worst
    assert np.array_equal(got, got.T) and not np.diag(got).any()


def test_scores_match_oracle_on_a_tanks_sized_model():
    c, xyz, ptr, img = synth_scenes.sparse_tracks(300, 500_000, (3, 11), seed=3)
    got = colmap.view_scores(c, xyz, ptr, img, DEV).cpu().numpy()
    want = O.view_scores_vec(c, xyz, ptr, img, 300)
    worst, ok = _within_bound(got, want)
    assert ok, worst
    assert (got > 0).sum() > 300 * 20


def test_scores_are_deterministic_across_buffers_and_chunks():
    c, xyz, ptr, img = synth_scenes.sparse_tracks(120, 60_000, (1, 30), seed=4)
    a = colmap.view_scores(c, xyz, ptr, img, DEV)
    pad = torch.empty(4097, dtype=torch.uint8, device=DEV)        # shifts the allocator's offsets
    b = colmap.view_scores(c, xyz, ptr, img, DEV)
    n_pairs = int((np.diff(ptr) * (np.diff(ptr) - 1) // 2).sum())
    chunked = colmap.view_scores(c, xyz, ptr, img, DEV, max_chunk_pairs=1024)
    assert n_pairs > 100 * 1024                                    # many chunks
    del pad
    assert torch.equal(a, b) and torch.equal(a, chunked)


def test_out_of_range_ids_contribute_nothing_and_empty_models_are_zero():
    c, xyz, ptr, img = synth_scenes.sparse_tracks(10, 200, (2, 6), seed=5)
    bad = img.copy()
    bad[::7] = 10                                                  # one past the last image
    got = colmap.view_scores(c, xyz, ptr, bad, DEV).cpu().numpy()
    worst, ok = _within_bound(got, O.view_scores(c, xyz, ptr, bad, 10))
    assert ok, worst
    n0 = _lib.launch_count()
    z = colmap.view_scores(c, xyz[:0], np.zeros(1, np.int64), img[:0], DEV)
    one = colmap.view_scores(c[:1], xyz, ptr, np.zeros_like(img), DEV)
    assert _lib.launch_count() == n0                               # no kernel for an empty model
    assert not z.any() and z.shape == (10, 10) and one.shape == (1, 1) and not one.any()


def test_source_lists_match_oracle_up_to_ties():
    c, xyz, ptr, img = synth_scenes.sparse_tracks(80, 20_000, (2, 12), seed=6)
    got = colmap.view_scores(c, xyz, ptr, img, DEV).cpu().numpy()
    want = O.view_scores_vec(c, xyz, ptr, img, 80)
    mine = [[j for j, _ in r] for r in colmap.select_sources(got)]
    ref = O.select_sources(want)
    near_ties = 0
    for v in range(80):
        row = want[v]
        for a, b in zip(mine[v], ref[v]):
            if a != b:          # only where the two candidates' scores lie within the bound
                assert abs(row[a] - row[b]) <= 2e-12 * (1 + max(row[a], row[b])), (v, a, b)
                near_ties += 1
        assert len(mine[v]) == len(ref[v])
    print(f"source lists: {near_ties} positions decided by a near tie")


def _model():
    from casmvsnet_pl_b200 import ABN, synth
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    torch.manual_seed(0)
    model = CascadeMVSNet(norm_act=ABN)
    synth.randomize_model_(model, 0)
    return model.eval().cuda()


def test_colmap_scan_end_to_end(tmp_path):
    depth = 3.0
    root = tmp_path / "capture"
    model = synth_scenes.make_colmap(str(root), n_views=8, image_wh=(160, 120), depth=depth,
                                     n_points=3000, seed=7, fmt="both")
    out = tmp_path / "out"
    ep.main(["--dataset_name", "colmap", "--root_dir", str(root), "--out", str(out),
             "--img_wh", "128", "96", "--n_views", "3", "--conf", "0", "--min_geo_consistent", "0",
             "--save_visual"])
    assert os.path.getsize(out / "points" / "capture.ply") > 0
    metas = cio.read_pair_file(str(out / "capture" / "pair.txt"))
    sc = colmap.load_scene(str(root))
    assert len(metas) == 8 and [r for r, _ in metas] == list(range(8))
    names = open(out / "capture" / "view_names.txt").read().split()
    assert names[1::2] == sc.names
    for ref, srcs in metas:
        assert len(srcs) == 7 and ref not in srcs
        K, E, dmin = cio.read_cam_file(str(out / "capture" / "cams" / f"{ref:08d}_cam.txt"))
        assert np.array_equal(E, sc.E[ref].astype(np.float32))
        assert np.array_equal(K, sc.K[ref].astype(np.float32))
        wh = tuple(int(x) for x in sc.wh[ref])
        assert torch.equal(cio.pyramid_proj_mats(K, E, 3, (128, 96), wh),
                           cio.pyramid_proj_mats(sc.K[ref].astype(np.float32),
                                                 sc.E[ref].astype(np.float32), 3, (128, 96), wh))
        interval = float(open(out / "capture" / "cams" / f"{ref:08d}_cam.txt").read().split()[-3])
        assert dmin <= depth <= dmin + 192 * interval, (ref, dmin, interval)
        assert os.path.isfile(out / "depth" / "capture" / f"depth_visual_{ref:04d}.jpg")
    assert len(model.images) == 8


def test_colmap_device_ingest_equals_host_route(tmp_path):
    root = tmp_path / "cap"
    synth_scenes.make_colmap(str(root), n_views=6, image_wh=(150, 100), n_points=2000, seed=8)
    net = _model()
    res = {}
    for host in (False, True):
        scan = ep.ColmapScan(str(root), img_wh=(128, 96), n_views=3, host_images=host)
        tag = "host" if host else "dev"
        xyz, rgb = ep.run_scan(net, scan, conf=0.0, min_geo_consistent=0,
                               depth_dir=str(tmp_path / tag / "depth"),
                               ply_path=str(tmp_path / tag / "s.ply"))
        d = tmp_path / tag / "depth" / "cap"
        res[tag] = ({f: cio.read_pfm(d / f)[0] for f in sorted(os.listdir(d))},
                    (tmp_path / tag / "s.ply").read_bytes(), len(xyz))
    (dm, dp, dn), (hm, hp, _) = res["dev"], res["host"]
    assert dm.keys() == hm.keys() and len(dm) == 12
    for k in dm:
        assert np.array_equal(dm[k], hm[k]), k
    assert dp == hp and dn > 0
