"""Statistical outlier removal without a GPU: the float64 oracle against brute force, the rule's
behaviour on known clouds, the refusals that need no device, the PLY writer and the
eval_pipeline flags."""
import math

import numpy as np
import pytest
import torch

from casmvsnet_pl_b200 import cloud_filter, eval_pipeline, fusion, io
from oracle import cloud_filter_oracle as O


def _tied_cloud(seed, n=400):
    """Random points snapped to a coarse float grid (mass ties) with exact duplicates."""
    rng = np.random.default_rng(seed)
    p = np.round(rng.uniform(-3, 3, (n, 3)) * 4) / 4
    p[rng.choice(n, n // 5, replace=False)] = p[rng.choice(n, n // 5, replace=False)]
    return p.astype(np.float32)


@pytest.mark.parametrize("k", [1, 2, 7, 20, 64])
@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_matches_brute_force_with_ties_and_duplicates(k, seed):
    rng = np.random.default_rng(seed)
    for xyz in (rng.normal(size=(300, 3)).astype(np.float32) * 1e3, _tied_cloud(seed)):
        got = O.mean_distance(xyz, k)
        want = O.brute_mean_distance(xyz, k)
        assert np.array_equal(got, want)


def test_oracle_counts_duplicates_but_not_the_point_itself():
    xyz = np.array([[0, 0, 0], [0, 0, 0], [3, 0, 0], [0, 4, 0]], np.float32)
    assert O.mean_distance(xyz, 1).tolist() == [0.0, 0.0, 3.0, 4.0]
    assert O.mean_distance(xyz, 2).tolist() == [1.5, 1.5, 3.0, 4.0]
    assert O.mean_distance(xyz, 3).tolist() == [7 / 3, 7 / 3, 11 / 3, 13 / 3]


def test_statistics_sum_in_chunks_in_order():
    rng = np.random.default_rng(3)
    m = rng.uniform(0, 1, 5000) ** 7
    mu, sigma, thr, chunks = O.statistics(m, 2.0)
    assert chunks.shape == (2, 5)
    s = 0.0
    for c in range(5):
        cs = 0.0
        for v in m[c * 1024:(c + 1) * 1024].tolist():
            cs = cs + v
        assert cs == chunks[0, c]
        s = s + cs
    assert mu == s / len(m)
    assert sigma == pytest.approx(float(np.std(m, ddof=1)), rel=1e-12)
    assert thr == mu + 2.0 * sigma


def noisy_sphere(n, outliers, seed):
    """n points on the unit sphere with 1 % radial noise and `outliers` points 1.5..3 radii out."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = d * (1 + 0.01 * rng.normal(size=(n, 1)))
    o = rng.normal(size=(outliers, 3))
    o *= rng.uniform(1.5, 3.0, (outliers, 1)) / np.linalg.norm(o, axis=1, keepdims=True)
    return np.concatenate([p, o]).astype(np.float32)


def test_far_outliers_go_and_the_sphere_stays():
    xyz = noisy_sphere(20000, 200, 0)
    keep, m, mu, sigma, thr = O.remove_statistical_outliers(xyz, 20, 2.0)
    assert not keep[20000:].any()
    assert keep[:20000].mean() > 0.97


@pytest.mark.parametrize("k", [1, 2, 3])
def test_a_regular_lattice_keeps_every_point(k):
    g = np.arange(8, dtype=np.float32)
    xyz = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    keep, m, mu, sigma, thr = O.remove_statistical_outliers(xyz, k, 2.0)
    assert sigma == 0.0 and (m == 1.0).all() and keep.all()


@pytest.mark.parametrize("k, message", [(0, "got 0"), (65, "got 65"), (2.5, "got 2.5"),
                                        (True, "got True")])
def test_bad_k_is_refused_with_its_value(k, message):
    with pytest.raises(ValueError, match=f"k must be an integer in 1..64, {message}"):
        cloud_filter.remove_statistical_outliers(torch.zeros(100, 3), k=k)


@pytest.mark.parametrize("r", [0.0, -1.0, math.inf, math.nan, "2"])
def test_bad_std_ratio_is_refused_with_its_value(r):
    with pytest.raises(ValueError, match=f"std_ratio must be a finite number > 0, got {r!r}"):
        cloud_filter.remove_statistical_outliers(torch.zeros(100, 3), std_ratio=r)


def test_bad_clouds_are_refused_with_their_values():
    with pytest.raises(ValueError, match=r"a cloud of 20 points cannot be filtered with k = 20"):
        cloud_filter.remove_statistical_outliers(torch.zeros(20, 3))
    with pytest.raises(ValueError, match=r"a cloud of 4 points .* k = 4"):
        cloud_filter.mean_neighbour_distance(torch.zeros(4, 3), k=4)
    with pytest.raises(ValueError, match=r"shape \(N, 3\), got \(30, 2\)"):
        cloud_filter.remove_statistical_outliers(torch.zeros(30, 2))
    with pytest.raises(ValueError, match=r"got ndarray"):
        cloud_filter.remove_statistical_outliers(np.zeros((30, 3), np.float32))
    with pytest.raises(ValueError, match=r"got torch.float32 on cpu"):
        cloud_filter.remove_statistical_outliers(torch.zeros(30, 3))
    with pytest.raises(ValueError, match=r"got torch.float64 on cpu"):
        cloud_filter.remove_statistical_outliers(torch.zeros(30, 3, dtype=torch.float64))


def test_ply_writer_round_trips_every_property(tmp_path):
    rng = np.random.default_rng(0)
    dt = [("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
          ("red", "u1"), ("green", "u1"), ("blue", "u1"), ("id", "<i4"), ("w", "<f8")]
    v = np.zeros(50, dtype=dt)
    for name, t in dt:
        v[name] = rng.integers(0, 200, 50) if t[-2] in "ui" else rng.normal(size=50)
    cloud_filter.write_vertices(tmp_path / "v.ply", v)
    back = io.read_ply(tmp_path / "v.ply")
    assert back.dtype == np.dtype(dt) and back.tobytes() == v.tobytes()
    cloud_filter.write_vertices(tmp_path / "e.ply", v[:0])
    assert len(io.read_ply(tmp_path / "e.ply")) == 0


def test_ply_writer_writes_fusions_bytes_for_xyz_rgb(tmp_path):
    rng = np.random.default_rng(1)
    xyz = rng.normal(size=(40, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (40, 3)).astype(np.uint8)
    fusion.write_ply(tmp_path / "f.ply", xyz, rgb)
    cloud_filter.write_vertices(tmp_path / "c.ply", io.read_ply(tmp_path / "f.ply"))
    assert (tmp_path / "c.ply").read_bytes() == (tmp_path / "f.ply").read_bytes()


def test_outlier_flags_need_the_switch():
    base = ["--root_dir", "x"]
    for extra in (["--outlier_neighbours", "10"], ["--outlier_std", "1.5"]):
        with pytest.raises(SystemExit):
            eval_pipeline.parse_args(base + extra)
    for extra in (["--outlier_neighbours", "0"], ["--outlier_neighbours", "65"],
                  ["--outlier_std", "0"], ["--outlier_std", "nan"]):
        with pytest.raises(SystemExit):
            eval_pipeline.parse_args(base + ["--remove_outliers"] + extra)
    a = eval_pipeline.parse_args(base)
    assert not a.remove_outliers and eval_pipeline._outlier_options(a) is None
    a = eval_pipeline.parse_args(base + ["--remove_outliers"])
    assert eval_pipeline._outlier_options(a) == {}
    a = eval_pipeline.parse_args(base + ["--remove_outliers", "--outlier_neighbours", "8",
                                         "--outlier_std", "1.5"])
    assert eval_pipeline._outlier_options(a) == dict(k=8, std_ratio=1.5)
