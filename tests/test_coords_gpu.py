"""utils.coords' neighbour searches on the GPU: bit-identical to the reference's outputs
(tests/golden/coords_ref.npz); 10⁵-point and 100-frame random cases against the host restatement
(oracle/coords_ref.py), DBSCAN labels included; the tie rule on an integer lattice; repeatability;
ensemble_locate; empty frames and frames with too few atoms."""
import os

import numpy as np
import pytest

import coords_cases as cc
import make_golden_coords as mg
from atomai_b200.utils import coords
from oracle import coords_ref

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("cuda")]

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "coords_ref.npz"))


def split(key):
    flat, lens = GOLD[f"{key}/flat"], GOLD[f"{key}/len"]
    return np.split(flat, np.cumsum(lens)[:-1]) if len(lens) else []


def assert_list(got, key):
    ref = split(key)
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        a = np.asarray(a)
        np.testing.assert_array_equal(a.reshape(len(a), int(np.prod(a.shape[1:]))), b)


def assert_same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape and x.dtype == y.dtype
        np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize("ub", [None, 9.0, 12.0])
@pytest.mark.parametrize("nn", [1, 2, 6])
@pytest.mark.parametrize("tag", ["movie", "single"])
def test_nn_distances_equal_reference(tag, nn, ub):
    d, p = coords.get_nn_distances(mg.nn_cases()[tag], nn, ub)
    assert_list(d, f"nn/{tag}_{nn}_{ub}/d")
    assert_list(p, f"nn/{tag}_{nn}_{ub}/p")


def test_map_bonds_equal_reference():
    with pytest.warns(UserWarning, match="plot skipped") if _no_matplotlib() else _null():
        got = coords.map_bonds(cc.movie(5, 12, 3, drop=0.1), 4, None, plot_results=False)
    np.testing.assert_array_equal(got, GOLD["bonds"])


def _no_matplotlib():
    try:
        import matplotlib  # noqa: F401
        return False
    except ImportError:
        return True


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def test_compare_and_clusters_equal_reference():
    c1, c2 = mg.compare_case()
    for got, k in zip(coords.compare_coordinates(c1, c2, 3.0), ("c1", "c2", "d")):
        np.testing.assert_array_equal(got, GOLD[f"compare/{k}"])
    mv = cc.movie(10, 10, 7)
    m, s, cl = coords.find_coord_clusters({0: mv[0]}, mv, 3)
    np.testing.assert_array_equal(m, GOLD["fcc/mean"])
    np.testing.assert_array_equal(s, GOLD["fcc/std"])
    assert_list(cl, "fcc/rows")


@pytest.mark.parametrize("tag", ["noise", "movie"])
def test_cluster_coord_equal_reference(tag):
    fr, eps, ms = mg.dbscan_cases()[tag]
    cl, m, v = coords.cluster_coord(fr, eps, ms)
    assert isinstance(cl, list)
    assert_list(cl, f"dbscan_{tag}/rows")
    np.testing.assert_array_equal(m, GOLD[f"dbscan_{tag}/mean"])
    np.testing.assert_array_equal(v, GOLD[f"dbscan_{tag}/var"])


@pytest.mark.parametrize("key", list(mg.traj_cases()))
def test_trajectories_equal_reference(key):
    img, fr, r = mg.traj_cases()[key]
    t = coords.subimg_trajectories(img, fr, r, 2, 3).get_all_trajectories()
    tag = f"traj_{key[0]}_{key[1]}"
    for got, k in zip(t, ("flow", "frames", "crops")):
        assert_list(got, f"{tag}/{k}")
    for c in t[2]:
        assert c.dtype == img.dtype
    ref = coords_ref.trajectory(img, fr, r, 3, fr[0][5, :2])
    assert_same(coords.subimg_trajectories(img, fr, r, 2, 3).get_trajectory(None, fr[0][5, :2]), ref)


def test_large_random_cases_equal_oracle():
    rng = np.random.default_rng(21)
    # 100 frames of ~1000 atoms (random points, some frames tiny or empty)
    mv = {}
    for f in range(100):
        n = [1000, 0, 3, 1][f] if f < 4 else int(rng.integers(800, 1200))
        mv[f] = np.concatenate([rng.uniform(0, 256, (n, 2)), rng.integers(0, 3, (n, 1))], 1)
    for nn, ub in ((1, 20.0), (4, None), (6, 10.0), (31, None)):
        got, ref = coords.get_nn_distances(mv, nn, ub), coords_ref.get_nn_distances(mv, nn, ub)
        assert_same(got[0], ref[0])
        assert_same(got[1], ref[1])
    # 10⁵ points
    big = np.concatenate([rng.uniform(0, 1000, (100000, 2)), rng.integers(0, 3, (100000, 1))], 1)
    c2 = big[rng.permutation(len(big))[:60000]].copy()
    c2[:, :2] += rng.normal(0, 1.0, (len(c2), 2))
    assert_same(coords.compare_coordinates(big, c2, 2.5), coords_ref.compare_coordinates(big, c2, 2.5))
    fr = cc.as_frames(big, 7)
    got, ref = coords.cluster_coord(fr, 2.0, 5), coords_ref.cluster_coord(fr, 2.0, 5)
    assert len(got[0]) == len(ref[0]) > 100
    assert_same(got[0], ref[0])
    assert_same(got[1:], ref[1:])
    labels = coords.dbscan_labels(big[:, :2], 2.0, 5)
    np.testing.assert_array_equal(labels, coords_ref.dbscan(big[:, :2], 2.0, 5))
    q = {0: big[:2000]}
    g, r = coords.find_coord_clusters(q, fr, 6.0), coords_ref.find_coord_clusters(q, fr, 6.0)
    assert_same(g[2], r[2])
    assert_same(g[:2], r[:2])
    # walks over a 30-frame movie
    mvw = cc.movie(30, 20, 5, drift=0.8, drop=0.05)
    img = cc.images(30, 160, 160, 4, 2)
    got = coords.subimg_trajectories(img, mvw, 10, 5, 3.0).get_all_trajectories()
    ref = coords_ref.all_trajectories(img, mvw, 10, 5, 3.0)
    assert len(got[0]) > 100
    for a, b in zip(got, ref):
        assert_same(a, b)


def test_integer_lattice_ties_go_to_the_lower_index():
    ij = np.stack(np.meshgrid(np.arange(30), np.arange(30), indexing="ij"), -1).reshape(-1, 2)
    c = np.concatenate([ij.astype(np.float64), np.zeros((len(ij), 1))], 1)
    c = c[np.random.default_rng(0).permutation(len(c))]
    for nn in (4, 8, 12):
        d, p = coords.get_nn_distances(c, nn)
        rd, rp = coords_ref.get_nn_distances(c, nn)
        assert_same(d, rd)
        assert_same(p, rp)
    q = c.copy()
    q[:, :2] += 0.5                                  # four nearest at the same distance
    assert_same(coords.compare_coordinates(q, c, 1.0), coords_ref.compare_coordinates(q, c, 1.0))
    m = coords.find_coord_clusters({0: q}, {0: c}, 2.0)
    assert_same(m[2], coords_ref.find_coord_clusters({0: q}, {0: c}, 2.0)[2])
    got = coords.dbscan_labels(c[:, :2], 1.0, 5)     # pairs at exactly eps are neighbours
    np.testing.assert_array_equal(got, coords_ref.dbscan(c[:, :2], 1.0, 5))


def test_repeatable():
    rng = np.random.default_rng(2)
    pts = rng.uniform(0, 300, (50000, 2))
    a = [coords.dbscan_labels(pts, 1.5, 4) for _ in range(3)]
    assert all(np.array_equal(a[0], x) for x in a[1:])
    mv = cc.movie(20, 16, 1)
    b = [coords.get_nn_distances(mv, 6) for _ in range(2)]
    for x, y in zip(b[0][0], b[1][0]):
        assert np.array_equal(x, y)


def test_ensemble_locate_equals_oracle_dbscan():
    from atomai_b200.predictors import ensemble_locate
    from atomai_b200.predictors.predictor import Locator
    rng = np.random.default_rng(3)
    base = np.zeros((2, 64, 64, 2), np.float32)
    for i in range(2):
        for x, y in rng.uniform(4, 60, (25, 2)):
            base[i, int(x) - 1:int(x) + 2, int(y) - 1:int(y) + 2, 0] = 1   # atoms: class 0
    base[..., 1] = 1 - base[..., 0]                                         # background last
    ens = np.stack([np.roll(base, (k % 2, k // 2), (1, 2)) for k in range(5)])
    mean, var = ensemble_locate(ens, eps=1.5)
    for i in range(2):
        fr = {k: Locator(0.5).run(ens[k, i][None])[0] for k in range(5)}
        assert min(len(c) for c in fr.values()) > 10
        _, m, v = coords_ref.cluster_coord(fr, 1.5)
        np.testing.assert_array_equal(mean[i], m)
        np.testing.assert_array_equal(var[i], v)


def test_empty_and_small_frames():
    c = cc.lattice(6, 1)
    fr = {0: c, 1: c[:0], 2: c[:2], 3: c[:3]}
    d, p = coords.get_nn_distances(fr, 2)
    assert [len(x) for x in d] == [36, 0, 0, 3]
    assert d[1].shape == (0, 2) and p[1].shape == (0, 3, 3) and p[2].shape == (0, 3, 3)
    assert_same(d, coords_ref.get_nn_distances(fr, 2)[0])
    out = coords.compare_coordinates(c[:0], c, 3.0)
    assert out[0].shape == (0, 3) and out[2].shape == (0,)
    m, s, cl = coords.find_coord_clusters({0: c[:4]}, {0: c[:0]}, 3)
    assert [len(x) for x in cl] == [0] * 4
    img = cc.images(4, 48, 48, 0)
    t = coords.subimg_trajectories(img, fr, 8, 0, 3).get_all_trajectories()
    r = coords_ref.all_trajectories(img, fr, 8, 0, 3)
    for a, b in zip(t, r):
        assert_same(a, b)
