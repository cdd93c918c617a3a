"""utils.coords' neighbour searches without a GPU: the host restatement (oracle/coords_ref.py)
reproduces the reference's outputs stored in tests/golden/coords_ref.npz; argument errors are
raised before any device work; the public signatures are the reference's; ensemble_locate uses the
one DBSCAN of the package."""
import inspect
import os

import numpy as np
import pytest

import coords_cases as cc
import make_golden_coords as mg
from atomai_b200 import utils
from atomai_b200.predictors import epredictor
from atomai_b200.utils import coords
from oracle import coords_ref

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


@pytest.mark.parametrize("tag", ["movie", "single"])
@pytest.mark.parametrize("nn", [1, 2, 6])
@pytest.mark.parametrize("ub", [None, 9.0, 12.0])
def test_oracle_nn_distances(tag, nn, ub):
    d, p = coords_ref.get_nn_distances(mg.nn_cases()[tag], nn, ub)
    assert_list(d, f"nn/{tag}_{nn}_{ub}/d")
    assert_list(p, f"nn/{tag}_{nn}_{ub}/p")


def test_oracle_compare_and_clusters():
    c1, c2 = mg.compare_case()
    for got, k in zip(coords_ref.compare_coordinates(c1, c2, 3.0), ("c1", "c2", "d")):
        np.testing.assert_array_equal(got, GOLD[f"compare/{k}"])
    mv = cc.movie(10, 10, 7)
    m, s, cl = coords_ref.find_coord_clusters({0: mv[0]}, mv, 3)
    np.testing.assert_array_equal(m, GOLD["fcc/mean"])
    np.testing.assert_array_equal(s, GOLD["fcc/std"])
    assert_list(cl, "fcc/rows")


@pytest.mark.parametrize("tag", ["noise", "movie"])
def test_oracle_dbscan(tag):
    fr, eps, ms = mg.dbscan_cases()[tag]
    cl, m, v = coords_ref.cluster_coord(fr, eps, ms)
    assert_list(cl, f"dbscan_{tag}/rows")
    np.testing.assert_array_equal(m, GOLD[f"dbscan_{tag}/mean"])
    np.testing.assert_array_equal(v, GOLD[f"dbscan_{tag}/var"])


def test_dbscan_case_has_noise_and_shared_border_points():
    rows, eps, ms = cc.dbscan_points(0)
    labels = coords_ref.dbscan(rows[:, :2], eps, ms)
    assert (labels == -1).any()
    qi, pj, _ = coords_ref.pairs_within(rows[:, :2], rows[:, :2], eps, True)
    core = np.bincount(qi, minlength=len(rows)) >= ms
    shared = 0
    for i in np.flatnonzero(~core & (labels >= 0)):
        shared += len(set(labels[pj[(qi == i) & core[pj]]])) > 1
    assert shared == 2


@pytest.mark.parametrize("key", list(mg.traj_cases()))
def test_oracle_trajectories(key):
    img, fr, r = mg.traj_cases()[key]
    t = coords_ref.all_trajectories(img, fr, r, 2, 3)
    tag = f"traj_{key[0]}_{key[1]}"
    for got, k in zip(t, ("flow", "frames", "crops")):
        assert_list(got, f"{tag}/{k}")
    if key[0] % 2:
        assert t[0] == []


def test_exports_and_one_dbscan():
    for name in ("get_nn_distances", "map_bonds", "compare_coordinates", "find_coord_clusters",
                 "cluster_coord", "subimg_trajectories"):
        assert getattr(utils, name) is getattr(coords, name)
    assert epredictor.cluster_coord is coords.cluster_coord
    assert "sklearn" not in inspect.getsource(epredictor)


def test_signatures_equal_the_reference():
    ref = {
        "get_nn_distances": "(coordinates, nn=2, upper_bound=None)",
        "map_bonds": "(coordinates, nn=2, upper_bound=None, distance_ideal=None, "
                     "plot_results=True, **kwargs)",
        "compare_coordinates": "(coordinates1, coordinates2, d_max, plot_results=False, **kwargs)",
        "find_coord_clusters": "(coord_class_dict_1, coord_class_dict_2, rmax)",
        "cluster_coord": "(coord_class_dict, eps, min_samples=10)",
        "subimg_trajectories": "(imgdata, coord_class_dict, window_size, min_length=0, rmax=10)",
    }
    for name, sig in ref.items():
        s = inspect.signature(getattr(coords, name))
        plain = s.replace(parameters=[p.replace(annotation=p.empty) for p in s.parameters.values()],
                          return_annotation=s.empty)
        assert str(plain) == sig, name
    t = coords.subimg_trajectories
    assert str(inspect.signature(t.get_trajectory).replace(
        parameters=[p.replace(annotation=p.empty)
                    for p in inspect.signature(t.get_trajectory).parameters.values()],
        return_annotation=inspect.Signature.empty)) == "(self, img, start_coord)"


def _no_device(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("device touched before the argument checks")
    monkeypatch.setattr(coords, "_nn_device", fail)
    monkeypatch.setattr(coords.torch.cuda, "mem_get_info", fail)


def test_argument_errors_before_device_work(monkeypatch):
    _no_device(monkeypatch)
    c = cc.lattice(5, 0)
    for nn in (0, 32, 2.0, True):
        with pytest.raises(ValueError, match="32"):
            coords.get_nn_distances(c, nn)
    bad = c.copy()
    bad[3, 1] = np.nan
    with pytest.raises(ValueError, match="finite"):
        coords.get_nn_distances({0: c, 1: bad})
    with pytest.raises(ValueError, match="finite"):
        coords.compare_coordinates(c, bad, 3.0)
    with pytest.raises(ValueError, match="columns"):
        coords.compare_coordinates(c, c[:, :2], 3.0)
    with pytest.raises(AssertionError, match="expdata"):
        coords.compare_coordinates(c, c, 3.0, plot_results=True)
    with pytest.raises(ValueError, match="finite"):
        coords.find_coord_clusters({0: c}, {0: bad}, 3)
    with pytest.raises(ValueError, match="finite"):
        coords.cluster_coord({0: bad}, 1.0)
    for eps in (0, -1.0, np.inf):
        with pytest.raises(ValueError, match="eps"):
            coords.cluster_coord({0: c}, eps)
    with pytest.raises(ValueError, match="min_samples"):
        coords.cluster_coord({0: c}, 1.0, 0)
    with pytest.raises(ValueError, match="0 sample"):
        coords.cluster_coord({0: c[:0]}, 1.0)
    img = cc.images(2, 32, 32, 0)
    with pytest.raises(ValueError, match="imgdata"):
        coords.subimg_trajectories(img[0], {0: c}, 8).get_all_trajectories()
    with pytest.raises(ValueError, match="finite"):
        coords.subimg_trajectories(img, {0: c, 1: bad}, 8).get_all_trajectories()
    with pytest.raises(ValueError, match="window_size"):
        coords.subimg_trajectories(img, {0: c}, 8.0).get_all_trajectories()


def test_oracle_knn_tie_rule():
    p = np.array([[0.0, 0], [1, 0], [2, 0], [0.5, 0]])
    i, d = coords_ref.knn(np.array([[0.5, 0.0]]), p[:3], 2)
    assert i.tolist() == [[0, 1]] and d.tolist() == [[0.5, 0.5]]
