"""utils.graphx without a GPU: the host restatement (oracle/graph_ref.py) reproduces the reference's
outputs stored in tests/golden/graph_ref.npz; the covalent-radius table; argument errors raised
before any device work; the recursive single-node searches refused."""
import os

import numpy as np
import pytest

import graph_cases as gc
from atomai_b200 import utils
from atomai_b200.utils import graphx
from oracle import graph_ref

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "graph_ref.npz"))
CASES = {"single": gc.single, "z": gc.with_z, "multi": gc.multi}


def _sorted_rows(a):
    return a[np.lexsort(a.T[::-1])]


@pytest.mark.parametrize("tag", list(CASES))
def test_oracle_reproduces_reference(tag):
    c = CASES[tag]()
    exact = tag != "multi"      # multi-class neighbour lists are in k-d tree order in the reference
    for cyc in ([6], [5, 7], list(range(3, 10))):
        got = graph_ref.find_cycles(c, cyc, gc.MAP_DICT, gc.PX2ANG)
        ref = GOLD[f"{tag}/cycles_{''.join(map(str, cyc))}"]
        if exact:
            np.testing.assert_array_equal(got, ref)
        else:
            np.testing.assert_array_equal(_sorted_rows(got), _sorted_rows(ref))
    _, _, nb, rl = graph_ref.analyse(c, 9, gc.MAP_DICT, gc.PX2ANG)
    ids, lens = GOLD[f"{tag}/rings_9"], GOLD[f"{tag}/rings_9_len"]
    ref_rings = np.split(ids, np.cumsum(lens)[:-1])
    if exact:
        assert [list(r) for r in ref_rings] == rl
    else:
        assert sorted(tuple(sorted(r)) for r in ref_rings) == sorted(tuple(sorted(r)) for r in rl)
    if exact:
        cl = graph_ref.find_cycle_clusters(c, [5, 7], gc.MAP_DICT, gc.PX2ANG)
        np.testing.assert_array_equal(np.concatenate(cl), GOLD[f"{tag}/clusters_57"])
        np.testing.assert_array_equal([len(x) for x in cl], GOLD[f"{tag}/clusters_57_len"])
        np.testing.assert_array_equal(graph_ref.filter_subgraphs_(c, gc.MAP_DICT, gc.PX2ANG),
                                      GOLD[f"{tag}/filter"])


def test_oracle_frames():
    for k, c in gc.frames().items():
        np.testing.assert_array_equal(graph_ref.filter_subgraphs_(c, gc.MAP_DICT, gc.PX2ANG),
                                      GOLD[f"frames/{k}"])


def test_radii_table():
    pinned = {"H": 32, "B": 85, "C": 75, "N": 71, "O": 63, "P": 111, "S": 103, "Si": 116}
    for el, r in pinned.items():
        assert graphx.COVALENT_RADII[el] == r
        assert graph_ref.RADII[el] == r
    assert len(graphx.COVALENT_RADII) == 118
    assert graphx.get_interatomic_r(["C", "C"], 1.2) == 1.2 * ((75.0 + 75.0) / 100)
    assert graphx.get_interatomic_r(("C", "Si")) == (75.0 + 116.0) / 100
    with pytest.raises(ValueError, match="Xx"):
        graphx.get_interatomic_r(["C", "Xx"])


def test_exports():
    for name in ("Graph", "Node", "find_cycles", "find_cycle_clusters", "filter_subgraphs",
                 "filter_subgraphs_", "get_interatomic_r", "plot_graph"):
        assert getattr(utils, name) is getattr(graphx, name)


def _no_device(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("device touched before the argument checks")
    monkeypatch.setattr(graphx, "_device", fail)
    monkeypatch.setattr(graphx.torch.cuda, "mem_get_info", fail)


def test_argument_errors_before_device_work(monkeypatch):
    _no_device(monkeypatch)
    c = gc.single()[:50]
    with pytest.raises(ValueError, match="N, 3"):
        graphx.find_cycles(c[:, :2], [6], gc.MAP_DICT, gc.PX2ANG)
    with pytest.raises(ValueError, match="N, 3"):
        graphx.filter_subgraphs(np.zeros((4, 5)), gc.MAP_DICT, gc.PX2ANG)
    bad = c.copy()
    bad[3, 2] = 5
    with pytest.raises(KeyError):
        graphx.find_cycles(bad, [6], gc.MAP_DICT, gc.PX2ANG)
    with pytest.raises(KeyError):
        graphx.filter_subgraphs({0: c, 1: bad}, gc.MAP_DICT, gc.PX2ANG)
    with pytest.raises(ValueError, match="Qq"):
        graphx.find_cycle_clusters(c, [5, 7], {0: "Qq"}, gc.PX2ANG)
    for cyc in ([2], [33], [5, 7.0], 40, [True]):
        with pytest.raises(ValueError, match="32"):
            graphx.find_cycles(c, cyc, gc.MAP_DICT, gc.PX2ANG)
    G = graphx.Graph(c, gc.MAP_DICT)
    with pytest.raises(ValueError, match="32"):
        G.polycount(max_depth=None)
    with pytest.raises(ValueError, match="32"):
        G.polycount(max_depth=64)


def test_recursive_searches_refused():
    G = graphx.Graph(gc.single()[:10], gc.MAP_DICT)
    with pytest.raises(NotImplementedError, match="polycount"):
        G.find_rings(G.vertices[0])
    with pytest.raises(NotImplementedError, match="remove_filled_polygons"):
        G.shortest_path(G.vertices[0], G.vertices[1], 3)


def test_plot_graph_skips_without_matplotlib(monkeypatch):
    import builtins
    real = builtins.__import__

    def imp(name, *a, **k):
        if name.startswith("matplotlib"):
            raise ImportError(name)
        return real(name, *a, **k)
    monkeypatch.setattr(builtins, "__import__", imp)
    with pytest.warns(UserWarning, match="plot skipped"):
        graphx.plot_graph(None)


def _unpruned_rings(nbrs, max_depth):
    """the recursive search restated without pruning: from each root, every path over atoms above
    it of up to max_depth atoms; a path closes at an atom bonded to the root unless that atom was
    the first step of an earlier, finished branch of the same root"""
    out = []
    for root in range(len(nbrs)):
        path, spent = [root], set()

        def walk(v):
            for n in nbrs[v]:
                n = int(n)
                if n == root:
                    if len(path) >= 3 and v not in spent:
                        out.append(list(path))
                elif n > root and n not in path and len(path) < max_depth:
                    path.append(n)
                    walk(n)
                    path.pop()
                    if len(path) == 1:
                        spent.add(n)
        walk(root)
    return out


def test_pruned_search_equals_unpruned_search():
    """the hop-distance pruning of oracle/graph_ref.py (the kernel's rule) changes no ring and no
    order, on a dense random graph at depth 10"""
    pts = []
    for p in np.random.default_rng(11).uniform(0, 26.0, (20000, 2)):
        if all(np.hypot(*(p - q)) >= 1.2 for q in pts):   # saturates near 340 atoms
            pts.append(p)
    c = np.concatenate([np.array(pts), np.zeros((len(pts), 1))], 1)
    nb = graph_ref.bonds(c, {0: "C"})
    assert np.mean([len(x) for x in nb]) > 3
    got = graph_ref.rings(nb, 10)
    assert len(got) > 5000
    assert got == _unpruned_rings(nb, 10)
