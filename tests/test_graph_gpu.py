"""utils.graphx on the GPU: bit-identical to the reference's outputs (tests/golden/graph_ref.npz)
for single-class input and equal up to order for multi-class input; Graph's ring discovery order
and neighbour-list state; 2·10⁴-atom graphs against the host restatement (oracle/graph_ref.py);
repeatability; batched filter_subgraphs against per-frame calls."""
import os

import numpy as np
import pytest
import torch

import graph_cases as gc
from atomai_b200.utils import graphx
from oracle import graph_ref

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "graph_ref.npz"))
CASES = {"single": gc.single, "z": gc.with_z, "multi": gc.multi}
CYCLES = ([6], [5, 7], list(range(3, 10)))


def _rows(a):
    return a[np.lexsort(a.T[::-1])]


def _tag(cyc):
    return "".join(map(str, cyc))


@pytest.mark.parametrize("tag", ["single", "z"])
def test_single_class_bit_identical(tag):
    c = CASES[tag]()
    for cyc in CYCLES:
        got = graphx.find_cycles(c, cyc, gc.MAP_DICT, gc.PX2ANG)
        assert got.dtype == c.dtype
        np.testing.assert_array_equal(got, GOLD[f"{tag}/cycles_{_tag(cyc)}"])
    cl = graphx.find_cycle_clusters(c, [5, 7], gc.MAP_DICT, gc.PX2ANG)
    np.testing.assert_array_equal(np.concatenate(cl), GOLD[f"{tag}/clusters_57"])
    np.testing.assert_array_equal([len(x) for x in cl], GOLD[f"{tag}/clusters_57_len"])
    np.testing.assert_array_equal(graphx.filter_subgraphs(c, gc.MAP_DICT, gc.PX2ANG)[0],
                                  GOLD[f"{tag}/filter"])


def test_multi_class_equal_up_to_order():
    c = gc.multi()
    for cyc in CYCLES:
        got = graphx.find_cycles(c, cyc, gc.MAP_DICT, gc.PX2ANG)
        np.testing.assert_array_equal(_rows(got), _rows(GOLD[f"multi/cycles_{_tag(cyc)}"]))
    cl = graphx.find_cycle_clusters(c, [5, 7], gc.MAP_DICT, gc.PX2ANG)
    ref = np.split(GOLD["multi/clusters_57"], np.cumsum(GOLD["multi/clusters_57_len"])[:-1])
    key = lambda xs: sorted(tuple(map(tuple, _rows(x))) for x in xs)  # noqa: E731
    assert key(cl) == key(ref)
    got = graphx.filter_subgraphs(c, gc.MAP_DICT, gc.PX2ANG)[0]
    np.testing.assert_array_equal(_rows(got), _rows(GOLD["multi/filter"]))


@pytest.mark.parametrize("tag", ["single", "z", "multi"])
def test_graph_rings_and_neighbour_state(tag):
    c = graph_ref.scaled(CASES[tag](), gc.PX2ANG)
    nb = graph_ref.bonds(c, gc.MAP_DICT)
    G = graphx.Graph(c, gc.MAP_DICT)
    G.find_neighbors(expand=1.2)
    for v in G.vertices:
        assert [n.id for n in v.neighbors] == nb[v.id].tolist()
        assert [n.id for n in v.neighborscopy] == nb[v.id].tolist()
    G.polycount(max_depth=9)
    assert [[v.id for v in r] for r in G.rings] == graph_ref.rings(nb, 9)
    for v in G.vertices:
        assert not v.ingraph
        assert [n.id for n in v.neighbors] == [w for w in nb[v.id].tolist() if w > v.id]
        assert [n.id for n in v.neighborscopy] == nb[v.id].tolist()
    G.remove_filled_polygons()
    assert all(v.ingraph for v in G.vertices)
    got = [[v.id for v in r] for r in G.rings]
    ids, lens = GOLD[f"{tag}/rings_9"], GOLD[f"{tag}/rings_9_len"]
    ref = [r.tolist() for r in np.split(ids, np.cumsum(lens)[:-1])]
    if tag == "multi":
        assert sorted(map(sorted, got)) == sorted(map(sorted, ref))
    else:
        assert got == ref


def test_nx_graphs_match_reference_construction():
    nx = pytest.importorskip("networkx")
    c = graph_ref.scaled(gc.single(), gc.PX2ANG)
    G = graphx.Graph(c, gc.MAP_DICT)
    G.find_neighbors()
    g = G.nx_graph()
    nb0 = [n.id for n in G.vertices[0].neighbors]
    assert list(g.nodes)[:1 + len(nb0)] == [0] + nb0
    assert g.number_of_edges() == sum(len(v.neighbors) for v in G.vertices) // 2
    G.polycount(7)
    G.remove_filled_polygons()
    h = G.rings_to_nx_graph([5, 7])
    ref = graphx.find_cycle_clusters(gc.single(), [5, 7], gc.MAP_DICT, gc.PX2ANG)
    comps = [list(h.subgraph(s).copy().nodes) for s in nx.connected_components(h)]
    assert len(comps) == len(ref) > 0
    for x, idx in zip(ref, comps):
        np.testing.assert_array_equal(x, gc.single()[idx][:, :-1] * gc.PX2ANG * (1 / gc.PX2ANG))


@pytest.mark.parametrize("kind,cycles", [("lattice", [5, 6, 7, 8]), ("amorphous", list(range(3, 11)))])
def test_large_graphs_equal_oracle(kind, cycles):
    c = gc.large(kind)
    _, s, nb, rl = graph_ref.analyse(c, cycles, gc.MAP_DICT, gc.PX2ANG)
    G = graphx.Graph(s, gc.MAP_DICT)
    G.find_neighbors()
    for v in G.vertices[::97]:
        assert [n.id for n in v.neighborscopy] == nb[v.id].tolist()
    G.polycount(max(cycles))
    G.remove_filled_polygons()
    assert [[v.id for v in r] for r in G.rings] == rl
    np.testing.assert_array_equal(graphx.find_cycles(c, cycles, gc.MAP_DICT, gc.PX2ANG),
                                  graph_ref.find_cycles(c, cycles, gc.MAP_DICT, gc.PX2ANG))
    pytest.importorskip("networkx")
    got = graphx.find_cycle_clusters(c, cycles[:2], gc.MAP_DICT, gc.PX2ANG)
    ref = graph_ref.find_cycle_clusters(c, cycles[:2], gc.MAP_DICT, gc.PX2ANG)
    assert len(got) == len(ref)
    for a, b in zip(got, ref):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(graphx.filter_subgraphs_(c, gc.MAP_DICT, gc.PX2ANG),
                                  graph_ref.filter_subgraphs_(c, gc.MAP_DICT, gc.PX2ANG))


def test_repeatable():
    c = gc.large("amorphous")
    a = graphx._Bonds([graph_ref.scaled(c, gc.PX2ANG)], gc.MAP_DICT, 1.2).rings(10)
    b = graphx._Bonds([graph_ref.scaled(c, gc.PX2ANG)], gc.MAP_DICT, 1.2).rings(10)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


def test_batched_frames_equal_per_frame_calls():
    fr = gc.frames()
    fr[3] = gc.with_z()
    batched = graphx.filter_subgraphs(fr, gc.MAP_DICT, gc.PX2ANG)
    assert list(batched) == list(fr)
    for k, c in fr.items():
        np.testing.assert_array_equal(batched[k], graphx.filter_subgraphs_(c, gc.MAP_DICT, gc.PX2ANG))
    for k in (0, 1, 7):
        np.testing.assert_array_equal(batched[k], GOLD[f"frames/{k}"])


def test_one_frame_dict_array_and_no_ring():
    c = gc.single()
    one = graphx.filter_subgraphs({5: c}, gc.MAP_DICT, gc.PX2ANG)
    assert list(one) == [5]
    np.testing.assert_array_equal(one[5], GOLD["single/filter"])
    arr = graphx.filter_subgraphs(c, gc.MAP_DICT, gc.PX2ANG)
    assert list(arr) == [0]
    np.testing.assert_array_equal(arr[0], GOLD["single/filter"])
    with pytest.raises(ValueError):
        graphx.find_cycles(c[:3], [6], gc.MAP_DICT, gc.PX2ANG)   # no ring: np.concatenate([])


def test_polycount_again_finds_no_rings():
    c = graph_ref.scaled(gc.single(), gc.PX2ANG)
    G = graphx.Graph(c, gc.MAP_DICT)
    G.find_neighbors()
    G.polycount(8)
    rings = [[v.id for v in r] for r in G.rings]
    assert rings
    state = [[n.id for n in v.neighbors] for v in G.vertices]
    G.polycount(8)                       # nodes not ingraph: nothing found
    G.remove_filled_polygons()
    kept = [[v.id for v in r] for r in G.rings]
    G.polycount(8)                       # lists already cut to higher-index neighbours
    assert [[v.id for v in r] for r in G.rings] == kept
    assert [[n.id for n in v.neighbors] for v in G.vertices] == state
    G.find_neighbors()                   # fresh lists, but no node ingraph after polycount
    G.polycount(8)
    assert [[v.id for v in r] for r in G.rings] == kept
    assert all(len(v.neighbors) == len(v.neighborscopy) for v in G.vertices)
    G.remove_filled_polygons()
    G.find_neighbors()                   # fresh lists and every node ingraph: found again
    G.polycount(8)
    assert [[v.id for v in r] for r in G.rings] == kept + rings


def test_pairs_just_inside_the_largest_cutoff_bond():
    """a pair one largest cutoff apart (less 1e-9 of it) bonds wherever it lies in the cell grid"""
    rng = np.random.default_rng(3)
    r = graphx.get_interatomic_r(["C", "C"], 1.2)
    n = 4000
    x = rng.uniform(0, 2e4, n)
    y = np.arange(n) * 5.0
    pos = np.stack([np.concatenate([x, x + r * (1 - 1e-9)]), np.concatenate([y, y])], 1)
    c = np.concatenate([pos, np.zeros((2 * n, 1))], 1)
    G = graphx.Graph(c, gc.MAP_DICT)
    G.find_neighbors()
    for i in range(n):
        assert [v.id for v in G.vertices[i].neighbors] == [i + n]
