"""
Generates tests/golden/graph_ref.npz by running the UNMODIFIED reference's atomai.utils.graphx
(through oracle/ref_shim.py) on the cases of graph_cases.py, with `graphx.element` replaced by an
object that serves the Pyykkö & Atsumi single-bond radii (mendeleev's `covalent_radius`):

  single/cycles_<sizes>   find_cycles for [6], [5, 7] and [3 ... 9]
  single/rings_9          Graph.rings after polycount(9) + remove_filled_polygons, as id lists in
                          discovery order (flat ids + lengths)
  single/clusters_57      find_cycle_clusters([5, 7]) (flat rows + cluster lengths)
  single/filter           filter_subgraphs
  multi/..., z/...        the same for the multi-class and the (x, y, z, class) cases
  frames/<k>              filter_subgraphs of the three-frame dict

Inputs are regenerated from seeds by graph_cases.py.  Run in the build container only:

    python tests/golden/make_golden_graph.py
"""
import os
import sys
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import graph_cases as gc  # noqa: E402
from oracle import graph_ref, ref_shim  # noqa: E402


def _element(atoms):
    return [SimpleNamespace(covalent_radius=graph_ref.RADII[a]) for a in atoms]


def _margin(c, map_dict, expand=1.2):
    """least |distance - cutoff| over all atom pairs (Å)"""
    s = graph_ref.scaled(c, gc.PX2ANG)
    pos = np.zeros((len(s), 3))
    pos[:, :s.shape[1] - 1] = s[:, :-1]
    el = [map_dict[k] for k in s[:, -1]]
    cut = np.array([[graph_ref.cutoff(a, b, expand) for b in el] for a in el])
    d = np.sqrt(((pos[:, None] - pos[None]) ** 2).sum(-1))
    return np.abs(d - cut).min()


def main():
    aoi = ref_shim.import_reference()
    from atomai.utils import graphx
    graphx.element = _element
    out = {}
    cases = {"single": gc.single(), "multi": gc.multi(), "z": gc.with_z()}
    for tag, c in cases.items():
        assert _margin(c, gc.MAP_DICT) > 1e-6, tag
        for cyc in ([6], [5, 7], list(range(3, 10))):
            out[f"{tag}/cycles_{''.join(map(str, cyc))}"] = graphx.find_cycles(
                c, cyc, gc.MAP_DICT, gc.PX2ANG)
        s = graph_ref.scaled(c, gc.PX2ANG)
        G = graphx.Graph(s, gc.MAP_DICT)
        G.find_neighbors(expand=1.2)
        G.polycount(max_depth=9)
        n_all = len(G.rings)
        G.remove_filled_polygons()
        assert len(G.rings) < n_all, "no ring removed by the shortest-path filter"
        lens = [len(r) for r in G.rings]
        assert 5 in lens and 7 in lens
        out[f"{tag}/rings_9"] = np.array([v.id for r in G.rings for v in r])
        out[f"{tag}/rings_9_len"] = np.array(lens)
        cl = graphx.find_cycle_clusters(c, [5, 7], gc.MAP_DICT, gc.PX2ANG)
        out[f"{tag}/clusters_57"] = np.concatenate(cl)
        out[f"{tag}/clusters_57_len"] = np.array([len(x) for x in cl])
        out[f"{tag}/filter"] = graphx.filter_subgraphs(c, gc.MAP_DICT, gc.PX2ANG)[0]
    fr = gc.frames()
    for k, c in fr.items():
        assert _margin(c, gc.MAP_DICT) > 1e-6, k
    for k, v in graphx.filter_subgraphs(fr, gc.MAP_DICT, gc.PX2ANG).items():
        out[f"frames/{k}"] = v
    np.savez_compressed(os.path.join(HERE, "graph_ref.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
