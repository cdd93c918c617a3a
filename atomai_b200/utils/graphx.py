"""Bond graphs of atomic coordinates, their shortest-path rings and ring-defect clusters, after
atomai.utils.graphx, with every pass over the atoms on the GPU (csrc/graph.cu):

  bonds     cell list of side just above the largest bond cutoff, float64 distances, CSR rows ascending;
  hops      hop table: for every atom, the atoms within max_depth // 2 bonds and their distance;
  rings     every simple cycle of 3 ... max_depth atoms, found once from its lowest atom, in the
            order of the reference's recursive search over ascending neighbour lists;
  filter    drops the rings with a shorter path through the graph between two of their atoms.

`find_cycles`, `find_cycle_clusters` and `filter_subgraphs` go from arrays to arrays; `Graph` keeps
the reference's node-level interface on top of the same kernels.  Connected components are taken
on the host and ordered as networkx orders them in the reference.
"""
import warnings
from copy import copy, deepcopy
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from .. import _C, ops

MAX_RING = _C.GRAPH_MAX_RING

# Single-bond covalent radii in pm: P. Pyykkö and M. Atsumi, Chem. Eur. J. 15, 186-197 (2009),
# the values `mendeleev.element(sym).covalent_radius` returns
_SYMBOLS = (
    "H He Li Be B C N O F Ne Na Mg Al Si P S Cl Ar K Ca Sc Ti V Cr Mn Fe Co Ni Cu Zn Ga Ge As Se "
    "Br Kr Rb Sr Y Zr Nb Mo Tc Ru Rh Pd Ag Cd In Sn Sb Te I Xe Cs Ba La Ce Pr Nd Pm Sm Eu Gd Tb Dy "
    "Ho Er Tm Yb Lu Hf Ta W Re Os Ir Pt Au Hg Tl Pb Bi Po At Rn Fr Ra Ac Th Pa U Np Pu Am Cm Bk Cf "
    "Es Fm Md No Lr Rf Db Sg Bh Hs Mt Ds Rg Cn Nh Fl Mc Lv Ts Og").split()
_RADII = (
    32, 46, 133, 102, 85, 75, 71, 63, 64, 67, 155, 139, 126, 116, 111, 103, 99, 96, 196, 171, 148,
    136, 134, 122, 119, 116, 111, 110, 112, 118, 124, 121, 121, 116, 114, 117, 210, 185, 163, 154,
    147, 138, 128, 125, 125, 120, 128, 136, 142, 140, 140, 136, 133, 131, 232, 196, 180, 163, 176,
    174, 173, 172, 168, 169, 168, 167, 166, 165, 164, 170, 162, 152, 146, 137, 131, 129, 122, 123,
    124, 133, 144, 144, 151, 145, 147, 142, 223, 201, 186, 175, 169, 170, 171, 172, 166, 166, 168,
    168, 165, 167, 173, 176, 161, 157, 149, 143, 141, 134, 129, 128, 121, 122, 136, 143, 162, 175,
    165, 157)
COVALENT_RADII = dict(zip(_SYMBOLS, (float(r) for r in _RADII)))


def covalent_radius(symbol: str) -> float:
    """Single-bond covalent radius (pm) of a chemical element"""
    try:
        return COVALENT_RADII[symbol]
    except (KeyError, TypeError):
        raise ValueError(f"unknown chemical element {symbol!r}") from None


def get_interatomic_r(atoms: Union[Tuple[str], List[str]],
                      expand: Optional[float] = None) -> float:
    """Largest bonding distance (Å) of two elements: the sum of their covalent radii, times
    `expand` when that is given and non-zero.  The graph functions pass expand=1.2 by default,
    which lets a bond stretch by 20 %.

    Args:
        atoms: the two element symbols, e.g. ("C", "Si")
        expand: stretch factor of the bond, or None for the bare sum
    """
    atom1, atom2 = atoms
    r12 = (covalent_radius(atom1) + covalent_radius(atom2)) / 100
    if expand:
        r12 = expand * r12
    return r12


# ------------------------------------------------------------------ host checks

def _check_coordinates(coordinates: np.ndarray, map_dict: Dict) -> None:
    if not isinstance(coordinates, np.ndarray) or coordinates.ndim != 2 or \
            coordinates.shape[1] not in (3, 4) or len(coordinates) == 0:
        raise ValueError("coordinates must be a non-empty (N, 3) array of (x, y, class) or an "
                         f"(N, 4) array of (x, y, z, class), got {getattr(coordinates, 'shape', None)}")
    for c in np.unique(coordinates[:, -1]):
        map_dict[c]  # KeyError for a class missing from map_dict, as in the reference
    for c in np.unique(coordinates[:, -1]):
        covalent_radius(map_dict[c])


def _check_cycles(cycles) -> List[int]:
    if isinstance(cycles, (int, np.integer)) and not isinstance(cycles, bool):
        cycles = [cycles]
    cycles = list(cycles)
    if not cycles:
        raise ValueError("cycles must name at least one ring size")
    for c in cycles:
        if isinstance(c, bool) or not isinstance(c, (int, np.integer)) or not 3 <= c <= MAX_RING:
            raise ValueError(f"ring sizes must be integers in 3 ... {MAX_RING}, got {c!r}")
    return [int(c) for c in cycles]


def _check_free(need: int, what: str) -> None:
    free, _ = torch.cuda.mem_get_info()
    if need > free:
        raise MemoryError(f"{what} needs about {need / 2**30:.1f} GiB of device memory, "
                          f"{free / 2**30:.1f} GiB are free")


def _device() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("utils.graphx runs on a CUDA device; none is available")
    return torch.device("cuda")


def _scaled(coordinate_data: np.ndarray, px2ang: float) -> np.ndarray:
    coordinates = deepcopy(coordinate_data)
    coordinates[:, :-1] = coordinates[:, :-1] * px2ang
    return coordinates


def _xyz(coordinates: np.ndarray) -> np.ndarray:
    """float64 (N, 3) positions of (x, y, class) or (x, y, z, class) rows"""
    pos = np.zeros((len(coordinates), 3))
    pos[:, :coordinates.shape[1] - 1] = coordinates[:, :-1]
    return pos


# ------------------------------------------------------------------ device pipeline

class _Bonds:
    """Bond graph of one or more frames: CSR (rowptr, cols) on the device and on the host."""

    def __init__(self, frames: List[np.ndarray], map_dict: Dict, expand: float):
        dev = _device()
        pos = np.concatenate([_xyz(c) for c in frames])
        if not np.isfinite(pos).all():
            raise ValueError("coordinates must be finite")
        classes = np.concatenate([c[:, -1] for c in frames])
        uval = np.unique(classes)
        elems = [map_dict[u] for u in uval]
        cut = np.array([[get_interatomic_r([a, b], expand) for b in elems] for a in elems],
                       dtype=np.float64)
        N = len(pos)
        if N >= 1 << 26:
            raise ValueError(f"at most {(1 << 26) - 1} atoms per call, got {N}")
        lo = pos.min(0)
        rmax = float(cut.max()) if cut.max() > 0 else 1.0
        # Two atoms one largest cutoff apart must land in neighbouring cells.  floor((p - lo) /
        # side) carries a rounding error of a few ulps of the cell index, so the side exceeds the
        # cutoff by that much relative to the largest index.
        span = float((pos.max(0) - lo).max())
        side = rmax * (1 + 2.0 ** -48 * (span / rmax + 1))
        dims = np.floor((pos.max(0) - lo) / side).astype(np.int64) + 1
        if np.prod(dims.astype(np.float64)) * len(frames) >= 2.0 ** 62:
            raise ValueError("the coordinates span too many bond lengths for the cell grid")
        _check_free(N * 64, "the bond search")
        self.N = N
        t_pos = torch.from_numpy(pos).to(dev)
        t_cls = torch.from_numpy(np.searchsorted(uval, classes).astype(np.int32)).to(dev) \
            if len(uval) > 1 else None
        t_frame = torch.from_numpy(np.repeat(np.arange(len(frames), dtype=np.int32),
                                             [len(c) for c in frames])).to(dev) \
            if len(frames) > 1 else None
        t_cut = torch.from_numpy(cut).to(dev)
        keys = torch.empty(N, dtype=torch.int64, device=dev)
        ops.graph_cell_keys(t_pos, t_frame, lo, side, dims, keys)
        keys, perm = torch.sort(keys, stable=True)
        deg = torch.empty(N, dtype=torch.int32, device=dev)
        args = (t_pos, t_cls, t_frame, keys, perm, t_cut, lo, side, dims)
        ops.graph_bonds(*args, None, deg)
        self.rowptr = _offsets(deg)
        nnz = int(self.rowptr[-1])
        _check_free(nnz * 4, "the bond lists")
        self.cols = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
        ops.graph_bonds(*args, self.rowptr, self.cols)
        self.rowptr_h = self.rowptr.cpu().numpy()
        self.cols_h = self.cols[:nnz].cpu().numpy()
        self.ball = None

    def row(self, i: int) -> np.ndarray:
        return self.cols_h[self.rowptr_h[i]:self.rowptr_h[i + 1]]

    def hop_table(self, radius: int):
        """(bptr, ball): the atoms within `radius` bonds of every atom, packed (id << 5 | hops)"""
        if self.ball is not None and self.ball[0] >= radius:
            return self.ball[1:]
        dev = self.rowptr.device
        bptr = torch.arange(self.N + 1, dtype=torch.int64, device=dev)
        ball = torch.arange(self.N, dtype=torch.int32, device=dev) << 5
        cnt = torch.empty(self.N, dtype=torch.int64, device=dev)
        for _ in range(radius):
            ops.graph_hops(self.rowptr, self.cols, bptr, ball, None, None, cnt)
            optr = _offsets(cnt)
            total = int(optr[-1])
            _check_free(total * 4, f"the hop table of radius {radius}")
            nxt = torch.empty(total, dtype=torch.int32, device=dev)
            ops.graph_hops(self.rowptr, self.cols, bptr, ball, optr, nxt, None)
            bptr, ball = optr, nxt
        self.ball = (radius, bptr, ball)
        return bptr, ball

    def rings(self, max_depth: int):
        """Shortest-path rings of 3 ... max_depth atoms in discovery order: (lens, atoms, keep,
        steps) on the host, with keep the shortest-path filter and steps the search's path count"""
        bptr, ball = self.hop_table(max_depth // 2)
        dev = self.rowptr.device
        cnt = torch.empty(self.N, 3, dtype=torch.int64, device=dev)
        ops.graph_rings(self.rowptr, self.cols, bptr, ball, max_depth, cnt=cnt)
        ring_base = _offsets(cnt[:, 0])
        atom_base = _offsets(cnt[:, 1])
        R, A = int(ring_base[-1]), int(atom_base[-1])
        steps = int(cnt[:, 2].sum())
        if R == 0:
            return np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, bool), steps
        _check_free(R * 13 + A * 4, "the rings")
        lens = torch.empty(R, dtype=torch.int32, device=dev)
        atoms = torch.empty(A, dtype=torch.int32, device=dev)
        ops.graph_rings(self.rowptr, self.cols, bptr, ball, max_depth, ring_base[:-1],
                        atom_base[:-1], lens, atoms)
        keep = self.ring_filter(lens, atoms)
        return lens.cpu().numpy(), atoms.cpu().numpy(), keep, steps

    def ring_filter(self, lens: torch.Tensor, atoms: torch.Tensor) -> np.ndarray:
        bptr, ball = self.hop_table(int(lens.max()) // 2)
        keep = torch.empty(len(lens), dtype=torch.uint8, device=lens.device)
        ops.graph_ring_filter(_offsets(lens)[:-1], lens, atoms, bptr, ball, keep)
        return keep.cpu().numpy().astype(bool)


def _offsets(counts: torch.Tensor) -> torch.Tensor:
    out = torch.zeros(len(counts) + 1, dtype=torch.int64, device=counts.device)
    torch.cumsum(counts, 0, out=out[1:])
    return out


def _kept_rings(bonds: _Bonds, max_depth: int) -> List[np.ndarray]:
    lens, atoms, keep, _ = bonds.rings(max_depth)
    starts = np.concatenate(([0], np.cumsum(lens, dtype=np.int64)))
    return [atoms[starts[r]:starts[r + 1]] for r in np.flatnonzero(keep)]


# ------------------------------------------------------------------ networkx ordering

def _nx_components(order: List[int], adj: Dict[int, List[int]]) -> List[List[int]]:
    """Node lists of `G.subgraph(c).copy()` for c in networkx's connected_components(G), for a
    graph with node insertion order `order` and adjacency (insertion-ordered) lists `adj`"""
    n = len(order)
    seen, comps = set(), []
    for v in order:
        if v in seen:
            continue
        c = _plain_bfs(adj, n - len(seen), v)
        seen.update(c)
        comps.append(_subgraph_order(order, c))
    return comps


def _plain_bfs(adj: Dict[int, List[int]], n: int, source: int) -> set:
    seen = {source}
    nextlevel = [source]
    while nextlevel:
        thislevel = nextlevel
        nextlevel = []
        for v in thislevel:
            for w in adj[v]:
                if w not in seen:
                    seen.add(w)
                    nextlevel.append(w)
            if len(seen) == n:
                return seen
    return seen


def _subgraph_order(order: List[int], comp: set) -> List[int]:
    """networkx iterates the nodes of a subgraph view in the order of its node set when that set
    is under half the graph, else in the graph's insertion order"""
    nodes = set(v for v in comp)
    if 2 * len(nodes) < len(order):
        return list(nodes)
    return [v for v in order if v in nodes]


def _star_graph(stars, prune: bool) -> Tuple[List[int], Dict[int, List[int]]]:
    """Node order and adjacency lists of a graph grown one star at a time, as networkx records
    them: for each (centre, leaves) the centre, then the leaves, then the centre–leaf edges, each
    node and each neighbour placed where it first appears.  With `prune`, the nodes of degree < 2
    are dropped afterwards, in one sweep."""
    adj: Dict[int, dict] = {}
    for c, leaves in stars:
        adj.setdefault(c, {})
        for w in leaves:
            adj.setdefault(w, {})
        for w in leaves:
            adj[c][w] = adj[w][c] = None
    drop = {v for v, a in adj.items() if len(a) < 2} if prune else set()
    order = [v for v in adj if v not in drop]
    return order, {v: [w for w in adj[v] if w not in drop] for v in order}


def _networkx(stars, attrs, prune: bool):
    """The networkx graph grown as in _star_graph, with node attributes attrs(id)"""
    import networkx as nx
    g = nx.Graph()
    for c, leaves in stars:
        g.add_nodes_from((v, attrs(v)) for v in [c, *leaves])
        g.add_edges_from((c, w) for w in leaves)
    if prune:
        g.remove_nodes_from([v for v, k in g.degree() if k < 2])
    return g


def _ring_stars(rings, higher):
    """(atom, its higher-index neighbours) for every atom of every ring, in ring order: the stars
    of the ring-defect graph"""
    return ((int(v), higher(int(v))) for ring in rings for v in ring)


# ------------------------------------------------------------------ public functions

def _rings_of(coordinate_data, cycles, map_dict, px2ang, kwargs):
    cycles = _check_cycles(cycles)
    coordinates = _scaled(coordinate_data, px2ang)
    _check_coordinates(coordinates, map_dict)
    bonds = _Bonds([coordinates], map_dict, kwargs.get("expand", 1.2))
    return cycles, coordinates, bonds, _kept_rings(bonds, max(cycles))


def find_cycles(coordinate_data: np.ndarray,
                cycles: Union[int, List[int]],
                map_dict: Dict[int, str],
                px2ang: float,
                **kwargs: float) -> np.ndarray:
    """Rows of the atoms of every shortest-path ring of the requested sizes, e.g. the 5- and
    7-membered rings of a Stone–Wales defect in graphene.

    Args:
        coordinate_data: (N, 3) rows (x, y, class) or (N, 4) rows (x, y, z, class), positions in
            pixels; every class must be a key of map_dict
        cycles: a ring size or a list of them, integers in 3 ... 32
        map_dict: class -> chemical symbol, e.g. {0: "C", 1: "Si"}
        px2ang: Å per pixel; bonds are judged in Å
        **expand: stretch factor of the covalent bond length (default 1.2)

    Returns:
        The rings' rows stacked, positions in pixels and the class column as given.  Rings are
        ordered by size, then by their three lowest atom ids; the atoms of a ring by id, so an atom
        shared by several rings appears once per ring.  ValueError when there is no such ring.
    """
    cycles, coordinates, _, rings = _rings_of(coordinate_data, cycles, map_dict, px2ang, kwargs)
    rings = [np.sort(r) for r in rings if len(r) in cycles]
    if not rings:
        raise ValueError("need at least one array to concatenate")
    key = np.array([(len(r), r[0], r[1], r[2]) for r in rings])
    idx = np.lexsort(key.T[::-1])
    coordinates_ = coordinates[np.concatenate([rings[i] for i in idx])]
    coordinates_[:, :-1] = coordinates_[:, :-1] * (1 / px2ang)
    return coordinates_


def find_cycle_clusters(coordinate_data: np.ndarray,
                        cycles: Union[int, List[int]],
                        map_dict: Dict[int, str],
                        px2ang: float,
                        **kwargs: float) -> List[np.ndarray]:
    """Connected clusters of shortest-path rings of the requested sizes, e.g. the extended
    topological defects of a graphene sheet.

    The cluster graph joins every atom of those rings to its bonded atoms of higher index; the
    atoms left with fewer than two links are dropped, once.

    Args:
        coordinate_data: (N, 3) rows (x, y, class) or (N, 4) rows (x, y, z, class), positions in
            pixels; every class must be a key of map_dict
        cycles: a ring size or a list of them, integers in 3 ... 32
        map_dict: class -> chemical symbol, e.g. {0: "C", 1: "Si"}
        px2ang: Å per pixel; bonds are judged in Å
        **expand: stretch factor of the covalent bond length (default 1.2)

    Returns:
        One array per cluster: the positions (pixels, no class column) of its atoms.  Clusters and
        their atoms come in the order networkx gives them in the reference implementation.
    """
    cycles, coordinates, bonds, rings = _rings_of(coordinate_data, cycles, map_dict, px2ang,
                                                  kwargs)
    rings = [r for r in rings if len(r) in cycles]
    order, adj = _star_graph(_ring_stars(rings, lambda v: [int(w) for w in bonds.row(v) if w > v]),
                             prune=True)
    return [coordinates[c][:, :-1] * (1 / px2ang) for c in _nx_components(order, adj)]


def _largest_component(bonds: _Bonds, start: int, n: int) -> np.ndarray:
    """Atom ids (local to the frame) of the first largest connected component of the whole bond
    graph grown atom by atom (star of atom 0, of atom 1, ...), in networkx's node order"""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import connected_components
    rp = bonds.rowptr_h[start:start + n + 1] - bonds.rowptr_h[start]
    cols = bonds.cols_h[bonds.rowptr_h[start]:bonds.rowptr_h[start + n]] - start
    # insertion order: v, then v's neighbours, for v = 0, 1, ...
    first = np.arange(n, dtype=np.int64) + rp[:-1]
    slot = np.arange(len(cols), dtype=np.int64) + np.repeat(np.arange(n) + 1, np.diff(rp))
    np.minimum.at(first, cols, slot)
    order = np.argsort(first, kind="stable")
    g = csr_matrix((np.ones(len(cols), np.int8), cols, rp), shape=(n, n))
    _, label = connected_components(g, directed=False)
    size = np.bincount(label)
    # components in the order of their first node; np.argmax takes the first largest
    comp_order = label[order][np.sort(np.unique(label[order], return_index=True)[1])]
    best = comp_order[np.argmax(size[comp_order])]
    if 2 * size[best] >= n:
        return order[label[order] == best]
    # a component under half the graph: networkx's set order, from the same breadth-first search
    members = np.flatnonzero(label == best)
    adj = {int(v): cols[rp[v]:rp[v + 1]].tolist() for v in members}
    src = int(order[label[order] == best][0])
    seen_before = int(size[comp_order[:list(comp_order).index(best)]].sum())
    c = _plain_bfs(adj, n - seen_before, src)
    return np.array(_subgraph_order(order.tolist(), c), dtype=np.int64)


def _filter_frames(frames: List[np.ndarray], map_dict: Dict, px2ang: float,
                   kwargs) -> List[np.ndarray]:
    scaled = [_scaled(c, px2ang) for c in frames]
    for c in scaled:
        _check_coordinates(c, map_dict)
    bonds = _Bonds(scaled, map_dict, kwargs.get("expand", 1.2))
    # the class written back is the last key that maps to the atom's element
    cls_of = {sym: k for k, sym in map_dict.items()}
    out, start = [], 0
    for c in scaled:
        idx = _largest_component(bonds, start, len(c))
        start += len(c)
        cls = np.array([cls_of[map_dict[k]] for k in c[idx, -1]], dtype=np.float64)
        out.append(np.concatenate([c[idx, :2].astype(np.float64) / px2ang, cls[:, None]], 1))
    return out


def filter_subgraphs_(coordinate_arr: np.ndarray,
                      map_dict: Dict[int, str],
                      px2ang: float,
                      **kwargs: float) -> np.ndarray:
    """Keeps the atoms of the largest connected piece of the bond graph of one frame, which
    drops isolated false detections away from the lattice.

    Args:
        coordinate_arr: (N, 3) rows (x, y, class) or (N, 4) rows (x, y, z, class), positions in
            pixels; every class must be a key of map_dict
        map_dict: class -> chemical symbol, e.g. {0: "C", 1: "Si"}
        px2ang: Å per pixel; bonds are judged in Å
        **expand: stretch factor of the covalent bond length (default 1.2)

    Returns:
        (M, 3) float64 rows (x, y, class) of the kept atoms, in the order networkx gives them in
        the reference implementation.  When several classes map to one element, the class written
        is the last of them in map_dict.
    """
    return _filter_frames([coordinate_arr], map_dict, px2ang, kwargs)[0]


def filter_subgraphs(coordinates: Union[Dict[int, np.ndarray], np.ndarray],
                     map_dict: Dict[int, str],
                     px2ang: float,
                     **kwargs: float) -> Dict[int, np.ndarray]:
    """filter_subgraphs_ for every frame of a movie; the bonds of all frames are searched in one
    batch on the GPU.

    Args:
        coordinates: frame -> coordinate array (e.g. the output of a predictor), or one array,
            which is treated as frame 0
        map_dict: class -> chemical symbol, e.g. {0: "C", 1: "Si"}
        px2ang: Å per pixel; bonds are judged in Å
        **expand: stretch factor of the covalent bond length (default 1.2)

    Returns:
        frame -> the filtered rows of that frame
    """
    if isinstance(coordinates, np.ndarray):
        coordinates = {0: coordinates}
    keys = list(coordinates)
    if not keys:
        return {}
    out = _filter_frames([coordinates[k] for k in keys], map_dict, px2ang, kwargs)
    return dict(zip(keys, out))


# ------------------------------------------------------------------ node-level interface

class Node:
    """One atom of a Graph.

    Attributes:
        id: index of the atom in the graph's coordinates
        pos: its position as a list (x, y, z), Å
        atom: its chemical symbol
        neighbors, neighborscopy: bonded Nodes, ascending by id (after Graph.polycount,
            `neighbors` keeps only those of higher id, as the reference's search leaves it)
        ingraph: the search flag of the reference's ring search
        nn, visited: kept for compatibility; not used
    """

    def __init__(self, idx: int = 0, pos: List[float] = None, atom: str = 'C') -> None:
        self.id = idx
        self.pos = [] if pos is None else pos
        self.atom = atom
        self.neighbors, self.neighborscopy = [], []
        self.ingraph, self.visited = True, False
        self.nn = 0


class Graph:
    """Node-level bond graph of one frame, on the same GPU passes as find_cycles.

    Args:
        coordinates: (N, 3) rows (x, y, class) or (N, 4) rows (x, y, z, class), positions in Å;
            a 3-column array gets z = 0
        map_dict: class -> chemical symbol, e.g. {0: "C", 1: "Si"}

    The usual sequence is find_neighbors(), polycount(max_depth), remove_filled_polygons(); the
    rings are then in `rings` (lists of Node, in discovery order) and rings_to_nx_graph / nx_graph
    export networkx graphs.
    """

    def __init__(self, coordinates: np.ndarray, map_dict: Dict) -> None:
        _check_coordinates(coordinates, map_dict)
        if coordinates.shape[1] == 3:
            coordinates = np.insert(coordinates, 2, 0, axis=1)
        self.coordinates = coordinates
        self.map_dict = map_dict
        self.size = len(coordinates)
        self.vertices = [Node(i, row[:3].tolist(), map_dict[row[3]])
                         for i, row in enumerate(coordinates)]
        self.rings, self.path, self.improper = [], [], []
        self._bonds = None
        self._searched = False  # polycount has run on the current neighbour lists

    def find_neighbors(self, **kwargs: float):
        """Bonds every atom to the atoms within the covalent bond length of the pair (times
        `expand`, default 1.2).  Both `neighbors` and `neighborscopy` of every node are rebuilt,
        ascending by id."""
        self._bonds = _Bonds([self.coordinates], self.map_dict, kwargs.get("expand", 1.2))
        self._searched = False
        for i, v in enumerate(self.vertices):
            v.neighbors = [self.vertices[j] for j in self._bonds.row(i)]
            v.neighborscopy = list(v.neighbors)

    def find_rings(self, *args, **kwargs):
        raise NotImplementedError(
            "the recursive single-node search is not provided: Graph.polycount(max_depth) finds "
            "the rings from every atom at once on the GPU")

    def polycount(self, max_depth: int) -> None:
        """Appends to `rings` every ring of 3 ... max_depth atoms (an integer up to 32), each
        once, found from its lowest atom, in the reference's discovery order.

        Afterwards, as in the reference, no node is `ingraph` and each node's `neighbors` holds
        only its higher-index neighbours.  Rings are found only on the neighbour lists of a
        find_neighbors call with every node `ingraph`; in any other state, e.g. on a second call,
        none are found, which is what the reference's search finds there too.
        """
        max_depth = _check_cycles([max_depth])[0]
        fresh = self._bonds is not None and not self._searched and \
            all(v.ingraph for v in self.vertices)
        if fresh:
            lens, atoms, _, _ = self._bonds.rings(max_depth)
            ends = np.cumsum(lens, dtype=np.int64)
            self.rings.extend([self.vertices[i] for i in atoms[e - n:e]]
                              for n, e in zip(lens, ends))
            for v in self.vertices:
                v.neighbors = [n for n in v.neighbors if n.id > v.id]
            self._searched = True
        for v in self.vertices:
            v.ingraph = False
        self.neighbors = list(self.vertices[-1].neighborscopy)

    def remove_filled_polygons(self):
        """Drops from `rings` every ring two of whose atoms are joined by a shorter path through
        the bond graph than around the ring, keeping the order of the others; marks every node
        `ingraph` again."""
        for v in self.vertices:
            v.ingraph = True
        if not self.rings:
            return
        dev = self._bonds.rowptr.device
        lens = torch.tensor([len(r) for r in self.rings], dtype=torch.int32, device=dev)
        atoms = torch.tensor([v.id for r in self.rings for v in r], dtype=torch.int32, device=dev)
        keep = self._bonds.ring_filter(lens, atoms)
        self.rings = [r for r, k in zip(self.rings, keep) if k]

    def shortest_path(self, *args, **kwargs):
        raise NotImplementedError(
            "the recursive single-pair search is not provided: Graph.remove_filled_polygons() "
            "checks every ring at once on the GPU")

    def _attrs(self, flat: bool):
        def attrs(i):
            v = self.vertices[i]
            return {"pos": tuple(v.pos[:2] if flat else v.pos), "atom": v.atom}
        return attrs

    def rings_to_nx_graph(self, ring_size: List[int]):
        """networkx graph of the rings whose size is in `ring_size`: each ring atom joined to its
        current `neighbors` (the higher-index ones after polycount), then the nodes with fewer
        than two links dropped once.  Nodes carry `pos` (x, y, z) and `atom`."""
        rings = [[v.id for v in r] for r in self.rings if len(r) in ring_size]
        return _networkx(_ring_stars(rings, lambda i: [n.id for n in self.vertices[i].neighbors]),
                         self._attrs(False), prune=True)

    def nx_graph(self):
        """networkx graph of every atom and its current `neighbors`, nodes in the order the atoms
        and their neighbours are met.  Nodes carry `atom` and `pos`: (x, y) when all atoms share
        one z, else (x, y, z)."""
        flat = bool(np.all(self.coordinates[:, 2] == self.coordinates[0, 2]))
        return _networkx(((v.id, [n.id for n in v.neighbors]) for v in self.vertices),
                         self._attrs(flat), prune=False)


def plot_graph(G,
               img: Optional[np.ndarray] = None,
               fsize: Union[int, Tuple[int, int]] = 8,
               show_labels: bool = False,
               **kwargs: Union[int, str, float]) -> None:
    """Draws a graph's atoms and bonds, optionally over the image the atoms were found in.

    Args:
        G: a networkx graph with node attribute `pos` (x, y, ...), or a Graph (its nx_graph())
        img: 2-D image drawn underneath, origin at the lower left
        fsize: figure size, one number for a square figure
        show_labels: write each node's id, or its element with show_elements=True
        **kwargs: node_size (30), node_color, edge_color ("orange"), alpha, cmap ("gray"),
            label_size (7), label_color ("black"), show_elements

    Positions are drawn as (row, column) = (x, y), matching the image's array axes; the graph's
    own `pos` attributes are left as they are.  Without matplotlib or networkx installed, the plot
    is skipped with a warning.
    """
    try:
        import matplotlib.pyplot as plt
        import networkx as nx
    except ImportError:
        warnings.warn("matplotlib or networkx is not installed: plot skipped")
        return
    if isinstance(G, Graph):
        G = G.nx_graph()
    size = fsize if isinstance(fsize, tuple) else (fsize, fsize)
    ax = plt.subplots(1, 1, figsize=size)[1]
    if img is not None:
        ax.imshow(img, origin="lower", cmap=kwargs.get("cmap", "gray"))
    xy = {n: p[::-1] for n, p in nx.get_node_attributes(G, "pos").items()}
    alpha = kwargs.get("alpha")
    nx.draw_networkx_nodes(G, xy, nodelist=list(G.nodes), ax=ax, alpha=alpha,
                           node_size=kwargs.get("node_size", 30),
                           node_color=kwargs.get("node_color", "#1f78b4"))
    nx.draw_networkx_edges(G, xy, width=1, ax=ax, alpha=alpha,
                           edge_color=kwargs.get("edge_color", "orange"))
    if show_labels:
        labels = nx.get_node_attributes(G, "atom") if kwargs.get("show_elements") else None
        nx.draw_networkx_labels(G, xy, labels=labels, ax=ax,
                                font_size=kwargs.get("label_size", 7),
                                font_color=kwargs.get("label_color", "black"))
    plt.show()
