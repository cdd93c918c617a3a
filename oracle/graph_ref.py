"""
Host restatement of atomai.utils.graphx (reference atomai/utils/graphx.py) for the tests of
atomai_b200.utils.graphx: brute-force float64 bonds, a depth-first ring search over atoms above
each root, breadth-first hop distances for the shortest-path filter, and the node orders of the
reference's networkx graphs (networkx itself, imported where those are built).

Neighbour lists are ascending, as the reference's single-class k-d tree query returns them.
"""
from collections import deque

import numpy as np

RADII = {"H": 32.0, "B": 85.0, "C": 75.0, "N": 71.0, "O": 63.0, "P": 111.0, "S": 103.0,
         "Si": 116.0}


def cutoff(a: str, b: str, expand=1.2) -> float:
    r12 = (RADII[a] + RADII[b]) / 100
    if expand:
        r12 = expand * r12
    return r12


def scaled(coordinate_data, px2ang):
    c = coordinate_data.copy()
    c[:, :-1] = c[:, :-1] * px2ang
    return c


def bonds(coords, map_dict, expand=1.2):
    """ascending neighbour lists of scaled (N, 3) or (N, 4) rows"""
    pos = np.zeros((len(coords), 3))
    pos[:, :coords.shape[1] - 1] = coords[:, :-1]
    el = [map_dict[c] for c in coords[:, -1]]
    uniq = sorted(set(el))
    cut = {(a, b): cutoff(a, b, expand) for a in uniq for b in uniq}
    cmat = np.array([[cut[(a, b)] for b in uniq] for a in uniq])
    ci = np.array([uniq.index(e) for e in el])
    # every pair whose x differs by at most the largest cutoff, in blocks of atoms sorted by x
    order = np.argsort(pos[:, 0], kind="stable")
    xs = pos[order, 0]
    rmax = cmat.max()
    out = [None] * len(pos)
    for b0 in range(0, len(pos), 256):
        blk = order[b0:b0 + 256]
        lo = np.searchsorted(xs, xs[b0] - rmax, "left")
        hi = np.searchsorted(xs, xs[min(b0 + 256, len(pos)) - 1] + rmax, "right")
        cand = np.sort(order[lo:hi])
        d = np.sqrt(((pos[blk][:, None, :] - pos[cand][None, :, :]) ** 2).sum(-1))
        ok = d <= cmat[ci[blk]][:, ci[cand]]
        for r, i in enumerate(blk):
            row = cand[ok[r]]
            out[i] = row[row != i]
    return out


def hops_from(nbrs, src, limit):
    """{atom: hops} for the atoms within `limit` bonds of src"""
    dist = {src: 0}
    q = deque([src])
    while q:
        v = q.popleft()
        if dist[v] == limit:
            continue
        for w in nbrs[v]:
            if w not in dist:
                dist[w] = dist[v] + 1
                q.append(w)
    return dist


def rings(nbrs, max_depth):
    """every simple cycle of 3 ... max_depth atoms from its lowest atom, in discovery order: root
    ascending, then depth-first over ascending neighbours; a ring closes at its last atom when that
    atom is bonded to the root and above the root's first step"""
    out = []
    for root in range(len(nbrs)):
        near = hops_from(nbrs, root, max_depth // 2)
        path = [root]

        def dfs(v):
            for n in nbrs[v]:
                n = int(n)
                if n <= root or n in path:
                    continue
                h = near.get(n)
                if h is None or h > max_depth - len(path):
                    continue
                path.append(n)
                if len(path) >= 3 and h == 1 and n > path[1]:
                    out.append(list(path))
                if len(path) < max_depth:
                    dfs(n)
                path.pop()
        dfs(root)
    return out


def shortest_path_rings(nbrs, rl):
    """the rings without a shorter path through the graph between two of their atoms"""
    keep = []
    for r in rl:
        l = len(r)
        ok = True
        for j in range(l):
            dist = hops_from(nbrs, r[j], l // 2)
            for k in range(j + 2, l):
                if dist.get(r[k], l) < min(k - j, l - k + j):
                    ok = False
        if ok:
            keep.append(r)
    return keep


def analyse(coordinate_data, cycles, map_dict, px2ang, expand=1.2):
    cycles = [cycles] if isinstance(cycles, int) else list(cycles)
    c = scaled(coordinate_data, px2ang)
    nb = bonds(c, map_dict, expand)
    return cycles, c, nb, shortest_path_rings(nb, rings(nb, max(cycles)))


def find_cycles(coordinate_data, cycles, map_dict, px2ang, expand=1.2):
    cycles, c, _, rl = analyse(coordinate_data, cycles, map_dict, px2ang, expand)
    rl = sorted((sorted(r) for r in rl), key=lambda x: (len(x), x[0], x[1], x[2]))
    out = np.concatenate([c[r] for r in rl if len(r) in cycles])
    out[:, :-1] = out[:, :-1] * (1 / px2ang)
    return out


def find_cycle_clusters(coordinate_data, cycles, map_dict, px2ang, expand=1.2):
    import networkx as nx
    cycles, c, nb, rl = analyse(coordinate_data, cycles, map_dict, px2ang, expand)
    g = nx.Graph()
    for r in rl:
        if len(r) not in cycles:
            continue
        for v in r:
            g.add_node(v)
            hi = [int(w) for w in nb[v] if w > v]
            for w in hi:
                g.add_node(w)
            for w in hi:
                g.add_edge(v, w)
    g.remove_nodes_from([v for v, d in g.degree() if d < 2])
    return [c[list(g.subgraph(s).copy().nodes)][:, :-1] * (1 / px2ang)
            for s in nx.connected_components(g)]


def filter_subgraphs_(coordinate_arr, map_dict, px2ang, expand=1.2):
    import networkx as nx
    c = scaled(coordinate_arr, px2ang)
    nb = bonds(c, map_dict, expand)
    g = nx.Graph()
    for v in range(len(c)):
        g.add_node(v)
        for w in nb[v]:
            g.add_node(int(w))
        for w in nb[v]:
            g.add_edge(v, int(w))
    subs = [g.subgraph(s).copy() for s in nx.connected_components(g)]
    main = subs[int(np.argmax([len(s) for s in subs]))]
    inv = {v: k for k, v in map_dict.items()}
    idx = list(main.nodes)
    cls = np.array([inv[map_dict[k]] for k in c[idx, -1]], dtype=np.float64)
    return np.concatenate([c[idx, :2].astype(np.float64) / px2ang, cls[:, None]], 1)
