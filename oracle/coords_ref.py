"""
Float64 numpy restatement of utils.coords' neighbour searches (csrc/coords.cu), for the tests: no
k-d tree and no sklearn.  Distances are sqrt(dx*dx + dy*dy [+ dz*dz]) with numpy's separate
roundings, in column order; an equal distance goes to the lower index.

  knn           brute force over each frame (chunked), or the pairs within an upper bound
  pairs_within  every (query, point) pair closer than r (or within r), from a host cell grid
  walk          subimg_trajectories' walk with numpy slicing
  dbscan        sklearn's dbscan_inner loop over the eps-neighbourhoods
"""
from typing import Dict, List

import numpy as np


def _dist(q: np.ndarray, p: np.ndarray) -> np.ndarray:
    """(len(q), len(p)) distances over the columns of q and p"""
    s = None
    for a in range(q.shape[1]):
        d = q[:, a][:, None] - p[:, a][None]
        s = d * d if s is None else s + d * d
    return np.sqrt(s)


def pairs_within(q: np.ndarray, p: np.ndarray, r: float, inclusive: bool):
    """(qi, pj, d) of every pair with d < r (d <= r when inclusive), over all columns of q and p,
    found through a grid of cells of side r on the first two columns"""
    side = r * (1 + 1e-9)
    lo = np.minimum(q[:, :2].min(0), p[:, :2].min(0)) if len(q) and len(p) else np.zeros(2)
    cq = np.floor((q[:, :2] - lo) / side).astype(np.int64)
    cp = np.floor((p[:, :2] - lo) / side).astype(np.int64)
    ny = int(max(cq[:, 1].max(initial=0), cp[:, 1].max(initial=0))) + 3
    key_p = cp[:, 0] * ny + cp[:, 1]
    order = np.argsort(key_p, kind="stable")
    sk = key_p[order]
    qis, pjs = [], []
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            kq = (cq[:, 0] + dx) * ny + (cq[:, 1] + dy)
            a, b = np.searchsorted(sk, kq, "left"), np.searchsorted(sk, kq, "right")
            n = b - a
            qi = np.repeat(np.arange(len(q)), n)
            start = np.repeat(a - np.concatenate(([0], np.cumsum(n)[:-1])), n)
            pjs.append(order[start + np.arange(n.sum())])
            qis.append(qi)
    qi, pj = np.concatenate(qis), np.concatenate(pjs)
    s = None
    for c in range(q.shape[1]):
        d = q[qi, c] - p[pj, c]
        s = d * d if s is None else s + d * d
    d = np.sqrt(s)
    keep = d <= r if inclusive else d < r
    return qi[keep], pj[keep], d[keep]


def knn(q: np.ndarray, p: np.ndarray, k: int, ub: float = np.inf, chunk: int = 2048):
    """(idx (Q, k) int64 with -1, dist (Q, k) with inf): the k nearest rows of p with d < ub"""
    idx = np.full((len(q), k), -1, np.int64)
    dist = np.full((len(q), k), np.inf)
    if len(p) == 0:
        return idx, dist
    if np.isfinite(ub):
        qi, pj, d = pairs_within(q, p, ub, False)
        o = np.lexsort((pj, d, qi))
        qi, pj, d = qi[o], pj[o], d[o]
        first = np.searchsorted(qi, qi, "left")
        rank = np.arange(len(qi)) - first
        m = rank < k
        idx[qi[m], rank[m]] = pj[m]
        dist[qi[m], rank[m]] = d[m]
        return idx, dist
    for s in range(0, len(q), chunk):
        d = _dist(q[s:s + chunk], p)
        o = np.argsort(d, axis=1, kind="stable")[:, :k]      # stable: a tie keeps index order
        n = o.shape[1]
        idx[s:s + chunk, :n] = o
        dist[s:s + chunk, :n] = np.take_along_axis(d, o, 1)
    return idx, dist


def get_nn_distances(coordinates, nn: int = 2, upper_bound=None):
    if isinstance(coordinates, np.ndarray):
        coordinates = {0: coordinates}
    ub = np.inf if upper_bound is None else upper_bound
    dists, pairs = [], []
    for c in coordinates.values():
        i, d = knn(c[:, :2].astype(np.float64), c[:, :2].astype(np.float64), nn + 1, ub)
        keep = (i >= 0).all(1)
        dists.append(d[keep][:, 1:])
        pairs.append(c[i[keep]])
    return dists, pairs


def compare_coordinates(c1: np.ndarray, c2: np.ndarray, d_max: float):
    if len(c1) and len(c2):
        if np.isfinite(d_max) and d_max > 0:
            qi, pj, d = pairs_within(c1.astype(np.float64), c2.astype(np.float64), d_max, False)
            o = np.lexsort((pj, d, qi))
            qi, pj, d = qi[o], pj[o], d[o]
            first = np.unique(qi, return_index=True)[1]
            keep, idx, dist = qi[first], pj[first], d[first]
        else:
            i, d = knn(c1.astype(np.float64), c2.astype(np.float64), 1)
            sel = d[:, 0] < d_max
            keep, idx, dist = np.flatnonzero(sel), i[sel, 0], d[sel, 0]
    else:
        keep = idx = np.zeros(0, np.int64)
        dist = np.zeros(0)
    if len(keep):
        return (np.append(np.empty((0, 3)), c1[keep], axis=0),
                np.append(np.empty((0, 3)), c2[idx], axis=0), dist)
    return np.empty((0, 3)), np.empty((0, 3)), dist


def stack(coord_dict, n: int) -> np.ndarray:
    return np.concatenate([np.empty((0, 3))] + [np.asarray(coord_dict[k]) for k in range(n)], axis=0)


def find_coord_clusters(d1, d2, rmax: float):
    allc = stack(d2, len(d2))
    q = np.asarray(d1[0])[:, :2].astype(np.float64)
    qi, pj, d = pairs_within(q, allc[:, :2], rmax, False) if rmax > 0 else (np.zeros(0, int),) * 3
    o = np.lexsort((pj, d, qi))
    qi, pj = qi[o], pj[o]
    bounds = np.searchsorted(qi, np.arange(len(q) + 1))
    clusters, means, stds = [], [], []
    for i in range(len(q)):
        c = allc[pj[bounds[i]:bounds[i + 1]]]
        means.append(np.mean(c[:, :2], axis=0))
        stds.append(np.std(c[:, :2], axis=0))
        clusters.append(c)
    return np.array(means), np.array(stds), clusters


def dbscan(xy: np.ndarray, eps: float, min_samples: int) -> np.ndarray:
    """labels of sklearn's dbscan_inner over the eps-neighbourhoods (inclusive, self included)"""
    n = len(xy)
    qi, pj, _ = pairs_within(xy.astype(np.float64), xy.astype(np.float64), eps, True)
    o = np.lexsort((pj, qi))
    qi, pj = qi[o], pj[o]
    bounds = np.searchsorted(qi, np.arange(n + 1))
    is_core = np.diff(bounds) >= min_samples
    labels = np.full(n, -1, np.int64)
    label_num = 0
    for i in range(n):
        if labels[i] != -1 or not is_core[i]:
            continue
        st = []
        while True:
            if labels[i] == -1:
                labels[i] = label_num
                if is_core[i]:
                    for v in pj[bounds[i]:bounds[i + 1]]:
                        if labels[v] == -1:
                            st.append(v)
            if not st:
                break
            i = st.pop()
        label_num += 1
    return labels


def cluster_coord(coord_dict, eps: float, min_samples: int = 10):
    allc = stack(coord_dict, len(coord_dict))
    labels = dbscan(allc[:, :2], eps, min_samples)
    clusters, var, mean = [], [], []
    for lab in np.unique(labels)[1:]:
        c = allc[np.where(labels == lab)]
        clusters.append(c)
        mean.append(np.mean(c[:, :2], axis=0))
        var.append(np.var(c[:, :2], axis=0))
    return clusters, np.array(mean), np.array(var)


def trajectory(imgdata, coord_dict: Dict, r: int, rmax: float, start) -> tuple:
    """one walk of subimg_trajectories with numpy slicing"""
    flow, frames, crops = [], [], []
    c0 = np.asarray(start, np.float64)[:2]
    for k, c in coord_dict.items():
        if len(c) == 0:
            continue
        d = np.sqrt((c0[0] - c[:, 0]) * (c0[0] - c[:, 0]) + (c0[1] - c[:, 1]) * (c0[1] - c[:, 1]))
        j = int(np.lexsort((np.arange(len(c)), d))[0])
        if not d[j] < rmax:
            continue
        cx, cy = int(np.around(c[j][0])), int(np.around(c[j][1]))
        crop = imgdata[k][cx - r // 2:cx + r // 2, cy - r // 2:cy + r // 2]
        if crop.shape[0:2] == (r, r):
            flow.append(c[j])
            crops.append(crop)
            frames.append(k)
            c0 = c[j][:2]
    return np.array(flow), np.array(frames), np.array(crops)


def all_trajectories(imgdata, coord_dict: Dict, r: int, min_length: int, rmax: float):
    out: List[list] = [[], [], []]
    first = coord_dict[list(coord_dict)[0]]
    for ck in first[:, :2]:
        t = trajectory(imgdata, coord_dict, r, rmax, ck)
        if len(t[0]) > min_length:
            for a, b in zip(out, t):
                a.append(b)
    return tuple(out)
