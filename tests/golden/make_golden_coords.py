"""
Generates tests/golden/coords_ref.npz by running the UNMODIFIED reference's atomai.utils.coords
(through oracle/ref_shim.py; scipy's cKDTree and sklearn's DBSCAN) on the tie-free cases of
coords_cases.py:

  nn/<case>_<nn>_<ub>        get_nn_distances: distances and rows of all frames (flat + lengths)
  bonds                      map_bonds(plot_results=False)
  compare/<c1|c2|d>          compare_coordinates on (x, y, class) rows, d_max = 3
  fcc/<mean|std|rows|len>    find_coord_clusters over a 10-frame movie, rmax = 3
  dbscan_<case>/<...>        cluster_coord: noise and two-cluster border points; and a movie
                             without noise (the first cluster is skipped)
  traj_<r>_<chan>/<...>      subimg_trajectories(...).get_all_trajectories() for window 8 and 7
                             on (n, h, w) and (n, h, w, 3) stacks, atoms up to the image edges

Inputs are regenerated from seeds by coords_cases.py.  Run in the build container only:

    python tests/golden/make_golden_coords.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import coords_cases as cc  # noqa: E402
from oracle import ref_shim  # noqa: E402


def flat(out, key, arrays):
    out[f"{key}/flat"] = np.concatenate(
        [np.asarray(a).reshape(len(a), int(np.prod(np.shape(a)[1:]))) for a in arrays]) \
        if arrays else np.zeros((0, 1))
    out[f"{key}/len"] = np.array([len(a) for a in arrays])


def nn_cases():
    mv = cc.movie(5, 12, 3, drop=0.1)
    mv[5] = cc.lattice(2, 9)[:2]          # fewer atoms than some nn: every row dropped
    return {"movie": mv, "single": cc.lattice(15, 4)}


def compare_case():
    rng = np.random.default_rng(5)
    c1 = cc.lattice(20, 6)
    c2 = c1.copy()
    c2[:, :2] += rng.normal(0, 0.8, (len(c2), 2))
    c2[rng.random(len(c2)) < 0.2, 2] += 2.0   # a changed class adds 2 to the distance
    c2 = c2[rng.random(len(c2)) >= 0.1]
    return c1, c2


def dbscan_cases():
    pts, eps, ms = cc.dbscan_points(0)
    mv = cc.movie(12, 6, 8, jitter=0.5, drift=0.1)
    return {"noise": (cc.as_frames(pts, 4), eps, ms), "movie": (mv, 1.0, 10)}


def traj_cases():
    mv = cc.movie(8, 8, 11, drift=0.5, drop=0.05)
    out = {}
    for r in (8, 7):
        for chan in (0, 3):
            out[(r, chan)] = (cc.images(8, 64, 64, 12 + chan, chan), mv, r)
    return out


class _RaggedNumpy:
    """numpy, except that np.array of a ragged list returns the list: the reference's
    cluster_coord ends in np.array(clusters), which numpy >= 1.24 refuses for clusters of
    different sizes"""

    def __getattr__(self, name):
        return getattr(np, name)

    @staticmethod
    def array(x, *a, **k):
        try:
            return np.array(x, *a, **k)
        except ValueError:
            return list(x)


def main():
    ref_shim.import_reference()
    from atomai.utils import coords
    out = {}
    for tag, c in nn_cases().items():
        for nn in (1, 2, 6):
            for ub in (None, 9.0, 12.0):
                d, p = coords.get_nn_distances(c, nn, ub)
                key = f"nn/{tag}_{nn}_{ub}"
                flat(out, f"{key}/d", d)
                flat(out, f"{key}/p", p)
    out["bonds"] = coords.map_bonds(cc.movie(5, 12, 3, drop=0.1), 4, None, plot_results=False)
    c1, c2 = compare_case()
    a, b, d = coords.compare_coordinates(c1, c2, 3.0)
    out["compare/c1"], out["compare/c2"], out["compare/d"] = a, b, d
    mv = cc.movie(10, 10, 7)
    m, s, cl = coords.find_coord_clusters({0: mv[0]}, mv, 3)
    out["fcc/mean"], out["fcc/std"] = m, s
    flat(out, "fcc/rows", cl)
    coords.np = _RaggedNumpy()
    for tag, (fr, eps, ms) in dbscan_cases().items():
        cl, m, v = coords.cluster_coord(fr, eps, ms)
        flat(out, f"dbscan_{tag}/rows", list(cl))
        out[f"dbscan_{tag}/mean"], out[f"dbscan_{tag}/var"] = m, v
    coords.np = np
    for (r, chan), (img, fr, r_) in traj_cases().items():
        t = coords.subimg_trajectories(img, fr, r_, 2, 3).get_all_trajectories()
        key = f"traj_{r}_{chan}"
        flat(out, f"{key}/flow", t[0])
        flat(out, f"{key}/frames", t[1])
        flat(out, f"{key}/crops", t[2])
    np.savez_compressed(os.path.join(HERE, "coords_ref.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
