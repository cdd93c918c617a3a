"""
Generates tests/golden/stat_*.npz by running the UNMODIFIED reference (AtomAI v0.8.1, CPU) through
oracle/ref_shim.py, and sklearn (the library the reference's atomai.stat calls):

  stat_separated.npz  imlocal(...).gmm(3) on the SEPARATED movies of stat_cases.py (cla, the
                      member count of each class, com_frames) and transition_matrix(3) of the
                      movie case (per-trajectory matrices, frames, all_transitions);
  stat_sklearn.npz    on the OVERLAP stacks: KMeans(n_init=1, random_state) labels, then
                      GaussianMixture (diag, spherical; same random_state) means_, covariances_,
                      weights_, fit_predict labels, n_iter_, lower_bounds_; and Lloyd from a fixed
                      centre array (KMeans(init=array, n_init=1)) labels, centres, n_iter_;
  stat_signatures.json  the public signatures of atomai.stat.

Inputs are regenerated from seeds by stat_cases.py.  Run in the build container only:

    python tests/golden/make_golden_stat.py
"""
import importlib
import inspect
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle.ref_shim import import_reference  # noqa: E402
import stat_cases  # noqa: E402

aoi = import_reference()


def signatures(mod):
    out = {}
    for name in mod.__all__:
        obj = getattr(mod, name)
        if inspect.isclass(obj):
            out[name] = str(inspect.signature(obj.__init__))
            if name == "imlocal":
                for m, f in inspect.getmembers(obj):
                    if not m.startswith("_") and callable(f):
                        out[f"imlocal.{m}"] = str(inspect.signature(f))
        else:
            out[name] = str(inspect.signature(obj))
    return out


def main():
    from sklearn.cluster import KMeans
    from sklearn.mixture import GaussianMixture
    stat = importlib.import_module(aoi.__name__ + ".stat")
    with open(os.path.join(HERE, "stat_signatures.json"), "w") as f:
        json.dump(signatures(stat), f, indent=1, sort_keys=True)
    sep = {}
    for tag, (w, c, frames) in stat_cases.SEPARATED.items():
        imgs, coords = stat_cases.separated_movie(w, c, frames)
        s = stat.imlocal(imgs, coords, w, 0)
        cla, cl_all, com_frames = s.gmm(3)
        sep[f"{tag}/cla"] = cla
        sep[f"{tag}/counts"] = np.array([len(x) for x in cl_all])
        sep[f"{tag}/com_frames"] = com_frames
        print(tag, s.imgstack.shape, sep[f"{tag}/counts"])
        if frames > 1:
            d = s.transition_matrix(3, rmax=5, sum_all_transitions=True)
            sep[f"{tag}/ntraj"] = np.array(len(d["trajectories"]))
            for i, (tr, m, fr) in enumerate(zip(d["trajectories"], d["transitions"], d["frames"])):
                sep[f"{tag}/traj{i}"], sep[f"{tag}/trans{i}"], sep[f"{tag}/frames{i}"] = tr, m, fr
            sep[f"{tag}/all_transitions"] = d["all_transitions"]
    np.savez_compressed(os.path.join(HERE, "stat_separated.npz"), **sep)
    sk = {}
    for tag, (N, dim, K, seed) in stat_cases.OVERLAP.items():
        X = stat_cases.overlapping(N, dim, K, seed)
        sk[f"{tag}/km_labels"] = KMeans(K, n_init=1, random_state=seed).fit(X).labels_
        for cov in ("diag", "spherical"):
            g = GaussianMixture(K, covariance_type=cov, random_state=seed)
            lab = g.fit_predict(X)
            p = f"{tag}/{cov}/"
            sk[p + "labels"], sk[p + "means"], sk[p + "covariances"] = lab, g.means_, g.covariances_
            sk[p + "weights"], sk[p + "n_iter"] = g.weights_, np.array(g.n_iter_)
            sk[p + "lower_bounds"] = np.array(g.lower_bounds_)
            print(tag, cov, g.n_iter_, g.lower_bound_)
        init = stat_cases.lloyd_init(X, K, seed)
        km = KMeans(K, init=init, n_init=1).fit(X)
        sk[f"{tag}/lloyd_labels"], sk[f"{tag}/lloyd_centres"] = km.labels_, km.cluster_centers_
        sk[f"{tag}/lloyd_n_iter"] = np.array(km.n_iter_)
        print(tag, "lloyd", km.n_iter_)
    np.savez_compressed(os.path.join(HERE, "stat_sklearn.npz"), **sk)


if __name__ == "__main__":
    main()
