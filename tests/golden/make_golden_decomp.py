"""
Generates tests/golden/decomp_sklearn.npz by running sklearn (the library the reference's
atomai.stat calls for its decompositions) on the float64 copy of each fp32 input of
decomp_cases.py:

  pca/<tag>/   PCA(svd_solver='full') with all components: explained_variance_, singular_values_,
               explained_variance_ratio_, mean_ and the first PCA_K components_ and projections;
  nmf/<tag>/   NMF(init='custom', tol=NMF_TOL) from the case's (W0, H0): W, H, n_iter_,
               reconstruction_err_; and NMF with its default init: reconstruction_err_ only;
  ica/<tag>/   FastICA(ICA_K, random_state=seed): components_, mixing_, mean_, n_iter_ and the
               sources.

Inputs are regenerated from seeds by decomp_cases.py.  Run in the build container only:

    python tests/golden/make_golden_decomp.py
"""
import os
import sys

import numpy as np
from sklearn.decomposition import NMF, PCA, FastICA

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import decomp_cases as dc  # noqa: E402


def main():
    out = {}
    for tag in dc.PCA:
        X = dc.pca_input(tag).astype(np.float64)
        p = PCA(svd_solver="full").fit(X)
        pre = f"pca/{tag}/"
        out[pre + "explained_variance"] = p.explained_variance_
        out[pre + "explained_variance_ratio"] = p.explained_variance_ratio_
        out[pre + "singular_values"] = p.singular_values_
        out[pre + "mean"] = p.mean_
        out[pre + "components"] = p.components_[:dc.PCA_K]
        out[pre + "transform"] = p.transform(X)[:, :dc.PCA_K]
    for tag, (N, d, k, seed) in dc.NMF.items():
        X, W0, H0 = dc.nmf_mixture(N, d, k, seed)
        X = X.astype(np.float64)
        m = NMF(k, init="custom", max_iter=200, tol=dc.NMF_TOL)
        W = m.fit_transform(X, W=W0.astype(np.float64), H=H0.astype(np.float64))
        pre = f"nmf/{tag}/"
        out[pre + "W"], out[pre + "H"] = W, m.components_
        out[pre + "n_iter"] = np.int64(m.n_iter_)
        out[pre + "err"] = np.float64(m.reconstruction_err_)
        out[pre + "default_err"] = np.float64(NMF(k, random_state=seed).fit(X).reconstruction_err_)
    for tag, (N, d, seed) in dc.ICA.items():
        X = dc.ica_mixture(N, d, seed).astype(np.float64)
        ica = FastICA(dc.ICA_K, random_state=seed)
        S = ica.fit_transform(X)
        pre = f"ica/{tag}/"
        out[pre + "components"], out[pre + "mixing"] = ica.components_, ica.mixing_
        out[pre + "mean"], out[pre + "sources"] = ica.mean_, S
        out[pre + "n_iter"] = np.int64(ica.n_iter_)
    np.savez_compressed(os.path.join(HERE, "decomp_sklearn.npz"), **out)


if __name__ == "__main__":
    main()
