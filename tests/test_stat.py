"""atomai_b200.stat without a GPU: public names and signatures against the reference's
(tests/golden/stat_signatures.json), the host-side trajectory and transition functions against
the reference's outputs (tests/golden/stat_separated.npz), and every argument error raised before a
device is touched."""
import inspect
import json
import os

import numpy as np
import pytest

import stat_cases
from atomai_b200 import stat

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEP = np.load(os.path.join(HERE, "stat_separated.npz"))


def test_public_names_and_signatures_match_reference():
    ref = json.load(open(os.path.join(HERE, "stat_signatures.json")))
    for key, sig in ref.items():
        name, _, meth = key.partition(".")
        obj = getattr(stat, name)
        got = inspect.signature(getattr(obj, meth) if meth else
                                (obj.__init__ if inspect.isclass(obj) else obj))
        assert str(got) == sig, key
    import atomai_b200
    assert "stat" in atomai_b200.__all__


def test_calculate_transition_matrix_and_renumerate():
    trace = np.array([0, 0, 2, 1, 2, 2, 0])
    M = stat.calculate_transition_matrix(trace)
    ref = np.zeros((3, 3))
    for i, j in zip(trace, trace[1:]):
        ref[i, j] += 1
    ref /= ref.sum(1, keepdims=True)
    np.testing.assert_array_equal(M, ref)
    np.testing.assert_array_equal(stat.imlocal.renumerate_classes(np.array([3., 1., 3., 5.])),
                                  [1, 0, 1, 2])


def test_transitions_of_golden_trajectories():
    tag = "w32c3"
    n = int(SEP[f"{tag}/ntraj"])
    trans = [stat.calculate_transition_matrix(
        stat.imlocal.renumerate_classes(SEP[f"{tag}/traj{i}"][:, -1])) for i in range(n)]
    for i, m in enumerate(trans):
        np.testing.assert_array_equal(m, SEP[f"{tag}/trans{i}"])
    d = {"trajectories": [SEP[f"{tag}/traj{i}"] for i in range(n)], "transitions": trans}
    np.testing.assert_allclose(stat.sum_transitions(d, 3), SEP[f"{tag}/all_transitions"],
                               rtol=1e-12)


def test_get_trajectory_matches_golden():
    tag = "w32c3"
    cf = SEP[f"{tag}/com_frames"]
    per_frame = {f: cf[cf[:, 3] == f][:, :3] for f in np.unique(cf[:, 3])}
    first = per_frame[0.0]
    for i in range(int(SEP[f"{tag}/ntraj"])):
        flow, frames = stat.imlocal.get_trajectory(per_frame, first[i, :2], 5)
        np.testing.assert_array_equal(flow, SEP[f"{tag}/traj{i}"])
        np.testing.assert_array_equal(frames, SEP[f"{tag}/frames{i}"])


X = np.zeros((10, 4), np.float32)


@pytest.mark.parametrize("make,exc", [
    (lambda: stat.GaussianMixture(3, covariance_type="full"), NotImplementedError),
    (lambda: stat.GaussianMixture(3, covariance_type="tied"), NotImplementedError),
    (lambda: stat.GaussianMixture(3, covariance_type="bogus"), ValueError),
    (lambda: stat.GaussianMixture(65, covariance_type="diag"), ValueError),
    (lambda: stat.GaussianMixture(0, covariance_type="diag"), ValueError),
    (lambda: stat.GaussianMixture(3, covariance_type="diag", init_labels=np.zeros(9)), ValueError),
    (lambda: stat.GaussianMixture(3, covariance_type="diag", init_labels=np.full(10, 3)), ValueError),
    (lambda: stat.KMeans(65), ValueError),
    (lambda: stat.KMeans(3, n_init=10), NotImplementedError),
    (lambda: stat.KMeans(3, init=np.zeros((3, 5))), ValueError),
    (lambda: stat.GaussianMixture(11, covariance_type="diag"), ValueError),   # n_samples < K
])
def test_argument_errors_raise_before_device(make, exc):
    with pytest.raises(exc):
        make().fit(X)


def test_not_native_paths_raise():
    for cls in (stat.SlidingFFTNMF, stat.SpectralUnmixer):
        with pytest.raises(NotImplementedError):
            cls()
    obj = object.__new__(stat.imlocal)
    for name in ("pca", "ica", "nmf", "imblock_pca", "imblock_ica", "imblock_nmf"):
        with pytest.raises(NotImplementedError, match="native"):
            getattr(obj, name)(2)
    with pytest.raises(NotImplementedError):
        obj.pca_gmm(2, 2)
    with pytest.raises(NotImplementedError):
        obj.pca_scree_plot()
    with pytest.raises(NotImplementedError):
        obj.pca_gmm_scree_plot(2)
    with pytest.raises(NotImplementedError, match="meanshift"):
        stat.update_classes(np.zeros((3, 3)), np.zeros((8, 8)), method="meanshift")


def test_get_intensities():
    from atomai_b200.utils import get_intensities
    img = np.arange(100, dtype=np.float64).reshape(1, 10, 10)
    v = get_intensities({0: np.array([[4.2, 5.0, 0.0]])}, img, 3)[0]
    assert v[0] == img[0, 3:6, 4:7].mean()
    v = get_intensities({0: np.array([[4.0, 5.0, 0.0]])}, img, 4)[0]
    assert v[0] == img[0, 2:6, 3:7].mean()
