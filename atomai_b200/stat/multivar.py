"""
Statistics of local image descriptors: sub-images cut around atoms of one class and clustered
with a Gaussian mixture, and Markov transitions of the classes along atom trajectories through a
movie (the API of atomai/stat/multivar.py).

The windows are cut on the GPU (utils.extract_subimages_cuda) and the mixture is fitted on the
device stack (stat.GaussianMixture); the trajectory bookkeeping works on small coordinate arrays
on the host.
"""
import copy
import warnings
from typing import Dict, List, Tuple, Union

import numpy as np
import torch
from scipy import spatial

from ..utils.coords import get_intensities
from ..utils.img import extract_subimages_cuda
from .mixture import GaussianMixture, KMeans


def _pyplot():
    """matplotlib.pyplot, or None when matplotlib is not installed (plots are then skipped)."""
    try:
        import matplotlib.pyplot as plt
    except ImportError:
        warnings.warn("matplotlib is not installed: plot skipped")
        return None
    return plt


def _not_native(name: str):
    raise NotImplementedError(
        f"imlocal.{name} is not on the native path yet; gmm, get_all_trajectories and "
        "transition_matrix are")


class imlocal:
    """
    Sub-images of side `window_size` centred on the atoms of class `coord_class` in
    `network_output` (images x height x width x channels, numpy or a CUDA tensor) with
    Locator-style coordinates {frame: (N, 3) array of x, y, class}, for clustering and
    trajectory analysis.  `imgstack`, `imgstack_com` and `imgstack_frames` are numpy arrays;
    the fits run on a copy of the stack kept on the GPU.
    """

    def __init__(self,
                 network_output: np.ndarray,
                 coord_class_dict_all: Dict[int, np.ndarray],
                 window_size: int = None,
                 coord_class: int = 0,
                 ) -> None:
        self.network_output = network_output
        self.nb_classes = network_output.shape[-1]
        self.coord_all = coord_class_dict_all
        self.coord_class = float(coord_class)
        self.r = window_size
        (self.imgstack,
         self.imgstack_com,
         self.imgstack_frames) = self.extract_subimages_()
        self.d0, self.d1, self.d2, self.d3 = self.imgstack.shape

    def extract_subimages_(self) -> Tuple[np.ndarray]:
        """Cuts the windows with one gather kernel; returns (stack, centres, frame index)."""
        img = self.network_output
        if not (isinstance(img, torch.Tensor) and img.is_cuda):
            img = torch.from_numpy(np.ascontiguousarray(np.asarray(img, dtype=np.float32))).cuda()
        stack, com, frames = extract_subimages_cuda(
            img.to(torch.float32), self.coord_all, self.r, self.coord_class)
        if len(stack) == 0:
            raise ValueError(f"no window of size {self.r} fits around an atom of class "
                             f"{self.coord_class:g}")
        self._stack = stack
        return stack.cpu().numpy(), com, frames

    def gmm(self,
            n_components: int,
            covariance: str = 'diag',
            random_state: int = 1,
            plot_results: bool = False) -> Tuple[np.ndarray, List]:
        """
        Gaussian mixture model of the stack.  Returns the mean image of every class
        (max(class) x r x r x channels, NaN for an empty class), the list of each class's
        images, and an (N, 4) array of x, y, class (from 1) and frame.
        """
        clf = GaussianMixture(n_components=n_components, covariance_type=covariance,
                              random_state=random_state)
        classes = clf.fit_predict(self._stack.reshape(self.d0, -1)) + 1
        ncl = int(classes.max())
        cla = np.ndarray(shape=(ncl, int(self.r), int(self.r), self.nb_classes))
        cl_all = []
        for i in range(ncl):
            members = self.imgstack[classes == i + 1]
            cl_all.append(members)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)   # empty class: NaN mean
                cla[i] = np.mean(members, axis=0)
        if plot_results:
            self._plot_classes(cla, cl_all, n_components)
        com_frames = np.concatenate(
            (self.imgstack_com, classes[:, None], self.imgstack_frames[:, None]), axis=-1)
        return cla, cl_all, com_frames

    def _plot_classes(self, cla, cl_all, n_components):
        plt = _pyplot()
        if plt is None:
            return
        if self.nb_classes not in (1, 3):
            raise NotImplementedError("Can plot only images with 3 and 1 channels")
        rows = int(np.ceil(n_components / 5))
        cols = int(np.ceil(len(cla) / rows))
        fig = plt.figure(figsize=(4 * cols, 4 * (1 + rows // 2)))
        for i, img in enumerate(cla):
            ax = fig.add_subplot(rows, cols, i + 1)
            if self.nb_classes == 3:
                ax.imshow(img, interpolation='gaussian')
            else:
                ax.imshow(img[..., 0], cmap='seismic', interpolation='gaussian')
            ax.axis('off')
            ax.set_title(f"Class {i + 1}\nCount: {len(cl_all[i])}")
        plt.subplots_adjust(hspace=0.6, wspace=0.4)
        plt.show()

    def pca(self, n_components: int, random_state: int = 1,
            plot_results: bool = False) -> Tuple[np.ndarray]:
        _not_native("pca")

    def ica(self, n_components: int, random_state: int = 1,
            plot_results: bool = False) -> Tuple[np.ndarray]:
        _not_native("ica")

    def nmf(self, n_components: int, random_state: int = 1, plot_results: bool = False,
            **kwargs: int) -> Tuple[np.ndarray]:
        _not_native("nmf")

    def pca_gmm(self, n_components_gmm: int, n_components_pca: int, plot_results: bool = False,
                covariance_type: str = 'diag', random_state: int = 1) -> Tuple[np.ndarray, List]:
        _not_native("pca_gmm")

    def pca_scree_plot(self, plot_results: bool = True) -> np.ndarray:
        _not_native("pca_scree_plot")

    def pca_gmm_scree_plot(self, n_components_gmm: int, covariance_type: str = 'diag',
                           random_state: int = 1, plot_results: bool = True) -> List[np.ndarray]:
        _not_native("pca_gmm_scree_plot")

    def imblock_pca(self, n_components: int, random_state: int = 1, plot_results: bool = False,
                    **kwargs: int) -> Tuple[np.ndarray]:
        _not_native("imblock_pca")

    def imblock_ica(self, n_components: int, random_state: int = 1, plot_results: bool = False,
                    **kwargs: int) -> Tuple[np.ndarray]:
        _not_native("imblock_ica")

    def imblock_nmf(self, n_components: int, random_state: int = 1, plot_results: bool = False,
                    **kwargs: int) -> Tuple[np.ndarray]:
        _not_native("imblock_nmf")

    @classmethod
    def plot_decomposition_results(cls, components: np.ndarray, X_vec_t: np.ndarray,
                                   image_hw: Tuple = None, xy_centers: np.ndarray = None,
                                   plot_loading_maps: bool = True, **kwargs: int) -> None:
        _not_native("plot_decomposition_results")

    @classmethod
    def get_trajectory(cls,
                       coord_class_dict: Dict[int, np.ndarray],
                       start_coord: np.ndarray,
                       rmax: int) -> Tuple[np.ndarray]:
        """
        Follows one atom through the frames: in every frame (dictionary order) the nearest
        atom within `rmax` of the last position found is appended and becomes the new position.
        Returns the (n, 3) rows found and their frame keys.
        """
        rows, frames = [], []
        pos = start_coord
        for key, c in coord_class_dict.items():
            dist, j = spatial.cKDTree(c[:, :2]).query(pos, distance_upper_bound=rmax)
            if np.isinf(dist):
                continue
            rows.append(c[j])
            frames.append(key)
            pos = c[j][:2]
        flow = np.array(rows, dtype=np.float64).reshape(-1, 3)
        return flow, np.array(frames)

    def get_all_trajectories(self,
                             min_length: int = 0,
                             run_gmm: bool = False,
                             rmax: int = 10,
                             **kwargs: Union[int, str]) -> Dict:
        """
        Trajectories of every atom of the first frame (longer than `min_length`), with the
        GMM class of each point when `run_gmm` (kwargs n_components = 5, covariance = 'diag',
        random_state = 1); returns {"trajectories", "frames"[, "gmm_components"]}.
        """
        if run_gmm:
            gmm_comps, _, com_frames = self.gmm(kwargs.get("n_components", 5),
                                                kwargs.get("covariance", "diag"),
                                                kwargs.get("random_state", 1))
            classes = com_frames[:, -2]
        else:
            classes = np.zeros(len(self.imgstack_frames))
        per_frame = {}
        for f in self.imgstack_frames:
            sel = self.imgstack_frames == f
            per_frame[f] = np.concatenate((self.imgstack_com[sel], classes[sel][:, None]), axis=-1)
        first = per_frame[next(iter(per_frame))]
        trajectories, frames = [], []
        for start in first[:, :2]:
            flow, fr = self.get_trajectory(per_frame, start, rmax)
            if len(flow) > min_length:
                trajectories.append(flow)
                frames.append(fr)
        result = {"trajectories": trajectories, "frames": frames}
        if run_gmm:
            result["gmm_components"] = gmm_comps
        return result

    @classmethod
    def renumerate_classes(cls, classes: np.ndarray) -> np.ndarray:
        """Maps the distinct values of `classes` (in sorted order) to 0, 1, 2, ..."""
        _, inverse = np.unique(classes, return_inverse=True)
        return inverse.reshape(-1).astype(np.int64)

    def transition_matrix(self,
                          n_components: int,
                          covariance: str = 'diag',
                          random_state: int = 1,
                          rmax: int = 10,
                          min_length: int = 0,
                          sum_all_transitions: bool = False) -> Dict:
        """
        GMM classes along every trajectory and the Markov transition matrix of each
        (get_all_trajectories with run_gmm plus "transitions"; "all_transitions" as well when
        `sum_all_transitions`).
        """
        result = self.get_all_trajectories(min_length, run_gmm=True, n_components=n_components,
                                           rmax=rmax, covariance=covariance,
                                           random_state=random_state)
        result["transitions"] = [calculate_transition_matrix(self.renumerate_classes(t[:, -1]))
                                 for t in result["trajectories"]]
        if sum_all_transitions:
            result["all_transitions"] = sum_transitions(result, n_components)
        return result


def calculate_transition_matrix(trace: Union[List, np.ndarray]) -> np.ndarray:
    """Row-normalised counts of the transitions trace[t] -> trace[t + 1] (states 0..max)."""
    trace = np.asarray(trace, dtype=np.int64)
    n = 1 + int(trace.max())
    M = np.zeros((n, n))
    np.add.at(M, (trace[:-1], trace[1:]), 1.0)
    s = M.sum(axis=1, keepdims=True)
    return np.divide(M, s, out=M, where=s > 0)


def sum_transitions(trans_dict: Dict, msize: int,
                    plot_results: bool = False, **kwargs: int) -> np.ndarray:
    """
    Adds the per-trajectory transition matrices of `trans_dict` (the output of
    imlocal.transition_matrix) into one msize x msize matrix over the GMM classes and normalises
    its rows.
    """
    total = np.zeros((msize, msize))
    for traj, trans in zip(trans_dict["trajectories"], trans_dict["transitions"]):
        states = np.unique(traj[:, -1]).astype(np.int64) - 1
        total[np.ix_(states, states)] += trans
    total = total / total.sum(axis=1, keepdims=True)
    if plot_results:
        plt = _pyplot()
        if plt is not None:
            plt.figure(figsize=(6, 6))
            plt.imshow(total, cmap="Reds")
            plt.colorbar()
            plt.title("Transition matrix")
            plt.show()
    return total


def update_classes(coordinates: Union[Dict[int, np.ndarray], np.ndarray],
                   nn_input: np.ndarray,
                   method: str = 'threshold',
                   **kwargs: float) -> Dict[int, np.ndarray]:
    """
    New atom classes from the intensity around each position ('threshold': kwarg thresh;
    'kmeans': kwarg n_components, native KMeans) or from a GMM of the sub-images around each
    position ('gmm_local': kwargs n_components, window_size, coord_class).  kwarg window_size
    (default 3) is the side of the intensity square.  Returns updated copies of the coordinates.
    """
    if method not in ("threshold", "kmeans", "meanshift", "gmm_local"):
        raise NotImplementedError(
            "Choose between 'threshold', 'kmeans', 'meanshift' and 'gmm_local' methods")
    if method == "meanshift":
        raise NotImplementedError("update_classes(method='meanshift') is not on the native path; "
                                  "use 'threshold', 'kmeans' or 'gmm_local'")
    if isinstance(coordinates, np.ndarray):
        coordinates = {0: coordinates}
    if np.ndim(nn_input) == 2:
        nn_input = nn_input[None, ..., None]
    elif np.ndim(nn_input) == 3:
        # (frames, h, w) when the last axis is long, (h, w, channels) otherwise (<= 10 classes)
        nn_input = nn_input[..., None] if nn_input.shape[-1] > 10 else nn_input[None, ...]
    updated = copy.deepcopy(coordinates)
    if method == "threshold":
        thresh = kwargs.get("thresh")
        if thresh is None:
            raise AttributeError("Specify intensity threshold value ('thresh'), e.g. thresh=.5")
        intensities = get_intensities(updated, nn_input, kwargs.get("window_size", 3))
        for i, v in zip(updated, intensities):
            updated[i][:, -1] = (v >= thresh).astype(updated[i].dtype)
        plt = _pyplot()
        if plt is not None:
            plt.figure(figsize=(5, 5))
            counts = plt.hist(np.concatenate(intensities), bins=20)[0]
            plt.vlines(thresh, counts.min(), counts.max(), linestyle='dashed', color='red',
                       label='threshold')
            plt.legend()
            plt.title('Intensities (arb. units)')
            plt.show()
    elif method == "kmeans":
        n_components = kwargs.get("n_components")
        if n_components is None:
            raise AttributeError("Specify number of components ('n_components')")
        intensities = get_intensities(updated, nn_input, kwargs.get("window_size", 3))
        km = KMeans(n_clusters=n_components, random_state=42).fit(
            np.concatenate(intensities)[:, None])
        for i, v in zip(updated, intensities):
            updated[i][:, -1] = km.predict(v[:, None])
    else:
        n_components, window_size = kwargs.get("n_components"), kwargs.get("window_size")
        if n_components is None or window_size is None:
            raise AttributeError(
                "Specify number of components ('n_components') and window size ('window_size')")
        s = imlocal(nn_input, updated, window_size, kwargs.get("coord_class", 0))
        _, _, com_frames = s.gmm(n_components, plot_results=True)
        for i in updated:
            rows = com_frames[com_frames[:, -1] == float(i)][:, :3]
            rows[:, -1] -= 1
            updated[i] = rows
    return updated
