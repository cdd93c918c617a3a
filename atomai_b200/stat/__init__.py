from .decomposition import NMF, PCA, FastICA
from .mixture import MAX_COMPONENTS, GaussianMixture, KMeans
from .multivar import calculate_transition_matrix, imlocal, sum_transitions, update_classes


class SlidingFFTNMF:
    """Sliding-window FFT with NMF unmixing (atomai.stat.SlidingFFTNMF): not on the native path."""

    def __init__(self, window_size_x=None, window_size_y=None, window_step_x=None,
                 window_step_y=None, interpolation_factor=2, zoom_factor=2, hamming_filter=True,
                 components=4):
        raise NotImplementedError("SlidingFFTNMF is not on the native path yet")


class SpectralUnmixer:
    """Decomposition of hyperspectral data (atomai.stat.SpectralUnmixer): not on the native path."""

    def __init__(self, method: str = 'nmf', n_components: int = 4, normalize: bool = False,
                 **kwargs):
        raise NotImplementedError("SpectralUnmixer is not on the native path yet")


__all__ = ['imlocal', 'calculate_transition_matrix', 'sum_transitions', 'update_classes',
           'SlidingFFTNMF', 'SpectralUnmixer', 'GaussianMixture', 'KMeans', 'PCA', 'NMF', 'FastICA',
           'MAX_COMPONENTS']
