"""
Loader for the UNMODIFIED reference (pycroscopy/atomai v0.8.1) as installed by

    python -m pip install --no-index --no-build-isolation --no-deps --find-links /opt/wheelhouse \
        --target baseline/_ref <copy of /root/reference>

(`baseline/_ref/` is git-ignored but travels to the GPU box).  The image lacks four of the
reference's import-time dependencies (matplotlib, skimage, mendeleev, gpytorch; SURVEY.md §8c,
Appendix A), none of which is on the Segmentor / VAE / ImSpec code path: they are replaced by
inert stub modules so that `import atomai` runs the reference's own code unchanged.

Used by bench.py's `--impl reference` (CPU) and `--impl torch-cuda` (stock PyTorch/cuDNN on the
GPU) arms and by oracle/ref_shim.py (golden generation).  Nothing under atomai_b200/ imports it.
"""
import os
import sys
import types
from unittest.mock import MagicMock

HERE = os.path.dirname(os.path.abspath(__file__))
VENDORED = os.path.join(HERE, "_ref")


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return MagicMock(name=f"{self.__name__}.{name}")


def _stub(name):
    m = _Stub(name)
    m.__path__ = []
    sys.modules[name] = m
    return m


def _importable(name):
    import importlib.util
    try:
        return importlib.util.find_spec(name) is not None
    except (ImportError, ValueError):
        return False


def import_reference(root: str = VENDORED):
    """Returns the reference's `atomai` package imported from `root` (default: baseline/_ref)."""
    import torch
    if "atomai" in sys.modules:
        f = getattr(sys.modules["atomai"], "__file__", "") or ""
        if f.startswith(os.path.abspath(root)):
            return sys.modules["atomai"]
        raise RuntimeError(f"a different `atomai` is already imported from {f}")
    if not os.path.isdir(os.path.join(root, "atomai")):
        raise FileNotFoundError(f"reference not installed under {root} (see DESIGN.md §5)")
    sys.path.insert(0, root)
    if not _importable("matplotlib"):
        for n in ["matplotlib", "matplotlib.pyplot", "matplotlib.gridspec", "matplotlib.cm",
                  "matplotlib.patches", "mpl_toolkits", "mpl_toolkits.axes_grid1"]:
            _stub(n)
        plt = sys.modules["matplotlib.pyplot"]
        plt.subplots = lambda *a, **k: (MagicMock(), MagicMock())
        sys.modules["matplotlib"].pyplot = plt
    if not _importable("skimage"):
        for n in ["skimage", "skimage.exposure", "skimage.util"]:
            _stub(n)
    for n in ["mendeleev", "progressbar"]:
        if not _importable(n):
            _stub(n)
    if not _importable("gpytorch"):
        g = _stub("gpytorch")

        class ExactGP(torch.nn.Module):
            pass
        for sub, attrs in {"models": {"ExactGP": ExactGP},
                           "distributions": {"MultivariateNormal": object},
                           "likelihoods": {"Likelihood": object, "GaussianLikelihood": object},
                           "kernels": {"Kernel": object}}.items():
            m = _stub(f"gpytorch.{sub}")
            for k, v in attrs.items():
                setattr(m, k, v)
            setattr(g, sub, m)
    import atomai  # noqa
    return atomai
