"""
BaseVAE / VAE — user-facing variational autoencoder (atomai/models/dgm/vae.py:28-747) on the
native sm_90a path.  Kept: construction kwargs, encode / decode / reconstruct, fit, save_model,
loss history.  The plotting helpers (manifold2d, visualize_manifold_learning, ...) depend on
matplotlib and are outside the hot-path scope (SURVEY.md §2.1).
"""
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from ...losses_metrics.vi_losses import vae_loss
from ...nets import init_VAE_nets
from ...trainers.vitrainer import viBaseTrainer
from ...utils.coords import imcoordgrid
from ...utils.nn import set_train_rng


def _host(y) -> np.ndarray:
    if isinstance(y, torch.Tensor):
        return y.detach().cpu().numpy()
    return np.asarray(y)


def host_labels(y, nb_classes: int) -> np.ndarray:
    """Class labels (int, array-like or tensor) as a 1-d int64 host array, checked against
    nb_classes the way the reference's to_onehot does (atomai/utils/preproc.py:916-923), and
    additionally refused when negative or not integral."""
    y = _host(y).reshape(-1)
    if y.dtype == np.bool_ or not (np.issubdtype(y.dtype, np.integer)
                                   or np.issubdtype(y.dtype, np.floating)):
        raise ValueError(f"class labels must be integers, got dtype {y.dtype}")
    if y.size and y.max() >= nb_classes:
        raise AssertionError(
            "Labelling must start from 0 and "
            "maximum label value must be less than total number of classes")
    if np.issubdtype(y.dtype, np.floating) and not np.all(np.floor(y) == y):
        raise ValueError("class labels must be integers, got non-integral values")
    if y.size and y.min() < 0:
        raise ValueError(f"class labels must be non-negative, got {y.min()}")
    return y.astype(np.int64)


class BaseVAE(viBaseTrainer):
    """
    General class for VAE models (atomai/models/dgm/vae.py:28-103).

    Args: in_dim, latent_dim, nb_classes, coord (0: VAE, 1: rotation, 2: translation,
    3: rotation + translation), discrete_dim (sizes of the Gumbel-softmax latents of jVAE /
    jrVAE), seed, and the **kwargs of init_VAE_nets (conv_encoder, conv_decoder, numlayers_*,
    numhidden_*, ...).
    """
    def __init__(self, in_dim: Tuple[int], latent_dim: int, nb_classes: int = 0, coord: int = 0,
                 discrete_dim: Optional[List] = None, seed: int = 0,
                 **kwargs: Union[int, bool]) -> None:
        super(BaseVAE, self).__init__()
        msg = ("You must specify the input dimensions and pass them as a tuple. "
               "For images, specify (height, width) or (height, width, channels)" +
               " if multiple channels. For spectra, specify (length,)")
        if in_dim is None or not isinstance(in_dim, (tuple, list)):
            raise AssertionError(msg)
        if isinstance(in_dim, tuple) and not isinstance(in_dim[0], int):
            raise AssertionError(msg)
        set_train_rng(seed)
        np.random.seed(seed)
        self.in_dim = in_dim
        self.z_dim = latent_dim
        if discrete_dim:
            self.z_dim = self.z_dim + sum(discrete_dim)
        self.discrete_dim = discrete_dim
        if coord:
            if len(in_dim) not in (2, 3):
                raise NotImplementedError(
                    "VAE with rotation and translational invariance are " +
                    "available only for 2D image data")
            self.z_dim = self.z_dim + coord
            self.x_coord = imcoordgrid(in_dim).to(self.device)
        self.nb_classes = nb_classes
        encoder_net, decoder_net, self.metadict = init_VAE_nets(
            in_dim, latent_dim, coord, discrete_dim, nb_classes, **kwargs)
        self.set_model(encoder_net, decoder_net)
        self.sigmoid_out = self.metadict["sigmoid_out"]
        self.coord = coord
        self.kdict_ = {"num_iter": 0}
        self.loss = "mse"

    # ------------------------------------------------------------------ inference API
    def encode_(self, x_new: Union[np.ndarray, torch.Tensor], **kwargs: int
                ) -> Tuple[np.ndarray]:
        """Encodes input data batch-by-batch; returns (z_mean, z_sd) numpy arrays, and for the
        joint VAEs also the (N, sum(discrete_dim)) alphas (vae.py:105-176)."""
        if isinstance(x_new, np.ndarray):
            x_new = torch.from_numpy(x_new).float()
        if (x_new.ndim == len(self.in_dim) == 2 or x_new.ndim == len(self.in_dim) == 3):
            x_new = x_new.unsqueeze(0)
        num_batches = kwargs.get("num_batches", 10)
        batch_size = max(len(x_new) // num_batches, 1)
        self.encoder_net.eval()
        mus, sds, alphas = [], [], []
        with torch.no_grad():
            for i in range(0, len(x_new), batch_size):
                z_mean, z_logsd, *alpha = self.encoder_net(x_new[i:i + batch_size].to(self.device))
                mus.append(z_mean.cpu())
                sds.append(torch.exp(z_logsd).cpu())
                if alpha:
                    alphas.append(torch.cat(alpha, 1).cpu())
        if alphas:
            return torch.cat(mus).numpy(), torch.cat(sds).numpy(), torch.cat(alphas).numpy()
        return torch.cat(mus).numpy(), torch.cat(sds).numpy()

    def encode(self, x_new, **kwargs: int) -> Tuple[np.ndarray]:
        return self.encode_(x_new, **kwargs)

    def encode_image_(self, img: np.ndarray, **kwargs: int) -> Tuple[np.ndarray, np.ndarray]:
        """Crops and encodes a sub-image around each pixel of a 2-D image (vae.py:300-344); the
        window size is the VAE's input size.  The reference extracts the windows coordinate by
        coordinate on the CPU; here the image lives on the GPU, every batch of windows is one
        gather kernel and goes straight into the encoder.  Returns the cropped original image
        and the (h', w', z_dim) encoded array (cropping is due to the finite window size)."""
        if self.discrete_dim:
            raise NotImplementedError("encode_image_ of the joint VAEs (the reference's cannot "
                                      "unpack their three outputs either)")
        from ...utils.img import crop_borders, extract_subimages_cuda, get_coord_grid
        num_batches = kwargs.get("num_batches", 10)
        inf = int(1e5)
        img_to_encode = np.array(img, dtype=np.float64, copy=True)
        dev_img = torch.from_numpy(img_to_encode.astype(np.float32))[None, ..., None].to(self.device)
        coordinates = get_coord_grid(img_to_encode, 1, return_dict=False)
        batch_size = max(coordinates.shape[0] // num_batches, 1)
        encoded_img = -inf * np.ones((*img_to_encode.shape, self.z_dim))
        self.encoder_net.eval()
        for i in range(0, coordinates.shape[0], batch_size):
            coord_i = coordinates[i:i + batch_size]
            subimgs_i, com_i, _ = extract_subimages_cuda(dev_img, coord_i, self.in_dim[0])
            if len(subimgs_i) == 0:
                continue
            if len(self.in_dim) == 2:
                subimgs_i = subimgs_i[..., 0]
            zs = []
            with torch.no_grad():
                for j in range(0, len(subimgs_i), 2048):
                    zs.append(self.encoder_net(subimgs_i[j:j + 2048])[0])
            z_mean = torch.cat(zs).cpu().numpy()
            encoded_img[com_i[:, 0].astype(int), com_i[:, 1].astype(int)] = z_mean
        img_to_encode[encoded_img[..., 0] == -inf] = 0
        img_to_encode = crop_borders(img_to_encode[..., None], 0)
        encoded_img = crop_borders(encoded_img, -inf)
        return img_to_encode[..., 0], encoded_img

    def encode_images(self, imgdata: np.ndarray, **kwargs: int) -> Tuple[np.ndarray, np.ndarray]:
        """encode_image_ for every image of a stack (vae.py:267-298)."""
        if (imgdata.ndim == len(self.in_dim) == 2 or imgdata.ndim == len(self.in_dim) == 3):
            imgdata = np.expand_dims(imgdata, axis=0)
        imgdata_encoded, imgdata_ = [], []
        for i, img in enumerate(imgdata):
            img_, img_encoded = self.encode_image_(img, **kwargs)
            imgdata_encoded.append(img_encoded)
            imgdata_.append(img_)
        return np.array(imgdata_), np.array(imgdata_encoded)

    def decode(self, z_sample: Union[np.ndarray, torch.Tensor],
               y: Optional[Union[int, np.ndarray, torch.Tensor]] = None) -> np.ndarray:
        """Decodes latent vector(s) into images (vae.py:178-221).  For coord > 0 the decoder is
        evaluated on the untransformed pixel grid, as in the reference.  A class-conditioned model
        needs `y`: an int, a 0-d / 1-d array or a tensor of labels; a single label applies to
        every row of z_sample."""
        if isinstance(z_sample, np.ndarray):
            z_sample = torch.from_numpy(z_sample).float()
        if z_sample.ndim == 1:
            z_sample = z_sample[None]
        if y is not None or self.nb_classes:
            if y is None:
                raise ValueError(f"this model is class-conditioned (nb_classes={self.nb_classes}): "
                                 "pass the label(s) y to decode")
            labels = host_labels(y, self.nb_classes)
            if labels.size == 1:
                labels = np.broadcast_to(labels.reshape(1), (len(z_sample),))
            elif len(labels) != len(z_sample):
                raise ValueError(f"got {len(labels)} labels for {len(z_sample)} latent vectors")
            onehot = torch.from_numpy(np.eye(self.nb_classes, dtype=np.float32)[labels])
            z_sample = torch.cat([z_sample.float().cpu(), onehot], 1)
        z_sample = z_sample.to(self.device)
        self.decoder_net.eval()
        with torch.no_grad():
            if self.coord > 0:
                x_decoded = self.decoder_net.decode(z_sample, None, None)
            else:
                x_decoded = self.decoder_net(z_sample)
        if self.sigmoid_out:
            x_decoded = torch.sigmoid(x_decoded)
        return x_decoded.cpu().numpy()

    def reconstruct(self, x_new, **kwargs: int) -> np.ndarray:
        """encode -> decode of the latent mean (vae.py:223-271).  A class-conditioned model needs
        `label` (one label for every row, or one per row) and decodes with its one-hot appended.
        The joint VAEs append the encoded alphas, or with `label` (an int, or one int per discrete
        head) the one-hot class vector."""
        if not self.discrete_dim:
            label = kwargs.get("label")
            if self.nb_classes and label is None:
                raise ValueError(f"this model is class-conditioned (nb_classes={self.nb_classes}): "
                                 "pass label=... to reconstruct")
            if label is not None:
                host_labels(label, self.nb_classes)
            z_mean, _ = self.encode(x_new, **kwargs)
            if self.coord > 0:
                z_mean = z_mean[:, self.coord:]
            return self.decode(z_mean, label)
        z_mean, _, alphas = self.encode(x_new, **kwargs)
        z_mean = z_mean[:, self.coord:]
        label = kwargs.get("label")
        if label is not None:
            labels = [label] if np.ndim(label) == 0 else list(label)
            if len(labels) != len(self.discrete_dim):
                raise ValueError("pass one label per discrete latent")
            onehot = np.concatenate([np.eye(d, dtype=np.float32)[int(k)]
                                     for k, d in zip(labels, self.discrete_dim)])
            alphas = np.broadcast_to(onehot, (len(z_mean), len(onehot)))
        return self.decode(np.concatenate([z_mean, alphas], 1).astype(np.float32))

    # ------------------------------------------------------------------ training helpers
    def _check_inputs(self, X_train, y_train=None, X_test=None, y_test=None) -> None:
        if self.in_dim != tuple(X_train.shape[1:]) and list(self.in_dim) != list(X_train.shape[1:]):
            raise RuntimeError("Training data must have the same dimensions as in_dim")
        if X_test is not None and tuple(X_test.shape[1:]) != tuple(X_train.shape[1:]):
            raise RuntimeError("Test data must have the same dimensions as the training data")
        if y_train is not None and self.nb_classes == 0:
            raise RuntimeError(
                "You must have forgotten to specify number of classes " +
                "during the initialization. Example of correct usage: " +
                "vae = VAE(in_dim=(28, 28), nb_classes=10)); " +
                "vae.fit(train_data, train_labels).")
        lbl_match = True
        if y_train is not None and y_test is None:
            lbl_match = self.nb_classes == len(np.unique(_host(y_train)))
        elif y_train is not None and y_test is not None:
            lbl_match = (self.nb_classes == len(np.unique(_host(y_train)))
                         == len(np.unique(_host(y_test))))
        if not lbl_match:
            raise RuntimeError(
                "The number of classes specified at initialization must be " +
                "equal the the number of classes in train and test labels")

    def _check_labels(self, X_test, y_train, y_test):
        """Labels of a class-conditioned fit, validated on the host and cast to int64 before any
        device work (the reference scatters them on the device: a negative or fractional label
        fails there, a missing one fails inside the decoder)."""
        if self.nb_classes:
            if y_train is None:
                raise ValueError(f"this model is class-conditioned (nb_classes={self.nb_classes}): "
                                 "pass the training labels y_train to fit")
            if X_test is not None and y_test is None:
                raise ValueError(f"this model is class-conditioned (nb_classes={self.nb_classes}): "
                                 "pass the test labels y_test with X_test")
        if y_train is not None:
            y_train = torch.from_numpy(host_labels(y_train, self.nb_classes))
        if y_test is not None:
            y_test = torch.from_numpy(host_labels(y_test, self.nb_classes))
        return y_train, y_test

    def _require_labels(self, y) -> None:
        if y is not None and not self.nb_classes:
            raise RuntimeError("labels were passed to a model built with nb_classes=0")
        if y is None and self.nb_classes:
            raise ValueError(f"this model is class-conditioned (nb_classes={self.nb_classes}): "
                             "its forward pass needs the labels y")

    def _onehot(self, y: torch.Tensor) -> torch.Tensor:
        """(B,) int64 labels (already validated) -> (B, nb_classes) float one-hot, on y's device."""
        return torch.zeros(len(y), self.nb_classes, device=y.device).scatter_(1, y.view(-1, 1), 1.0)

    def update_metadict(self):
        self.metadict["num_epochs"] = self.current_epoch
        self.metadict["num_iter"] = self.kdict_["num_iter"]

    def _fit_loop(self, _print_stats: bool = True, **kwargs) -> None:
        for e in range(self.training_cycles):
            self.current_epoch = e
            elbo_epoch = self.train_epoch()
            self.loss_history["train_loss"].append(elbo_epoch)
            if self.test_iterator is not None:
                self.loss_history["test_loss"].append(self.evaluate_model())
            if _print_stats:
                self.print_statistics(e)
            self.update_metadict()
            if kwargs.get("save_every_epoch", True):
                self.save_model(self.filename)


class VAE(BaseVAE):
    """
    Implements a standard Variational Autoencoder (atomai/models/dgm/vae.py:594-747).

    Example:
    >>> vae = VAE((28, 28), latent_dim=2, conv_encoder=True, conv_decoder=True)
    >>> vae.fit(imstack, training_cycles=100, batch_size=100)
    >>> z_mean, z_sd = vae.encode(imstack)
    """
    def __init__(self, in_dim: int = None, latent_dim: int = 2, nb_classes: int = 0,
                 seed: int = 0, **kwargs: Union[int, bool, str]) -> None:
        coord = kwargs.pop("coord", 0) if "coord" in kwargs else 0
        super(VAE, self).__init__(in_dim, latent_dim, nb_classes, coord, seed=seed, **kwargs)
        set_train_rng(seed)

    def elbo_fn(self, x, x_reconstr, *args, **kwargs) -> torch.Tensor:
        return vae_loss(self.loss, self.in_dim, x, x_reconstr, *args, **kwargs)

    def forward_compute_elbo(self, x: torch.Tensor, y: Optional[torch.Tensor] = None,
                             mode: str = "train", eps: Optional[torch.Tensor] = None
                             ) -> torch.Tensor:
        """VAE forward pass with ELBO (vae.py:661-687).  `y` (int64 labels, validated by fit)
        appends the one-hot class vector to the decoder input.  `eps` (optional) fixes the
        reparameterisation noise (tests)."""
        self._require_labels(y)
        grad = mode != "eval"
        with torch.set_grad_enabled(grad):
            z_mean, z_logsd = self.encoder_net(x)
            if grad:
                self.kdict_["num_iter"] += 1
            z_sd = torch.exp(z_logsd)
            z = z_mean + z_sd * eps if eps is not None else self.reparameterize(z_mean, z_sd)
            if y is not None:
                z = torch.cat((z, self._onehot(y)), -1)
            x_reconstr = self.decoder_net(z)
            return self.elbo_fn(x, x_reconstr, z_mean, z_logsd, **self.kdict_)

    def fit(self, X_train, y_train=None, X_test=None, y_test=None, loss: str = "mse", **kwargs):
        """Trains VAE model (vae.py:689-743): kwargs capacity, training_cycles, batch_size,
        filename.  With nb_classes > 0, y_train (and y_test with X_test) are the class labels
        0 .. nb_classes - 1 of the class-conditioned VAE."""
        self._check_inputs(X_train, y_train, X_test, y_test)
        y_train, y_test = self._check_labels(X_test, y_train, y_test)
        for k, v in kwargs.items():
            if k in ["capacity"]:
                self.kdict_[k] = v
        self.compile_trainer((X_train, y_train), (X_test, y_test) if X_test is not None else None,
                             **kwargs)
        self.loss = loss
        self._fit_loop(**kwargs)
