"""
Checkpoint loading with the reference's on-disk format (atomai/models/loaders.py:25-88): a
`*.tar` written by torch.save(meta_state_dict) holding the architecture kwargs, 'weights'
(state_dict with the reference's parameter names) and the pickled 'optimizer'.  Checkpoints
written by the reference (e.g. pretrained/bfo.tar, G_MD.tar) load unchanged.
"""
from typing import Type

import torch


def load_model(filepath: str):
    """Loads a trained AtomAI model from `filepath` (dispatch on meta['model_type'])."""
    device = 'cuda' if torch.cuda.is_available() else 'cpu'
    # The reference pickles the optimizer object itself; its class lives in torch.optim.
    meta = torch.load(filepath, map_location=device, weights_only=False)
    model_type = meta.get("model_type", "seg")
    if model_type in ("seg", "Seg"):
        return load_seg_model(meta)
    if model_type == "imspec":
        return load_imspec_model(meta)
    if model_type == "vae":
        return load_vae_model(meta)
    if model_type == "denoising_autoencoder":
        return load_denoising_autoencoder(meta)
    if model_type == "reg":
        return load_reg_model(meta)
    if model_type == "cls":
        return load_cls_model(meta)
    raise NotImplementedError(f"model_type '{model_type}' is not part of the atomai_b200 hot path")


def load_seg_model(meta_dict) -> Type["Segmentor"]:
    """Rebuilds a Segmentor from the stored kwargs and loads its weights (loaders.py:67-88)."""
    from .segmentor import Segmentor
    meta = dict(meta_dict)
    meta.pop("model_type", None)
    weights = meta.pop("weights")
    optimizer = meta.pop("optimizer", None)
    model_name = meta.pop("model")
    nb_classes = meta.pop("nb_classes")
    if "batchnorm" in meta and "batch_norm" not in meta:   # older checkpoints (G_MD.tar)
        meta["batch_norm"] = meta.pop("batchnorm")
    m = Segmentor(model_name, nb_classes, **meta)
    m.net.load_state_dict(weights)
    m.net.eval()
    m.optimizer = optimizer
    return m


def load_imspec_model(meta_dict):
    from .imspec import ImSpec
    meta = dict(meta_dict)
    meta.pop("model_type", None)
    weights = meta.pop("weights")
    optimizer = meta.pop("optimizer", None)
    in_dim, out_dim, latent_dim = meta.pop("in_dim"), meta.pop("out_dim"), meta.pop("latent_dim")
    m = ImSpec(in_dim, out_dim, latent_dim, **meta)
    m.net.load_state_dict(weights)
    m.net.eval()
    m.optimizer = optimizer
    return m


def load_vae_model(meta_dict):
    from .dgm import VAE, jrVAE, jVAE, rVAE
    meta = dict(meta_dict)
    meta.pop("model_type", None)
    coord = meta.get("coord", 0)
    enc, dec = meta.pop("encoder"), meta.pop("decoder")
    optimizer = meta.pop("optimizer", None)
    in_dim, latent_dim = meta.pop("in_dim"), meta.pop("latent_dim")
    meta.pop("coord", None)
    # any non-zero coord is an rVAE; coord == 3 adds translation; a non-empty discrete_dim makes
    # the joint models (atomai/models/loaders.py:163-195)
    joint = bool(meta.get("discrete_dim"))
    if coord:
        meta.pop("translation", None)
        m = (jrVAE if joint else rVAE)(in_dim, latent_dim, translation=(coord == 3), **meta)
    else:
        m = (jVAE if joint else VAE)(in_dim, latent_dim, **meta)
    if joint:
        m.kdict_["num_iter"] = meta.get("num_iter", 0)
    m.encoder_net.load_state_dict(enc)
    m.encoder_net.eval()
    m.decoder_net.load_state_dict(dec)
    m.decoder_net.eval()
    m.optim = optimizer
    return m


def load_denoising_autoencoder(meta_dict):
    """Rebuilds a DenoisingAutoencoder (loaders.py:198-235).  The defaults of missing keys are the
    reference loader's, including use_batch_norm=True where the class itself defaults to False."""
    from .denoiser import DenoisingAutoencoder
    meta = dict(meta_dict)
    meta.pop("model_type", None)
    weights = meta.pop("weights")
    optimizer = meta.pop("optimizer", None)
    m = DenoisingAutoencoder(
        encoder_filters=meta.pop("encoder_filters", [8, 16, 32, 64]),
        decoder_filters=meta.pop("decoder_filters", [64, 32, 16, 8]),
        encoder_layers=meta.pop("encoder_layers", [1, 2, 2, 2]),
        decoder_layers=meta.pop("decoder_layers", [2, 2, 2, 1]),
        use_batch_norm=meta.pop("use_batch_norm", True),
        upsampling_mode=meta.pop("upsampling_mode", 'nearest'),
        **meta)
    m.net.load_state_dict(weights)
    m.net.eval()
    m.optimizer = optimizer
    return m


def _regcls_kwargs(meta: dict) -> dict:
    # the checkpoint stores the image channels as 'in_channels'; the constructor takes
    # 'input_channels'
    meta.pop("model_type", None)
    if "in_channels" in meta:
        meta["input_channels"] = meta.pop("in_channels")
    return meta


def load_reg_model(meta_dict):
    """Rebuilds a Regressor from a 'reg' checkpoint (atomai/models/loaders.py:115-137)."""
    from .regcls import Regressor
    meta = _regcls_kwargs(dict(meta_dict))
    backbone = meta.pop("backbone")
    out_dim = meta.pop("out_dim")
    weights = meta.pop("weights")
    optimizer = meta.pop("optimizer", None)
    model = Regressor(backbone, out_dim, **meta)
    model.net.load_state_dict(weights)
    if optimizer is not None:
        model.optimizer = optimizer
    model.net.eval()
    return model


def load_cls_model(meta_dict):
    """Rebuilds a Classifier from a 'cls' checkpoint (atomai/models/loaders.py:140-160)."""
    from .regcls import Classifier
    meta = _regcls_kwargs(dict(meta_dict))
    backbone = meta.pop("backbone")
    nb_classes = meta.pop("nb_classes")
    weights = meta.pop("weights")
    optimizer = meta.pop("optimizer", None)
    model = Classifier(backbone, nb_classes, **meta)
    model.net.load_state_dict(weights)
    if optimizer is not None:
        model.optimizer = optimizer
    model.net.eval()
    return model
