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
