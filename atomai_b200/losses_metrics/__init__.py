from .losses import (BCEWithLogitsLoss, CrossEntropyLoss, MSELoss, dice_loss, focal_loss,
                     select_loss)
from .metrics import IoU
from .vi_losses import (infocapacity, joint_rvae_loss, joint_vae_loss, kld_discrete, kld_normal,
                        kld_rot, reconstruction_loss, rvae_loss, vae_loss)

__all__ = ["select_loss", "CrossEntropyLoss", "BCEWithLogitsLoss", "MSELoss", "dice_loss",
           "focal_loss", "IoU", "reconstruction_loss", "kld_normal", "kld_rot", "vae_loss",
           "rvae_loss", "infocapacity", "kld_discrete", "joint_vae_loss", "joint_rvae_loss"]
