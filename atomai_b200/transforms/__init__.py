from .imaug import datatransform, imspec_augmentor, reg_augmentor, seg_augmentor

__all__ = ["datatransform", "seg_augmentor", "imspec_augmentor", "reg_augmentor"]
