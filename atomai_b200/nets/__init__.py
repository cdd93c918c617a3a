from .blocks import ConvBlock, DilatedBlock, ResBlock, ResModule, UpsampleBlock
from .dae import DenoisingAutoencoderNet
from .ed import (SignalDecoder, SignalED, SignalEncoder, convDecoderNet, convEncoderNet,
                 coord_latent, fcDecoderNet, fcEncoderNet, init_imspec_model, init_VAE_nets,
                 jconvEncoderNet, jfcEncoderNet, rDecoderNet)
from .fcnn import ResHedNet, SegResNet, Unet, dilnet, init_fcnn_model
from .reg_cls import ClassifierNet, RegressorNet, init_cls_model, init_reg_model
from .gp import (DeepKernel, GPRegressionModel, ScaleToBounds, dense_gram, dense_rbf,
                 fcFeatureExtractor)

__all__ = ["ConvBlock", "UpsampleBlock", "DilatedBlock", "ResBlock", "ResModule", "Unet", "dilnet",
           "SegResNet", "ResHedNet", "init_fcnn_model", "DenoisingAutoencoderNet",
           "SignalEncoder", "SignalDecoder", "SignalED", "convEncoderNet", "convDecoderNet",
           "fcEncoderNet", "fcDecoderNet", "jfcEncoderNet", "jconvEncoderNet", "rDecoderNet", "coord_latent", "init_imspec_model",
           "init_VAE_nets", "fcFeatureExtractor", "DeepKernel", "dense_gram", "dense_rbf",
           "ScaleToBounds", "GPRegressionModel", "RegressorNet", "ClassifierNet",
           "init_reg_model", "init_cls_model"]
