"""k_diffusion -- H100-native drop-in for the sampling hot path of crowsonkb/k-diffusion.

Same import surface as the reference for the path in scope (`sampling`, `layers.Denoiser`,
`external.DiscreteSchedule`, `config.load_config / make_model / make_denoiser_wrapper`,
`models.ImageTransformerDenoiserModelV2`, `models.ImageTransformerDenoiserModelV1`, `models.ImageDenoiserModelV1`, `augmentation.KarrasAugmentWrapper`); everything on the latent runs in libkdb200.so.
"""
from . import augmentation, config, evaluation, external, gns, layers, models, parallel, sampling, synth, utils
from .layers import Denoiser

__all__ = ["augmentation", "config", "evaluation", "external", "gns", "layers", "models", "parallel", "sampling", "synth", "utils", "Denoiser"]
