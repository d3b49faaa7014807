"""KarrasAugmentWrapper (reference k_diffusion/augmentation.py:92-113).  The augmentation pipeline itself (training) is out of scope."""
import functools

import torch
from torch import nn

from . import _native
from .models.image_v1 import ImageDenoiserModelV1


class KarrasAugmentWrapper(nn.Module):
    """mapping_cond = cat([aug_cond or zeros(B, 9), mapping_cond]) for the inner model.

    Around a native ImageDenoiserModelV1 the concatenation happens inside the engine's conditioning kernel and the wrapper has the
    U-Net's native front end, asked for the augmented evaluation; any other inner model is called as in the reference."""

    def __init__(self, model):
        super().__init__()
        self.inner_model = model

    def is_unet(self):
        return isinstance(self.inner_model, ImageDenoiserModelV1)

    def forward(self, input, sigma, aug_cond=None, mapping_cond=None, **kwargs):
        if self.is_unet():
            if kwargs:
                return self.inner_model.forward(input, sigma, **kwargs)      # raises for the unsupported options
            return self.native_eval(input, sigma, aug_cond, mapping_cond=mapping_cond).forward(0.0)
        return self.inner_model(input, sigma, mapping_cond=self._mapping_cond(input, aug_cond, mapping_cond), **kwargs)

    @staticmethod
    def _mapping_cond(input, aug_cond, mapping_cond):
        if aug_cond is None:
            aug_cond = input.new_zeros([input.shape[0], 9])
        return aug_cond if mapping_cond is None else torch.cat([aug_cond, mapping_cond], dim=1)

    def param_groups(self, *args, **kwargs):
        return self.inner_model.param_groups(*args, **kwargs)

    # ------------------------------------------------------------------ native interface (Denoiser / sampler executor)
    @property
    def native_eval(self):
        """The U-Net's front end for the wrapper's evaluation; None around any other model, which is not native through the wrapper."""
        return functools.partial(self.inner_model.native_eval, augment=True) if self.is_unet() else None

    def denoise(self, x, sigma, sigma_data, aug_cond=None, mapping_cond=None, out=None):
        """Fused Karras-preconditioned evaluation of the U-Net with the wrapper's conditioning."""
        return self.native_eval(x, sigma, aug_cond, mapping_cond=mapping_cond).forward(float(sigma_data), out)

    denoise_jvp = denoise_vjp = _native.unet_has_no_derivative

    def engine(self):
        """The U-Net's engine with the wrapper's conditioning: the engine the wrapper's evaluations run on."""
        return self.inner_model.engine(augment=True)

    def set_precision(self, precision):
        self.inner_model.set_precision(precision)
        return self

    def set_train_precision(self, precision):
        """The inner model's training precision (image_transformer_v2 only; the U-Net raises NotImplementedError)."""
        self.inner_model.set_train_precision(precision)
        return self

    def resolved_precision(self):
        return self.inner_model.resolved_precision()

    @property
    def native_loss(self):
        """Denoiser.loss: the inner model's native loss with the wrapper's conditioning, where it has one."""
        if self.is_unet():
            return _native.unet_has_no_derivative
        return self._native_loss if hasattr(self.inner_model, "native_loss") else None

    def _native_loss(self, kind, input, noise, sigma, sigma_data, weight, aug_cond=None, mapping_cond=None, **kwargs):
        return self.inner_model.native_loss(kind, input, noise, sigma, sigma_data, weight,
                                            mapping_cond=self._mapping_cond(input, aug_cond, mapping_cond), **kwargs)
