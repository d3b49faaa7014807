"""KarrasAugmentWrapper (reference k_diffusion/augmentation.py:92-113).  The augmentation pipeline itself (training) is out of scope."""
import torch
from torch import nn

from . import _native
from .models.image_v1 import ImageDenoiserModelV1


class KarrasAugmentWrapper(nn.Module):
    """mapping_cond = cat([aug_cond or zeros(B, 9), mapping_cond]) for the inner model.

    Around a native ImageDenoiserModelV1 the concatenation happens inside the engine's conditioning kernel and the wrapper exposes
    the interface the sampler executor uses (engine, denoise, conditioning checks); any other inner model is called as in the
    reference."""

    def __init__(self, model):
        super().__init__()
        self.inner_model = model

    def is_unet(self):
        return isinstance(self.inner_model, ImageDenoiserModelV1)

    def forward(self, input, sigma, aug_cond=None, mapping_cond=None, **kwargs):
        if self.is_unet():
            if kwargs:
                return self.inner_model.forward(input, sigma, **kwargs)      # raises for the unsupported options
            return self.inner_model.run(input, sigma, 0.0, True, aug_cond, mapping_cond)
        if aug_cond is None:
            aug_cond = input.new_zeros([input.shape[0], 9])
        mapping_cond = aug_cond if mapping_cond is None else torch.cat([aug_cond, mapping_cond], dim=1)
        return self.inner_model(input, sigma, mapping_cond=mapping_cond, **kwargs)

    def param_groups(self, *args, **kwargs):
        return self.inner_model.param_groups(*args, **kwargs)

    # ------------------------------------------------------------------ native interface (Denoiser / sampler executor)
    def _native_loss(self, kind, input, noise, sigma, sigma_data, weight, aug_cond=None, mapping_cond=None, **kwargs):
        if aug_cond is None:
            aug_cond = input.new_zeros([input.shape[0], 9])
        mapping_cond = aug_cond if mapping_cond is None else torch.cat([aug_cond, mapping_cond], dim=1)
        return self.inner_model.native_loss(kind, input, noise, sigma, sigma_data, weight, mapping_cond=mapping_cond, **kwargs)

    def __getattr__(self, name):
        if name == "native_loss":   # Denoiser.loss: the inner model's native loss with the wrapper's conditioning, where it has one
            inner = self._modules["inner_model"]
            if isinstance(inner, ImageDenoiserModelV1):
                return _native.unet_has_no_derivative
            if hasattr(inner, "native_loss"):
                return self._native_loss
        if name in ("engine", "denoise", "levels", "resolved_precision", "_check_cond", "class_emb", "mapping_cond_in_proj",
                    "denoise_jvp", "denoise_vjp", "set_precision"):
            inner = self._modules["inner_model"]
            if isinstance(inner, ImageDenoiserModelV1):
                return getattr(_UNetView(self, inner), name)
        return super().__getattr__(name)


class _UNetView:
    """The wrapper's native interface: an ImageDenoiserModelV1 evaluated with the augment wrapper's conditioning."""

    class_emb = None

    def __init__(self, wrapper, unet):
        self.wrapper, self.unet = wrapper, unet

    @property
    def levels(self):
        return self.unet.levels

    @property
    def mapping_cond_in_proj(self):
        return True if self.unet.user_mapping_cond_dim(True) > 0 else None

    def engine(self):
        return self.unet.engine(augment=True)

    def resolved_precision(self):
        return self.unet.resolved_precision()

    def set_precision(self, precision):
        self.unet.set_precision(precision)
        return self.wrapper

    def _check_cond(self, class_cond, mapping_cond):
        self.unet.check_cond(True, class_cond, mapping_cond)

    def denoise(self, x, sigma, sigma_data, aug_cond=None, mapping_cond=None, out=None):
        return self.unet.run(x, sigma, float(sigma_data), True, aug_cond, mapping_cond, out=out)

    denoise_jvp = denoise_vjp = _native.unet_has_no_derivative
