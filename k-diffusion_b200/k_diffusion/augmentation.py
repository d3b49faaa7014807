"""KarrasAugmentationPipeline and KarrasAugmentWrapper (reference k_diffusion/augmentation.py:32-113).

The pipeline's warp runs on the GPU: one kdb_augment launch per batch forms each image's affine matrix from its draws and resamples it
(bicubic, numpy's 'reflect' border), where the reference runs one CPU skimage warp per image in the data-loader workers."""
import functools

import numpy as np
import torch
from torch import nn

from . import _native
from .models.image_v1 import ImageDenoiserModelV1


# the kinds of one image's 13 draws, in the reference's order: a0 (x-flip), the y-flip gate, a1, the scale gate, a2, the rotation gate,
# a3, the anisotropy gate, a4, a5, the translation gate, a6, a7
_DRAWS = ("randint", "rand", "randint", "rand", "randn", "rand", "rand", "rand", "rand", "randn", "rand", "randn", "randn")
_RANDINT = [k for k, d in enumerate(_DRAWS) if d == "randint"]
_RANDN = [k for k, d in enumerate(_DRAWS) if d == "randn"]


class KarrasAugmentationPipeline:
    """The reference's non-leaking augmentations (Karras et al. 2022): an x-flip with probability 1/2, then, each with probability a_prob,
    a y-flip, an isotropic scaling by a_scale ** N(0, 1), a rotation, an anisotropic scaling by a_aniso ** N(0, 1) along a random angle
    and a translation by a_trans * N(0, 1) of the image's extents; cond [9] describes the transform for the model's mapping network.

    `__call__(image)` keeps the reference's contract for one PIL image (a uint8 mode such as 'L' or 'RGB'): 13 scalar draws from torch's
    global CPU generator in the reference's order, then (image, image_orig, cond) as CPU fp32 tensors [C, H, W], [C, H, W], [9].  The warp
    runs on the current CUDA device, so a data loader that calls it needs CUDA in its worker processes.

    `augment(images, generator=None)` is the route for a training loop: a uint8 [B, C, H, W] CUDA batch (a PILToTensor dataset moved with
    .cuda()) -> (image, image_orig, cond) on its device, in one launch.  The draws are made on the device with torch, [B, 13] at once:
    the same law as the reference's per-image draws, not the same stream of numbers."""

    def __init__(self, a_prob=0.12, a_scale=2**0.2, a_aniso=2**0.2, a_trans=1/8, disable_all=False):
        self.a_prob = a_prob
        self.a_scale = a_scale
        self.a_aniso = a_aniso
        self.a_trans = a_trans
        self.disable_all = disable_all

    def __call__(self, image):
        d = torch.stack([torch.randint(2, []).float() if k == "randint" else torch.rand([]) if k == "rand" else torch.randn([])
                         for k in _DRAWS])
        x = np.asarray(image)
        if x.dtype != np.uint8 or x.ndim not in (2, 3):
            raise ValueError(f"expected an 8-bit PIL image (mode 'L', 'RGB', ...), got an array of {x.dtype} and shape {x.shape}")
        x = torch.from_numpy(x.reshape(x.shape[0], x.shape[1], -1).copy()).permute(2, 0, 1)
        device = torch.device("cuda", torch.cuda.current_device())
        out = self._run(x[None].contiguous().to(device), d[None].to(device))
        return tuple(t[0].cpu() for t in out)

    def augment(self, images, generator=None):
        _native.require_cuda(images)
        B = images.shape[0]
        draws = torch.rand(B, len(_DRAWS), generator=generator, device=images.device)
        draws[:, _RANDINT] = torch.randint(2, (B, len(_RANDINT)), generator=generator, device=images.device).float()
        draws[:, _RANDN] = torch.randn(B, len(_RANDN), generator=generator, device=images.device)
        return self._run(images, draws)

    def _run(self, images, draws, with_mat=False):
        return _native.augment(images, draws, self.a_prob, self.a_scale, self.a_aniso, self.a_trans, self.disable_all, with_mat)


class KarrasAugmentWrapper(_native.NativeLossCall, nn.Module):
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
            return_variance = kwargs.pop("return_variance", False)
            if kwargs:
                return self.inner_model.forward(input, sigma, **kwargs)      # raises for the unsupported options
            return self.inner_model.evaluate(return_variance, input, sigma, aug_cond, mapping_cond=mapping_cond, augment=True)
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
        """The inner model's training precision (image_transformer_v2 only; the U-Net, which trains at fp32 only, raises
        NotImplementedError)."""
        self.inner_model.set_train_precision(precision)
        return self

    def resolved_precision(self):
        return self.inner_model.resolved_precision()

    @property
    def native_loss(self):
        """Denoiser.loss: the inner model's native loss with the wrapper's conditioning, where it has one."""
        if self.is_unet():
            return functools.partial(self.inner_model.native_loss, augment=True)
        return self._native_loss if hasattr(self.inner_model, "native_loss") else None

    def _native_loss(self, kind, input, noise, sigma, sigma_data, weight, aug_cond=None, mapping_cond=None, **kwargs):
        return self.inner_model.native_loss(kind, input, noise, sigma, sigma_data, weight,
                                            mapping_cond=self._mapping_cond(input, aug_cond, mapping_cond), **kwargs)
