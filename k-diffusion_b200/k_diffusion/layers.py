"""Karras et al. preconditioner (reference: k_diffusion/layers.py:45-90) on native kernels."""
import torch
from torch import nn

from . import _native, utils


class Denoiser(nn.Module):
    """D(x, sigma) = c_skip x + c_out F(c_in x, sigma).

    With an `ImageTransformerDenoiserModelV2` inside, the three scalings are folded into the
    engine's first and last kernels; any other `inner_model` is wrapped with two elementwise
    kernels (scale-in, combine).  `loss` (training) is out of scope.
    """

    def __init__(self, inner_model, sigma_data=1., weighting='karras', scales=1):
        super().__init__()
        self.inner_model = inner_model
        self.sigma_data = sigma_data
        self.scales = scales
        named = {'karras': torch.ones_like, 'soft-min-snr': self._weighting_soft_min_snr, 'snr': self._weighting_snr}
        if callable(weighting):
            self.weighting = weighting
        elif weighting in named:
            self.weighting = named[weighting]
        else:
            raise ValueError(f'Unknown weighting type {weighting}')

    def _weighting_soft_min_snr(self, sigma):
        return (sigma * self.sigma_data) ** 2 / (sigma ** 2 + self.sigma_data ** 2) ** 2

    def _weighting_snr(self, sigma):
        return self.sigma_data ** 2 / (sigma ** 2 + self.sigma_data ** 2)

    def get_scalings(self, sigma):
        var = sigma ** 2 + self.sigma_data ** 2
        return self.sigma_data ** 2 / var, sigma * self.sigma_data / var ** 0.5, 1 / var ** 0.5

    def loss(self, *args, **kwargs):
        raise NotImplementedError('training losses are out of scope for the H100 sampling path')

    def is_native(self):
        return hasattr(self.inner_model, 'denoise') and hasattr(self.inner_model, 'engine')

    def forward(self, input, sigma, **kwargs):
        _native.require_cuda(input, sigma)
        if self.is_native():
            return self.inner_model.denoise(input, sigma, self.sigma_data, **kwargs)
        x = _native.f32c(input)
        sig = _native.f32c(sigma).expand(x.shape[0]).contiguous()
        f = self.inner_model(_native.precond_scale_in(x, sig, float(self.sigma_data)), sigma, **kwargs)
        return _native.precond_combine(_native.f32c(f), x, sig, float(self.sigma_data))


class DenoiserWithVariance(Denoiser):
    """reference layers.py:93-101: differs from Denoiser in `loss` only (training, out of scope); sampling is identical."""


class SimpleLossDenoiser(Denoiser):
    """L_simple with the Karras et al. preconditioner (reference layers.py:104-113): differs from Denoiser in `loss` only."""


class FourierFeatures(nn.Module):
    """Random Fourier features buffer (layers.py:285-293); evaluated inside the engine's conditioning kernel."""

    def __init__(self, in_features, out_features, std=1.):
        super().__init__()
        assert out_features % 2 == 0
        self.register_buffer('weight', torch.randn([out_features // 2, in_features]) * std)
